"""rtx_trace_otf_many and rayopt_b200.tolerance_mtf on the device.  Needs a
GPU.

Each item's rays are traced with rtx_trace through the item's table (keep
last) and its OTF sums are checked against the long-double sums of those
stored rows (tests/otf_many_oracle.py): counts exactly, every component
within include/rtx.h's bound plus the oracle's own error.  Then against the
two existing OTF calls on the same rows, bit-for-bit determinism, the
analysis end to end against the optimiser's trial scorer, mtf_jacobian and
tolerance(), the C refusals, and a 4096-variant run in chunks."""
import copy
import ctypes as C
import time

import numpy as np
import pytest

import otf_many_oracle as om
import ref_shim
from rayopt_b200.engine import otf_bound, otf_spec
from test_gpu_tolerance import MODES, NS, case, stored_last, variants

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from rayopt_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


Z = {1: np.array([0.]), 5: np.array([0., 1e-2, -1e-2, 3e-3, -5e-4]),
     16: np.r_[0., 1e-2, -1e-2, np.linspace(-2e-2, 2e-2, 13)]}


def freqs(F, seed):
    return np.r_[0., np.random.default_rng(seed).uniform(-80, 160, F - 1)] if F > 1 \
        else np.array([41.5])


def check_items(eng, tables, bundles, items, centers, z, nu, dtype, exact, clip, rot0):
    """rtx_trace_otf_many against the oracle sums of every item's stored
    rows; returns the sums and counts"""
    S, n = eng.trace_otf_many(tables, bundles, items, centers, z, nu, clip=clip, rot0=rot0,
                              exact=exact)
    assert S.shape == (len(items), len(z), 2, len(nu)) and n.shape == (len(items), len(z))
    cache = {}
    for i, (t, b) in enumerate(items):
        N = bundles[b][2]
        if N == 0:
            assert (S[i] == 0).all() and (n[i] == 0).all()
            continue
        if (t, b) not in cache:
            cache[t, b] = stored_last(eng, tables[t], bundles[b][0], bundles[b][1], N, dtype,
                                      exact, clip, rot0)
        y, inc = cache[t, b]
        re, im, cnt, phi = om.sums(y, inc, None if centers is None else centers[i], z, nu)
        assert np.array_equal(n[i], cnt), (i, n[i], cnt)
        tol = ((om.device_bound(N, phi) + om.oracle_error(cnt, phi))*cnt)[:, None, None]
        assert np.all(np.abs(S[i].real - re.astype(float)) <= tol), i
        assert np.all(np.abs(S[i].imag - im.astype(float)) <= tol), i
    return S, n


def device_bundles(eng, rays, dtype, Ns=NS):
    host = [rays(max(N, 1), 10 + k) for k, N in enumerate(Ns)]
    return [(eng.to_device(y, dtype), eng.to_device(u, dtype), N) for (y, u), N in zip(host, Ns)]


def free(bundles):
    for y, u, _ in bundles:
        y.free(), u.free()


@pytest.mark.parametrize("K, F", [(1, 7), (5, 64), (16, 1)])
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("name", ["double_gauss", "cooke_asph", "mirror", "zoom", "tilted_start3"])
def test_sums_match_stored_rows(eng, systems, name, mode, K, F):
    """up to 8 tables, one bundle per N, items that repeat and interleave
    tables and bundles, centres absent (FP32) and present"""
    dtype, exact = MODES[mode]
    table, rot0, clip, rays = case(name, systems)
    tabs = variants(table, 8, 3)
    bundles = device_bundles(eng, rays, dtype)
    rng = np.random.default_rng(K + F)
    items = np.c_[rng.integers(0, 8, 10), rng.integers(0, len(NS), 10)]
    items[:len(NS), 1] = np.arange(len(NS))
    centers = None if mode == "f32" else rng.normal(0, 1e-2, (len(items), 2))
    try:
        check_items(eng, tabs, bundles, items, centers, Z[K], freqs(F, K), dtype, exact, clip,
                    rot0)
    finally:
        free(bundles)


@pytest.mark.parametrize("mode", list(MODES))
def test_many_frequencies(eng, systems, mode):
    dtype, exact = MODES[mode]
    table, rot0, clip, rays = case("double_gauss", systems)
    bundles = device_bundles(eng, rays, dtype, (1, 513, 1500))
    items = np.array([[0, 0], [1, 1], [0, 2], [1, 2]])
    centers = np.random.default_rng(1).normal(0, 1e-2, (4, 2))
    try:
        for F in (64, 256):
            check_items(eng, variants(table, 2, 1), bundles, items, centers, Z[5], freqs(F, F),
                        dtype, exact, clip, rot0)
    finally:
        free(bundles)


@pytest.mark.parametrize("mode", ["f64_fast", "f32"])
def test_large_table_restaged(eng, systems, mode):
    """a 256-surface table (92 KB in FP64) restaged between items that
    alternate tables, beside the 16 KB of staged rays"""
    dtype, exact = MODES[mode]
    table, rot0, clip, rays = case("plates256", systems)
    bundles = device_bundles(eng, rays, dtype, (513, 2000))
    items = np.array([[0, 0], [1, 1], [2, 0], [0, 1], [1, 0]])
    try:
        check_items(eng, variants(table, 3, 1), bundles, items, None, Z[5], freqs(7, 2), dtype,
                    exact, clip, rot0)
    finally:
        free(bundles)


@pytest.mark.parametrize("exact", [True, False])
def test_against_otf_rows_and_otf_jacobian_sums(eng, systems, exact):
    """on the same stored rows: rtx_otf_rows at nu_j = fl(j dnu) within the
    sum of both bounds, and rtx_otf_jacobian_sums (P = 0, qstride 3) at z = 0
    within both bounds; counts exactly"""
    from otf_jac_oracle import device_bound
    table, rot0, clip, rays = case("double_gauss", systems)
    y0, u0 = rays(70001, 3)
    dy, du = eng.to_device(y0), eng.to_device(u0)
    c = np.array([1e-3, .02])
    dnu, F = 7.25, 33
    nu = np.arange(F)*dnu
    S, n = eng.trace_otf_many(table[None], [(dy, du, None)], [[0, 0]], c[None], Z[5], nu,
                              clip=clip, exact=exact)
    y, inc = stored_last(eng, table, dy, du, len(y0), np.float64, exact, clip, rot0)
    _, _, cnt, phi = om.sums(y, inc, c, Z[5], nu)
    Y, I = eng.to_device(np.ascontiguousarray(y)), eng.to_device(np.ascontiguousarray(inc))
    try:
        s, k = eng.otf_rows(Y, I, otf_spec(Z[5], dnu, F, c), N=len(y))
        assert np.array_equal(k, n[0])
        tol = (om.device_bound(len(y), phi)*cnt + otf_bound(None, len(y), cnt, phi))[:, None, None]
        d = S[0] - s
        assert np.all(np.abs(d.real) <= tol) and np.all(np.abs(d.imag) <= tol), "otf_rows"
        assert np.isfinite(inc[:, 2][np.isfinite(y[:, 0])]).all()
        j = eng.otf_jacobian_sums(Y, None, nu, c, N=len(y))
        assert j["n"] == n[0, 0]
        tol = (om.device_bound(len(y), phi[0]) + device_bound(len(y), phi[0])[0])*cnt[0]
        assert np.all(np.abs((S[0, 0] - j["S"]).real) <= tol)
        assert np.all(np.abs((S[0, 0] - j["S"]).imag) <= tol)
    finally:
        for a in (dy, du, Y, I):
            a.free()


@pytest.mark.parametrize("mode", list(MODES))
def test_deterministic(eng, systems, mode):
    """an item's sums are the same bits in two calls, in another context,
    alone, among 1000 other items and under a permutation of the items"""
    from rayopt_b200.engine import Engine
    dtype, exact = MODES[mode]
    table, rot0, clip, rays = case("double_gauss", systems)
    tabs = variants(table, 16, 9)
    bundles = device_bundles(eng, rays, dtype, (70001, 4099, 600))
    rng = np.random.default_rng(2)
    items = np.c_[rng.integers(0, 16, 1001), rng.integers(0, 3, 1001)]
    centers = rng.normal(0, 1e-2, (1001, 2))
    nu = freqs(5, 3)

    def run(e, it, c):
        S, n = e.trace_otf_many(tabs, bundles, it, c, Z[5], nu, clip=clip, exact=exact)
        return S.tobytes(), n.tobytes(), S, n
    try:
        a = run(eng, items, centers)
        assert run(eng, items, centers)[:2] == a[:2]
        e2 = Engine(0)
        try:
            assert run(e2, items, centers)[:2] == a[:2]
        finally:
            e2.close()
        alone = run(eng, items[:1], centers[:1])
        assert alone[2].tobytes() == a[2][:1].tobytes() and alone[3].tobytes() == a[3][:1].tobytes()
        p = rng.permutation(1001)
        b = run(eng, items[p], centers[p])
        assert b[2].tobytes() == a[2][p].tobytes() and b[3].tobytes() == a[3][p].tobytes()
    finally:
        free(bundles)


def test_refusals_launch_and_allocate_nothing(eng, systems):
    """each refusal returns its code with no launch and no allocation; the
    outputs have host guard bands that stay untouched"""
    from rayopt_b200 import _lib
    table, _, clip, rays = case("double_gauss", systems)
    y, u = rays(1000, 1)
    dy, du = eng.to_device(y), eng.to_device(u)
    tabs = np.ascontiguousarray(variants(table, 2, 1))
    S = tabs.shape[1]
    eng.trace_otf_many(tabs, [(dy, du, None)], [[0, 0]], None, Z[5], freqs(7, 1))  # warm

    def call(nt=2, tables=tabs, S=S, dtype=0, nb=1, N=(1000,), y0=(dy.ptr,), u0=(du.ptr,),
             it=(0,), ib=(0,), centers=None, K=2, z=(0., 1e-2), F=3, nu=(0., 10., 20.),
             sums=True, count=True, flags=0):
        Na = np.ascontiguousarray(N, np.int64)
        ya = (C.c_void_p*len(y0))(*y0) if y0 is not None else None
        ua = (C.c_void_p*len(u0))(*u0) if u0 is not None else None
        ita, iba = np.ascontiguousarray(it, np.int32), np.ascontiguousarray(ib, np.int32)
        ca = None if centers is None else np.ascontiguousarray(centers, np.float64)
        za = None if z is None else np.ascontiguousarray(z, np.float64)
        fa = None if nu is None else np.ascontiguousarray(nu, np.float64)
        n = len(it)
        out = np.full(n*4*max(K, 1)*max(F, 1) + 64, 7.25)
        cnt = np.full(n*max(K, 1) + 8, -5, np.int64)
        rc = eng.lib.rtx_trace_otf_many(
            eng.ctx, nt, _lib.ptr(tables) if tables is not None else None, S, None, dtype, nb,
            _lib.ptr(Na), ya, ua, n, _lib.ptr(ita), _lib.ptr(iba), _lib.ptr(ca), 1, K,
            _lib.ptr(za), F, _lib.ptr(fa), _lib.ptr(out) if sums else None,
            _lib.ptr(cnt) if count else None, flags)
        return rc, out, cnt

    E_BAD, E_UNS = -1, -2
    bad_asph = tabs.copy()
    bad_asph["n_asph"][1, 3] = 11
    cases = [(dict(tables=None), E_BAD), (dict(sums=False), E_BAD), (dict(count=False), E_BAD),
             (dict(z=None), E_BAD), (dict(nu=None), E_BAD), (dict(nt=0), E_BAD),
             (dict(nb=0), E_BAD), (dict(S=0), E_BAD), (dict(S=257), E_BAD),
             (dict(it=(2,)), E_BAD), (dict(it=(-1,)), E_BAD), (dict(ib=(1,)), E_BAD),
             (dict(N=(-1,)), E_BAD), (dict(y0=(None,)), E_BAD), (dict(u0=(None,)), E_BAD),
             (dict(y0=None), E_BAD), (dict(dtype=7), E_BAD),
             (dict(K=0, z=(0.,)), E_BAD), (dict(K=17, z=np.zeros(17)), E_BAD),
             (dict(F=0, nu=(1.,)), E_BAD), (dict(F=257, nu=np.zeros(257)), E_BAD),
             (dict(z=(0., np.nan)), E_BAD), (dict(nu=(0., np.inf, 1.)), E_BAD),
             (dict(centers=[[0., np.nan]]), E_BAD),
             (dict(tables=bad_asph), E_UNS), (dict(dtype=1, flags=1), E_UNS)]
    try:
        for kw, want in cases:
            eng.sync()
            fb, launches = eng.free_bytes(), eng.launch_count()
            rc, out, cnt = call(**kw)
            assert rc == want, (kw, rc)
            assert eng.launch_count() == launches and eng.free_bytes() == fb, kw
            assert (out == 7.25).all() and (cnt == -5).all(), kw
        rc, out, cnt = call()                                        # guard bands
        assert rc == 0 and (out[24:] == 7.25).all() and (cnt[2:] == -5).all()
        assert cnt[0] > 0 and out[0] == cnt[0]                       # nu = 0: the count
        rc, out, cnt = call(N=(0,), y0=(None,), u0=(None,))          # N = 0: zeros
        assert rc == 0 and (out[:24] == 0).all() and (cnt[:2] == 0).all()
        fb = eng.free_bytes()
        rc, _, _ = call(N=(2**52,))                                  # 2^43 tile rows
        assert rc == _lib.RTX_E_NOMEM and eng.free_bytes() == fb
    finally:
        dy.free(), du.free()


def test_scale_and_chunking(eng, systems):
    """4096 variants x 9 bundles x 1e4 rays of the double Gauss at K = 1,
    F = 3: every ray that reaches the image counts, and a run chunked into
    launches of half the variants gives the same bits"""
    from rayopt_b200.tolerance import perturbed_tables
    from rayopt_b200.rays import aim_infinite, disc
    ent = systems["double_gauss"]
    nominal = np.stack(ent["tables"][:3])
    params = [(1, "curvature"), (2, "distance"), (4, "conic"), (6, "tilt_x")]
    deltas = np.random.default_rng(1).uniform(-1, 1, (4096, 4))*[1e-4, 1e-2, 1e-2, 1e-3]
    N = 10000
    bundles = []
    for h in range(3):
        for w in range(3):
            aim = ent["aim"][w][(0, 3, 5)[h]]
            y, u = aim_infinite(aim["field"], disc(N, h*3 + w), aim["z"], aim["p"],
                                ent["object_angle"])
            bundles.append((eng.to_device(y), eng.to_device(u), N))
    V, H, W = 4096, 3, 3
    vv, hh, ww = np.meshgrid(np.arange(V), np.arange(H), np.arange(W), indexing="ij")
    items = np.stack([vv*W + ww, hh*W + ww], -1).reshape(-1, 2)
    nu = np.array([10., 30., 50.])

    def run(step):
        S, n = [], []
        for v0 in range(0, V, step):
            t = perturbed_tables(nominal, params, deltas[v0:v0 + step])
            k = len(t)
            it = items[v0*H*W:(v0 + k)*H*W].copy()
            it[:, 0] -= v0*W
            s, c = eng.trace_otf_many(t.reshape(k*W, -1), bundles, it, None, Z[1], nu, clip=True)
            S.append(s), n.append(c)
        return np.concatenate(S), np.concatenate(n)

    try:
        t0 = time.perf_counter()
        a = run(V)
        wall = time.perf_counter() - t0
        ms = eng.last_kernel_ms()
        b = run(V//2)
        assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes()
        assert (a[1] > 0).all() and (a[1] <= N).all()
        print("4096 x 9 x 1e4: kernel %.2f ms, call %.1f ms" % (ms, 1e3*wall))
    finally:
        free(bundles)


# ---- rayopt_b200.tolerance_mtf end to end on the reference's Cooke triplet ---
needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="no reference tree staged")
HEIGHTS = (0., .7, 1.)


def cooke():
    from test_gpu_optimize import cooke as c
    return c()


def cooke_case(s):
    from test_gpu_optimize import cooke_params
    from rayopt_b200.mtf import default_dnu
    params = cooke_params(s)
    rng = np.random.default_rng(4)
    deltas = np.r_[np.zeros((1, len(params))), rng.uniform(-1, 1, (6, len(params)))*1e-3]
    return params, deltas, np.arange(1, 5)*default_dnu(s, 8)


@needs_ref
def test_poly_mtf_matches_trial_scorer_and_mtf_jacobian(eng):
    """the poly MTF at defocus 0 against optimize._trial_mtf on the same
    deltas within both bounds; the nominal row against mtf_jacobian's otf;
    chunking does not change a bit"""
    from rayopt_b200 import optimize as opt
    from rayopt_b200.tolerance import tolerance_mtf
    s = cooke()
    params, deltas, nu = cooke_case(s)
    sw = np.ones(len(s.wavelengths))
    res = tolerance_mtf(copy.deepcopy(s), params, deltas, nu, HEIGHTS, nrays=2000, engine=eng,
                        targets=.2)
    B = opt._Bundles(copy.deepcopy(s), HEIGHTS, s.wavelengths, 2000, "hexapolar", eng, False)
    try:
        M = opt._trial_mtf(eng, B, params, deltas, nu, sw, True, False)
    finally:
        B.close()
    assert res["poly_mtf"].shape == (len(deltas), 3, 1, 2, 4)
    assert np.allclose(res["poly_mtf"][:, :, 0], M, rtol=0, atol=1e-12, equal_nan=True)
    j = opt.mtf_jacobian(copy.deepcopy(s), params, nu, HEIGHTS, nrays=2000, engine=eng)
    assert np.array_equal(res["count"][0, :, :, 0], j["n"].astype(np.int64))
    assert np.allclose(res["otf"][0, :, :, 0], j["otf"], rtol=0, atol=1e-12)
    again = tolerance_mtf(copy.deepcopy(s), params, deltas, nu, HEIGHTS, nrays=2000, engine=eng,
                          targets=.2, chunk=2)
    for k in ("otf", "count", "poly", "passed", "yield"):
        assert np.asarray(again[k]).tobytes() == np.asarray(res[k]).tobytes(), k
    assert np.array_equal(res["yield"], res["passed"].mean(0))


@needs_ref
def test_focus_matches_tolerance(eng):
    """compensate="focus" gives tolerance()'s focus shifts bit for bit"""
    import rayopt_b200
    s = cooke()
    params, deltas, nu = cooke_case(s)
    a = rayopt_b200.tolerance_mtf(copy.deepcopy(s), params, deltas, nu, HEIGHTS, nrays=500,
                                  defocus=(0., 1e-2), compensate="focus", engine=eng)
    b = rayopt_b200.tolerance(copy.deepcopy(s), params, deltas, HEIGHTS, nrays=500,
                              compensate="focus", engine=eng)
    assert a["focus"].tobytes() == b["focus"].tobytes()
    assert a["otf"].shape == (len(deltas), 3, 3, 2, 2, 4)
