"""rtx_trace_opd_many and rayopt_b200.tolerance_wavefront on the device.
Needs a GPU.

Each item's rays are traced with rtx_trace_opd through the item's table with
the item's sphere, and its 10 sums are checked against the long-double sums
of those per-ray (a, x, y): counts exactly, every sum within include/rtx.h's
bound.  Then per ray bit for bit, bit-for-bit determinism, the C refusals, a
4096-variant run in chunks, and the analysis end to end against the
reference's own opd() of every perturbed lens, wavefront_jacobian, the
optimiser's trial scorer and tolerance()'s focus."""
import copy
import ctypes as C
import time
import warnings

import numpy as np
import pytest

import ref_shim
from test_gpu_tolerance import NS, case, variants
from test_gpu_wavefront import opd_case

pytestmark = pytest.mark.gpu

EPS = 2.0**-52
MODES = {"f64_exact": True, "f64_fast": False}


@pytest.fixture(scope="module")
def eng():
    from rayopt_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def rotation(seed, angle=.02):
    """a small proper rotation: a non-identity frame change M"""
    rng = np.random.default_rng(seed)
    a = rng.normal(0, angle, 3)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    from scipy.linalg import expm
    return expm(K)


def spec_for(table, y0, u0, seed, rot=False, infinite=1):
    """a sphere about the image of launch ray 0: n_after of the table's last
    record, a radius of the order of the track, optionally a turned frame"""
    rng = np.random.default_rng(seed)
    return dict(y0_ref=y0[0], u0_ref=u0[0], n0=1., n_after=float(table["n"][-1]),
                M=rotation(seed) if rot else np.eye(3), d=rng.normal(0, 1e-2, 3) - [0, 0, 5.],
                radius=float(rng.choice([-1, 1])*rng.uniform(40, 120)), infinite=infinite)


def opd_rows(eng, table, dy, du, N, spec, exact, clip, rot0):
    """rtx_trace_opd's A (N,) and P (N, 3) of a bundle"""
    A, P = eng.empty((max(N, 1),)), eng.empty((max(N, 1), 3))
    try:
        eng.trace_opd(table, dy, du, spec, A, P, N=N, clip=clip, rot0=rot0, exact=exact)
        eng.sync()
        return A.download()[:N], P.download()[:N]
    finally:
        A.free(), P.free()


def oracle(A, P, a0, c):
    """the 10 sums (long double, pairwise) and sum |term| of each"""
    with np.errstate(all="ignore"):
        a = A - a0
        x = P[:, 0] - c[0]
        y = P[:, 1] - c[1]
    ok = np.isfinite(a) & np.isfinite(x) & np.isfinite(y)
    a, x, y = (np.asarray(v[ok], np.longdouble) for v in (a, x, y))
    terms = [np.ones_like(a), a, a*a, x, y, x*x, x*y, y*y, a*x, a*y]
    return (np.array([t.sum() for t in terms]), np.array([np.abs(t).sum() for t in terms]),
            int(ok.sum()))


def device_bundles(eng, rays, Ns=NS):
    host = [rays(max(N, 1), 10 + k) for k, N in enumerate(Ns)]
    return [(eng.to_device(y), eng.to_device(u), N) for (y, u), N in zip(host, Ns)], host


def free(bundles):
    for y, u, _ in bundles:
        y.free(), u.free()


def check_items(eng, tables, bundles, host, items, specs, a0, cen, exact, clip, rot0):
    s = eng.trace_opd_many(tables, bundles, items, specs, a0, cen, clip=clip, rot0=rot0,
                           exact=exact)
    assert s.shape == (len(items), 10)
    for i, (t, b) in enumerate(items):
        N = bundles[b][2]
        if N == 0:
            assert (s[i] == 0).all()
            continue
        A, P = opd_rows(eng, tables[t], bundles[b][0], bundles[b][1], N, specs[i], exact, clip,
                        rot0)
        want, mag, n = oracle(A, P, a0[i], cen[i])
        assert s[i, 0] == n, (i, s[i, 0], n)
        tol = (-(-N//512) + 64)*EPS*mag.astype(float)
        err = np.abs(s[i] - want.astype(float))
        assert np.all(err <= tol), (i, err, tol)
    return s


def item_specs(table, host, items, seed):
    rng = np.random.default_rng(seed)
    specs, a0, cen = [], rng.normal(0, 1e-3, len(items)), rng.normal(0, 1e-2, (len(items), 2))
    for k, (t, b) in enumerate(items):
        y0, u0 = host[b]
        specs.append(spec_for(table, y0, u0, seed + k, rot=k % 2 == 1, infinite=k % 3 != 2))
    return specs, a0, cen


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("name", ["double_gauss", "cooke_asph", "mirror", "zoom", "tilted_start3",
                                  "plates256"])
def test_sums_match_stored_rows(eng, systems, name, mode):
    """up to 8 tables, one bundle per N, items that repeat and interleave
    tables and bundles, each with its own sphere (some turned, some of a
    finite object), piston guess and centre"""
    exact = MODES[mode]
    table, rot0, clip, rays = case(name, systems)
    march = table if name == "plates256" else table[:-1]
    k = 3 if name == "plates256" else 8
    tabs = variants(march, k, 3)
    bundles, host = device_bundles(eng, rays)
    rng = np.random.default_rng(7)
    items = np.c_[rng.integers(0, k, 10), rng.integers(0, len(NS), 10)]
    items[:len(NS), 1] = np.arange(len(NS))
    specs, a0, cen = item_specs(march, host, items, 11)
    try:
        check_items(eng, tabs, bundles, host, items, specs, a0, cen, exact, clip, rot0)
    finally:
        free(bundles)


@pytest.mark.parametrize("exact", [True, False], ids=["exact", "fast"])
@pytest.mark.parametrize("clip", [True, False], ids=["clip", "noclip"])
@pytest.mark.parametrize("infinite, rot", [(1, False), (0, True), (1, True)])
def test_single_rays_are_trace_opd(eng, exact, clip, infinite, rot):
    """items of 1-ray bundles cut from a 200-ray bundle, a0 = 0 and c = 0:
    sum a, sum x and sum y are rtx_trace_opd's A, P_x and P_y bit for bit"""
    full, rot0, y0, u0, spec = opd_case("double_gauss", 200, seed=5, scale=1.05)
    spec = dict(spec, infinite=infinite, M=rotation(3) if rot else np.eye(3))
    table = full[:-1]
    dy, du = eng.to_device(y0), eng.to_device(u0)
    try:
        A, P = opd_rows(eng, table, dy, du, 200, spec, exact, clip, rot0)
        bundles = [(dy.rows(k, k + 1), du.rows(k, k + 1), None) for k in range(200)]
        items = np.c_[np.zeros(200, int), np.arange(200)]
        s = eng.trace_opd_many(table[None], bundles, items, [spec]*200, clip=clip, rot0=rot0,
                               exact=exact)
        ok = np.isfinite(A) & np.isfinite(P[:, 0]) & np.isfinite(P[:, 1])
        assert ok.sum() > 100 and (clip or ok.all())
        assert np.array_equal(s[:, 0], ok.astype(float))
        for col, want in ((1, A), (3, P[:, 0]), (4, P[:, 1])):
            w = np.where(ok, want, 0.)
            assert s[:, col].tobytes() == (w + 0.).tobytes(), col
    finally:
        dy.free(), du.free()


@pytest.mark.parametrize("mode", list(MODES))
def test_deterministic(eng, systems, mode):
    """an item's sums are the same bits in two calls, in another context,
    alone, among 1000 other items, under a permutation and in two halves"""
    from rayopt_b200.engine import Engine
    exact = MODES[mode]
    table, rot0, clip, rays = case("double_gauss", systems)
    march = table[:-1]
    tabs = variants(march, 16, 9)
    bundles, host = device_bundles(eng, rays, (70001, 4099, 600))
    rng = np.random.default_rng(2)
    items = np.c_[rng.integers(0, 16, 1001), rng.integers(0, 3, 1001)]
    specs, a0, cen = item_specs(march, host, items, 5)
    from rayopt_b200.engine import OPD_DTYPE, _opd_record
    recs = np.concatenate([_opd_record(s) for s in specs]).astype(OPD_DTYPE)

    def run(e, sel):
        return e.trace_opd_many(tabs, bundles, items[sel], recs[sel], a0[sel], cen[sel],
                                clip=clip, exact=exact)
    try:
        every = np.arange(1001)
        a = run(eng, every)
        assert run(eng, every).tobytes() == a.tobytes()
        e2 = Engine(0)
        try:
            assert run(e2, every).tobytes() == a.tobytes()
        finally:
            e2.close()
        assert run(eng, every[:1]).tobytes() == a[:1].tobytes()
        p = rng.permutation(1001)
        assert run(eng, p).tobytes() == a[p].tobytes()
        halves = np.concatenate([run(eng, every[:500]), run(eng, every[500:])])
        assert halves.tobytes() == a.tobytes()
    finally:
        free(bundles)


def test_refusals_launch_and_allocate_nothing(eng, systems):
    """each refusal returns its code with no launch and no allocation; the
    output has host guard bands that stay untouched"""
    from rayopt_b200 import _lib
    from rayopt_b200.engine import OPD_DTYPE, _opd_record
    table, _, clip, rays = case("double_gauss", systems)
    march = np.ascontiguousarray(variants(table[:-1], 2, 1))
    y, u = rays(1000, 1)
    dy, du = eng.to_device(y), eng.to_device(u)
    S = march.shape[1]
    good = _opd_record(spec_for(march[0], y, u, 1)).astype(OPD_DTYPE)
    eng.trace_opd_many(march, [(dy, du, None)], [[0, 0]], good)                 # warm

    def call(nt=2, tables=march, S=S, dtype=0, nb=1, N=(1000,), y0=(dy.ptr,), u0=(du.ptr,),
             it=(0,), ib=(0,), specs=good, a0=None, centers=None, sums=True, flags=0):
        Na = np.ascontiguousarray(N, np.int64)
        ya = (C.c_void_p*len(y0))(*y0) if y0 is not None else None
        ua = (C.c_void_p*len(u0))(*u0) if u0 is not None else None
        ita, iba = np.ascontiguousarray(it, np.int32), np.ascontiguousarray(ib, np.int32)
        sa = None if specs is None else np.ascontiguousarray(specs, OPD_DTYPE)
        aa = None if a0 is None else np.ascontiguousarray(a0, np.float64)
        ca = None if centers is None else np.ascontiguousarray(centers, np.float64)
        out = np.full(len(it)*10 + 64, 7.25)
        rc = eng.lib.rtx_trace_opd_many(
            eng.ctx, nt, _lib.ptr(tables) if tables is not None else None, S, None, dtype, nb,
            _lib.ptr(Na), ya, ua, len(it), _lib.ptr(ita), _lib.ptr(iba), _lib.ptr(sa),
            _lib.ptr(aa), _lib.ptr(ca), 1, _lib.ptr(out) if sums else None, flags)
        return rc, out

    def bad(field, value):
        r = good.copy()
        r[field] = value
        return r
    E_BAD, E_UNS = -1, -2
    bad_asph = march.copy()
    bad_asph["n_asph"][1, 3] = 11
    y32, u32 = eng.to_device(y.astype(np.float32)), eng.to_device(u.astype(np.float32))
    cases = [(dict(tables=None), E_BAD), (dict(sums=False), E_BAD), (dict(specs=None), E_BAD),
             (dict(nt=0), E_BAD), (dict(nb=0), E_BAD), (dict(S=0), E_BAD), (dict(S=257), E_BAD),
             (dict(it=(2,)), E_BAD), (dict(it=(-1,)), E_BAD), (dict(ib=(1,)), E_BAD),
             (dict(N=(-1,)), E_BAD), (dict(y0=(None,)), E_BAD), (dict(u0=(None,)), E_BAD),
             (dict(y0=None), E_BAD), (dict(dtype=7), E_BAD),
             (dict(a0=[np.nan]), E_BAD), (dict(a0=[np.inf]), E_BAD),
             (dict(centers=[[0., np.nan]]), E_BAD), (dict(centers=[[np.inf, 0.]]), E_BAD),
             (dict(specs=bad("radius", 0.)), E_BAD), (dict(specs=bad("radius", np.inf)), E_BAD),
             (dict(specs=bad("n0", np.nan)), E_BAD), (dict(specs=bad("n_after", np.inf)), E_BAD),
             (dict(specs=bad("M", np.r_[np.nan, np.zeros(8)])), E_BAD),
             (dict(specs=bad("d", [0., np.nan, 0.])), E_BAD),
             (dict(specs=bad("y0_ref", [np.inf, 0., 0.])), E_BAD),
             (dict(specs=bad("u0_ref", [0., 0., np.nan])), E_BAD),
             (dict(tables=bad_asph), E_UNS),
             (dict(dtype=1, y0=(y32.ptr,), u0=(u32.ptr,)), E_UNS),
             (dict(dtype=1, y0=(y32.ptr,), u0=(u32.ptr,), flags=1), E_UNS)]
    try:
        for kw, want in cases:
            eng.sync()
            fb, launches = eng.free_bytes(), eng.launch_count()
            rc, out = call(**kw)
            assert rc == want, (kw, rc)
            assert eng.launch_count() == launches and eng.free_bytes() == fb, kw
            assert (out == 7.25).all(), kw
        rc, out = call()                                              # guard bands
        assert rc == 0 and (out[10:] == 7.25).all() and 0 < out[0] <= 1000
        rc, out = call(N=(0,), y0=(None,), u0=(None,))                # N = 0: zeros
        assert rc == 0 and (out[:10] == 0).all() and (out[10:] == 7.25).all()
        fb = eng.free_bytes()
        rc, _ = call(N=(2**52,))                                      # 2^43 tile rows
        assert rc == _lib.RTX_E_NOMEM and eng.free_bytes() == fb
    finally:
        for a in (dy, du, y32, u32):
            a.free()


def test_scale_and_chunking(eng, systems):
    """4096 variants x 9 bundles x 1e4 rays of the double Gauss: every item
    counts rays, and a run chunked into launches of half the variants gives
    the same bits"""
    from rayopt_b200.tolerance import perturbed_tables
    from rayopt_b200.rays import aim_infinite, disc
    ent = systems["double_gauss"]
    nominal = np.stack(ent["tables"][:3])
    params = [(1, "curvature"), (2, "distance"), (4, "conic"), (6, "tilt_x")]
    deltas = np.random.default_rng(1).uniform(-1, 1, (4096, 4))*[1e-4, 1e-2, 1e-2, 1e-3]
    N = 10000
    bundles, specs = [], []
    for h in range(3):
        for w in range(3):
            aim = ent["aim"][w][(0, 3, 5)[h]]
            y, u = aim_infinite(aim["field"], disc(N, h*3 + w), aim["z"], aim["p"],
                                ent["object_angle"])
            bundles.append((eng.to_device(y), eng.to_device(u), N))
            specs.append(spec_for(nominal[w, :-1], y, u, h*3 + w))
    V, H, W = 4096, 3, 3
    vv, hh, ww = np.meshgrid(np.arange(V), np.arange(H), np.arange(W), indexing="ij")
    items = np.stack([vv*W + ww, hh*W + ww], -1).reshape(-1, 2)
    from rayopt_b200.engine import OPD_DTYPE, _opd_record
    recs = np.concatenate([_opd_record(s) for s in specs]).astype(OPD_DTYPE)

    def run(step):
        out = []
        for v0 in range(0, V, step):
            t = perturbed_tables(nominal, params, deltas[v0:v0 + step])[:, :, :-1]
            k = len(t)
            it = items[v0*H*W:(v0 + k)*H*W].copy()
            it[:, 0] -= v0*W
            out.append(eng.trace_opd_many(t.reshape(k*W, -1), bundles, it, recs[it[:, 1]],
                                          clip=True))
        return np.concatenate(out)

    try:
        t0 = time.perf_counter()
        a = run(V)
        wall = time.perf_counter() - t0
        ms = eng.last_kernel_ms()
        b = run(V//2)
        assert a.tobytes() == b.tobytes()
        assert (a[:, 0] > 0).all() and (a[:, 0] <= N).all()
        print("4096 x 9 x 1e4: kernel %.2f ms, call %.1f ms" % (ms, 1e3*wall))
    finally:
        free(bundles)


# ---- rayopt_b200.tolerance_wavefront end to end ------------------------------
needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="no reference tree staged")


@pytest.fixture(scope="module")
def R():
    warnings.simplefilter("ignore")
    np.seterr(all="ignore")
    return ref_shim.load()


def build(R, name):
    import yaml
    import systems_yaml
    s = R.System(**yaml.safe_load(systems_yaml.SYSTEMS[name]))
    s.update()
    s.paraxial.refocus()
    return s


def tol_case(name, S):
    """TOL-style sensitivity parameters with a tilt of the last lens surface
    and the image distance"""
    return {"cooke": [(1, "curvature", 1e-3), (2, "distance", 2e-2), (3, "conic", .05),
                      (S - 1, "tilt_x", 1e-3), (3, "index", 1e-3), (S, "distance", 2e-2)],
            "double_gauss": [(1, "curvature", 2e-4), (3, "conic", .05), (4, "tilt_y", 5e-4),
                             (S - 1, "tilt_y", 7e-4), (1, "index", 1e-3),
                             (S, "distance", -1e-2)]}[name]


@needs_ref
@pytest.mark.parametrize("exact", [True, False], ids=["exact", "fast"])
@pytest.mark.parametrize("name", ["cooke", "double_gauss"])
def test_against_reference_opd(eng, R, name, exact):
    """every (variant, height, wavelength) against the reference's
    GeometricTrace of the perturbed System fed the nominal launch rays
    (clip=True, ref = the chief) and opd(radius=R_nominal, resample=0):
    n the finite rays, rms = std(t), rms_tilt the lstsq residual on (1, x,
    y); compensate="focus" gives tolerance()'s shifts bit for bit.

    Both rms agree within 1e-10 rms + 1e-10 waves in both modes.  The
    device forms each ray's path and sphere intercept in rtx_trace_opd's
    operation order (the frame change y M + d), the reference in its own
    (from_normal, the origins, to_normal), so each ray's t differs by a
    rounding of order eps track/lambda ~ 5e-11 waves whatever the mode; the
    largest difference measured on an H100 was 7.5e-11 of rms."""
    import rayopt_b200
    from rayopt_b200.lazy import opd_spec
    from rayopt_b200.rays import grid_spec
    from rayopt_b200.surface_table import pack_system
    from rayopt_b200.tolerance import launch_bundles
    from test_tolerance_host import apply
    sys_ = build(R, name)
    S = len(pack_system(sys_, sys_.wavelengths[0], 1, None)[0])
    tol = tol_case(name, S)
    params = [(j, k) for j, k, _ in tol]
    deltas = rayopt_b200.sensitivity_deltas([t for _, _, t in tol])
    heights, nrays = (0., .7), 300
    ref_i = grid_spec("hexapolar", nrays)[0]
    rtol = 1e-10
    worst = 0.
    for comp in (None, "focus"):
        out = rayopt_b200.tolerance_wavefront(copy.deepcopy(sys_), params, deltas, heights,
                                              nrays=nrays, compensate=comp, engine=eng,
                                              exact=exact)
        W = len(sys_.wavelengths)
        nom = copy.deepcopy(sys_)
        bundles, _ = launch_bundles(nom, heights, nom.wavelengths, nrays, "hexapolar", eng)
        radius = opd_spec(nom, nom.track, nom.origins, len(nom) - 2, len(nom) - 1, 1., 1.,
                          np.zeros(3), np.zeros(3), np.zeros(3))["radius"]
        launch = [(y.download(), u.download()) for y, u in bundles]
        for y, u in bundles:
            y.free(), u.free()
        if comp == "focus":
            b = rayopt_b200.tolerance(copy.deepcopy(sys_), params, deltas, heights, nrays=nrays,
                                      compensate="focus", engine=eng, exact=exact)
            assert out["focus"].tobytes() == b["focus"].tobytes()
        for v, row in enumerate(deltas):
            ref = copy.deepcopy(sys_)
            for (j, kind), dv in zip(params, row):
                if dv:
                    apply(ref, j, kind, dv)
            if comp == "focus":
                ref[-1].distance += out["focus"][v]
            for h in range(len(heights)):
                for w, l in enumerate(sys_.wavelengths):
                    y0, u0 = launch[h*W + w]
                    g = R.GeometricTrace(ref)
                    g.rays_given(y0, u0, l, ref=ref_i)
                    g.propagate(clip=True)
                    assert out["chief"][v, h, w]
                    x, y, t = g.opd(radius=radius, resample=0)
                    ok = np.isfinite(x) & np.isfinite(y) & np.isfinite(t)
                    x, y, t = x[ok], y[ok], t[ok]
                    key = (comp, v, h, w)
                    assert out["sums"][v, h, w, 0] == ok.sum(), key
                    rms = np.std(t)
                    A = np.c_[np.ones_like(x), x, y]
                    r = t - A @ np.linalg.lstsq(A, t, rcond=None)[0]
                    rms_tilt = np.sqrt(np.mean(r*r))
                    e1 = abs(out["rms"][v, h, w] - rms)
                    e2 = abs(out["rms_tilt"][v, h, w] - rms_tilt)
                    worst = max(worst, e1/rms, e2/rms)
                    assert max(e1, e2) <= rtol*rms + 1e-10, (key, e1/rms, e2/rms)
                    assert out["rms_tilt"][v, h, w] <= out["rms"][v, h, w]
    print("%s %s: largest relative difference from opd() %.2e" % (name, exact, worst))


@needs_ref
def test_against_wavefront_jacobian_and_trial_scorer(eng):
    """the Cooke triplet: the nominal row's rms against wavefront_jacobian's
    (clip on), every variant's per-bundle rms^2 against the trial scorer
    _wavefront_merits on the same deltas (no last-surface tilts: it holds M
    fixed), rms_tilt <= rms, and chunking changes no bit.  The trial scorer
    takes every variant's residuals about the nominal lens's chief path,
    not the variant's, so its one-pass variance cancels more: 1e-10"""
    from rayopt_b200 import optimize as opt
    from rayopt_b200.tolerance import tolerance_wavefront
    from test_gpu_optimize import cooke, cooke_params
    s = cooke()
    params = cooke_params(s)
    rng = np.random.default_rng(4)
    deltas = np.r_[np.zeros((1, len(params))), rng.uniform(-1, 1, (6, len(params)))*1e-3]
    H = (0., .7, 1.)
    res = tolerance_wavefront(copy.deepcopy(s), params, deltas, H, nrays=1000, engine=eng,
                              targets=.5)
    V, nh, W = res["rms"].shape
    j = opt.wavefront_jacobian(copy.deepcopy(s), params, H, nrays=1000, clip=True, engine=eng)
    assert np.array_equal(res["sums"][0, ..., 0], j["n"])
    assert np.allclose(res["rms"][0], j["rms"], rtol=1e-12, atol=0)
    sb = copy.deepcopy(s)
    B = opt._Bundles(sb, H, s.wavelengths, 1000, "hexapolar", eng, False)
    st, worst = None, 0.
    try:
        st = opt._Wavefront(eng, sb, B, H, None, None, True, False)
        for b in range(nh*W):
            w = np.zeros(nh*W)
            w[b] = 1
            m = opt._wavefront_merits(eng, B, st, params, deltas, w, True, False)
            got = res["rms"][:, b//W, b % W]**2
            worst = max(worst, float(np.max(np.abs(got - m)/m)))
            assert np.allclose(got, m, rtol=1e-10, atol=0), (b, np.abs(got - m)/m)
    finally:
        if st is not None:
            st.close()
        B.close()
    print("largest relative difference of rms^2 from the trial scorer %.2e" % worst)
    assert np.all(res["rms_tilt"] <= res["rms"])
    again = tolerance_wavefront(copy.deepcopy(s), params, deltas, H, nrays=1000, engine=eng,
                                targets=.5, chunk=3)
    for k in ("sums", "rms", "rms_tilt", "strehl", "poly_rms_tilt", "passed"):
        assert np.asarray(again[k]).tobytes() == np.asarray(res[k]).tobytes(), k
    assert res["yield"] == res["passed"].mean()
