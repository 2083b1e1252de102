"""rtx_trace_reduce_many and rayopt_b200.tolerance on the device.  Needs a GPU.

Each item's rays are traced with rtx_trace through the item's table (keep
last) and the moments are checked against the exact sums of those stored
rows (oracle/epi_oracle.py): counts exactly, every sum within
(ceil(N/512) + 64) eps sum|term|.  The sums are deterministic, so an item's
20 doubles are also compared bit for bit across calls, launch mates and
item orders."""
import copy
import ctypes as C
import time
import warnings

import numpy as np
import pytest

import epi_oracle
import ref_shim
import tolerance_oracle
from conftest import load_golden
from rayopt_b200.rays import aim_infinite, disc

pytestmark = pytest.mark.gpu

EPS = 2.0**-52
MODES = {"f64_exact": (np.float64, True), "f64_fast": (np.float64, False),
         "f32": (np.float32, False)}
NS = [0, 1, 511, 512, 513, 70001]


@pytest.fixture(scope="module")
def eng():
    from rayopt_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def plates(S=256):
    """a stack of plane-parallel plates: its FP64 table is 92 KB"""
    from rayopt_b200.surface_table import SURFACE_DTYPE
    t = np.zeros(S, SURFACE_DTYPE)
    t["rot"] = np.eye(3).reshape(9)
    t["offset"][:, 2] = .01
    t["radius2"] = np.inf
    t["n_asph"] = -1
    n = np.where(np.arange(S) % 2 == 0, 1.5, 1.0)
    t["n0"], t["n"] = np.r_[1.0, n[:-1]], n
    t["mu"] = t["n0"]/t["n"]
    t["muf"], t["sgn"], t["mu2m1"] = np.abs(t["mu"]), np.sign(t["mu"]), t["mu"]**2 - 1
    return t


def case(name, systems):
    """(table, rot0, clip, rays(n, seed))"""
    if name == "plates256":
        def rays(n, seed):
            rng = np.random.default_rng(seed)
            u = rng.normal(0, .1, (n, 2))
            return np.c_[rng.normal(0, 1, (n, 2)), np.zeros(n)], \
                np.c_[u, np.sqrt(1 - np.square(u).sum(1))]
        return plates(), None, False, rays
    if name == "tilted_start3":
        c = load_golden(name)

        def rays(n, seed):
            k = np.random.default_rng(seed).integers(0, len(c["y0"]), n)
            return c["y0"][k], c["u0"][k]
        return c["table"], c["rot0"], c["clip"], rays
    key, clip = {"double_gauss": ("double_gauss", True), "cooke_asph": ("cooke_asph", True),
                 "mirror": ("mirror", False), "zoom": ("zoom", True)}[name]
    ent = systems[key]
    aim = ent["aim"][0][3]

    def rays(n, seed):
        return aim_infinite(aim["field"], disc(n, seed), aim["z"], aim["p"], ent["object_angle"])
    return ent["tables"][0], None, clip, rays


def variants(table, k, seed):
    """k tables: the nominal one and k-1 with curvatures and spacings scaled
    by up to 1e-3 (the same surfaces, so the same kind of march)"""
    rng = np.random.default_rng(seed)
    out = np.repeat(table[None], k, axis=0)
    for v in range(1, k):
        out["c"][v] *= 1 + 1e-3*rng.uniform(-1, 1, len(table))
        out["kc2"][v] = (1 + out["k"][v])*out["c"][v]**2
        out["offset"][v, :, 2] *= 1 + 1e-3*rng.uniform(-1, 1, len(table))
    return out


def stored_last(eng, table, dy0, du0, N, dtype, exact, clip, rot0):
    ld = (max(N, 1) + 63)//64*64
    Y, U, I = (eng.empty((1, ld, 3), dtype) for _ in range(3))
    eng.trace_device(table, dy0, du0, Y, U, I, None, N=N, ld=ld, clip=clip, keep_last=True,
                     rot0=rot0, exact=exact)
    eng.sync()
    y, i = Y.download()[0, :N], I.download()[0, :N]
    for a in (Y, U, I):
        a.free()
    return y, i


def check_items(eng, tables, bundles, host, items, centers, dtype, exact, clip, rot0):
    """rtx_trace_reduce_many against the exact sums of the stored rows of
    every item; returns the moments"""
    m = eng.trace_reduce_many(tables, bundles, items, centers, clip=clip, rot0=rot0, exact=exact)
    cache = {}
    for i, (t, b) in enumerate(items):
        N = bundles[b][2]
        if N == 0:
            assert np.array_equal(m[i], np.zeros(20))
            continue
        if (t, b) not in cache:
            cache[t, b] = stored_last(eng, tables[t], bundles[b][0], bundles[b][1], N, dtype, exact,
                                      clip, rot0)
        y, inc = cache[t, b]
        s, a = epi_oracle.reduce_sums(y, inc, None, None if centers is None else centers[i])
        for k in (4, 5, 8):
            assert m[i, k] == s[k], (i, k, m[i, k], s[k])
        tol = (-(-N//512) + 64)*EPS*a
        nan = np.isnan(s)
        assert np.array_equal(np.isnan(m[i]), nan)
        assert np.all(np.abs(m[i][~nan] - s[~nan]) <= tol[~nan]), (i, m[i], s)
    return m


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("name", ["double_gauss", "cooke_asph", "mirror", "zoom", "tilted_start3"])
def test_moments_match_stored_rows(eng, systems, name, mode):
    """up to 64 tables, one bundle per N, items that repeat and interleave
    tables and bundles, centres absent and present"""
    dtype, exact = MODES[mode]
    table, rot0, clip, rays = case(name, systems)
    nt = 64 if name == "double_gauss" else 5
    tabs = variants(table, nt, 3)
    host = [rays(max(N, 1), 10 + k) for k, N in enumerate(NS)]
    bundles = [(eng.to_device(y, dtype), eng.to_device(u, dtype), N)
               for (y, u), N in zip(host, NS)]
    rng = np.random.default_rng(5)
    items = np.c_[rng.integers(0, nt, 40), rng.integers(0, len(NS), 40)]
    items[:len(NS), 1] = np.arange(len(NS))
    centers = None
    if mode != "f32":
        centers = rng.normal(0, 1e-2, (len(items), 4))
    check_items(eng, tabs, bundles, host, items, centers, dtype, exact, clip, rot0)
    for y, u, _ in bundles:
        y.free(), u.free()


@pytest.mark.parametrize("mode", ["f64_fast", "f32"])
def test_large_table_restaged(eng, systems, mode):
    """a 256-surface table (92 KB in FP64) restaged between items: the launch
    opts into more shared memory"""
    dtype, exact = MODES[mode]
    table, rot0, clip, rays = case("plates256", systems)
    tabs = variants(table, 3, 1)
    host = [rays(N, k) for k, N in enumerate((513, 2000))]
    bundles = [(eng.to_device(y, dtype), eng.to_device(u, dtype), len(y)) for y, u in host]
    items = np.array([[0, 0], [1, 1], [2, 0], [0, 1], [1, 0]])
    check_items(eng, tabs, bundles, host, items, None, dtype, exact, clip, rot0)


@pytest.mark.parametrize("mode", list(MODES))
def test_deterministic(eng, systems, mode):
    """item i's 20 doubles are the same bits in two calls, alone, among 1000
    other items and under a permutation of the items"""
    dtype, exact = MODES[mode]
    table, rot0, clip, rays = case("double_gauss", systems)
    tabs = variants(table, 16, 9)
    host = [rays(N, k) for k, N in enumerate((70001, 4099, 600))]
    bundles = [(eng.to_device(y, dtype), eng.to_device(u, dtype), len(y)) for y, u in host]
    rng = np.random.default_rng(2)
    items = np.c_[rng.integers(0, 16, 1001), rng.integers(0, 3, 1001)]
    centers = rng.normal(0, 1e-2, (1001, 4))
    m1 = eng.trace_reduce_many(tabs, bundles, items, centers, clip=clip, exact=exact)
    m2 = eng.trace_reduce_many(tabs, bundles, items, centers, clip=clip, exact=exact)
    assert m1.tobytes() == m2.tobytes()
    alone = eng.trace_reduce_many(tabs, bundles, items[:1], centers[:1], clip=clip, exact=exact)
    assert alone.tobytes() == m1[:1].tobytes()
    p = rng.permutation(1001)
    mp = eng.trace_reduce_many(tabs, bundles, items[p], centers[p], clip=clip, exact=exact)
    assert mp.tobytes() == m1[p].tobytes()


@pytest.mark.parametrize("mode", list(MODES))
def test_zero_delta_matches_trace_reduce(eng, systems, mode):
    """the nominal table agrees with rtx_trace_reduce on the same bundle
    within the bound (not bit for bit: rtx_trace_reduce adds with atomics)"""
    dtype, exact = MODES[mode]
    table, rot0, clip, rays = case("double_gauss", systems)
    y, u = rays(100003, 4)
    dy, du = eng.to_device(y, dtype), eng.to_device(u, dtype)
    c = np.array([0., .5, 0., .01])
    m = eng.trace_reduce_many(table[None], [(dy, du, None)], [[0, 0]], c[None], clip=clip,
                              exact=exact)[0]
    r = eng.trace_reduce(table, dy, du, clip=clip, exact=exact, center=c)
    yl, il = stored_last(eng, table, dy, du, len(y), dtype, exact, clip, None)
    a = epi_oracle.reduce_sums(yl, il, None, c)[1]
    assert np.array_equal(m[[4, 5, 8]], r[[4, 5, 8]])
    assert np.all(np.abs(m - r) <= 2*(1600 + 64)*EPS*a)


def test_refusals_launch_and_allocate_nothing(eng, systems):
    """each refusal returns its code with no launch and no allocation; m has a
    host guard band after nitems*20 doubles that stays untouched"""
    from rayopt_b200 import _lib
    table, _, clip, rays = case("double_gauss", systems)
    y, u = rays(1000, 1)
    dy, du = eng.to_device(y), eng.to_device(u)
    tabs = np.ascontiguousarray(variants(table, 2, 1))
    S = tabs.shape[1]
    eng.trace_reduce_many(tabs, [(dy, du, None)], [[0, 0]])         # warm the workspace

    def call(nt=2, tables=tabs, S=S, dtype=0, nb=1, N=(1000,), y0=(dy.ptr,), u0=(du.ptr,),
             it=(0,), ib=(0,), m=True, flags=0, nitems=None):
        Na = np.ascontiguousarray(N, np.int64)
        ya = (C.c_void_p*len(y0))(*y0) if y0 is not None else None
        ua = (C.c_void_p*len(u0))(*u0) if u0 is not None else None
        ita = np.ascontiguousarray(it, np.int32)
        iba = np.ascontiguousarray(ib, np.int32)
        n = len(it) if nitems is None else nitems
        out = np.full(max(n, 0)*20 + 64, 7.25)
        rc = eng.lib.rtx_trace_reduce_many(
            eng.ctx, nt, _lib.ptr(tables) if tables is not None else None, S, None, dtype, nb,
            _lib.ptr(Na), ya, ua, n, _lib.ptr(ita), _lib.ptr(iba), None, 1,
            _lib.ptr(out) if m else None, flags)
        return rc, out

    E_BAD, E_UNS = -1, -2
    bad_asph = tabs.copy()
    bad_asph["n_asph"][1, 3] = 11
    cases = [(dict(tables=None), E_BAD), (dict(m=False), E_BAD), (dict(nt=0), E_BAD),
             (dict(nb=0), E_BAD), (dict(nitems=0), E_BAD), (dict(S=0), E_BAD),
             (dict(S=257), E_BAD), (dict(it=(2,)), E_BAD), (dict(it=(-1,)), E_BAD),
             (dict(ib=(1,)), E_BAD), (dict(N=(-1,)), E_BAD), (dict(y0=(None,)), E_BAD),
             (dict(u0=(None,)), E_BAD), (dict(y0=None), E_BAD), (dict(dtype=7), E_BAD),
             (dict(tables=bad_asph), E_UNS), (dict(dtype=1, flags=1), E_UNS)]
    for kw, want in cases:
        eng.sync()
        free, launches = eng.free_bytes(), eng.launch_count()
        rc, out = call(**kw)
        assert rc == want, (kw, rc)
        assert eng.launch_count() == launches and eng.free_bytes() == free, kw
        assert (out == 7.25).all(), kw
    assert eng.lib.rtx_trace_reduce_many(None, 1, None, 1, None, 0, 1, None, None, None, 1, None,
                                         None, None, 0, None, 0) == E_BAD
    rc, out = call()                                                 # guard band
    assert rc == 0 and (out[20:] == 7.25).all() and out[5] == 1000
    rc, out = call(N=(0,), y0=(None,), u0=(None,))                   # N = 0: zeros, no rays read
    assert rc == 0 and (out[:20] == 0).all() and (out[20:] == 7.25).all()
    free = eng.free_bytes()
    rc, _ = call(N=(2**52,))                                         # 2^43 tiles of sums
    assert rc == _lib.RTX_E_NOMEM and eng.free_bytes() == free


# ---- rayopt_b200.tolerance against the reference ----------------------------
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


TOL = {"cooke": [(1, "curvature", 1e-3), (2, "distance", 2e-2), (3, "conic", .05),
                 (2, "tilt_x", 1e-3), (3, "index", 1e-3), (6, "curvature", -1e-3)],
       "double_gauss": [(1, "curvature", 2e-4), (2, "distance", 1e-2), (3, "conic", .05),
                        (4, "tilt_y", 5e-4), (1, "index", 1e-3), (9, "distance", -1e-2)]}


@needs_ref
@pytest.mark.parametrize("exact", [True, False])
@pytest.mark.parametrize("name", ["cooke", "double_gauss"])
def test_tolerance_against_reference(eng, R, name, exact):
    """every (variant, height, wavelength) against the reference's
    GeometricTrace of the perturbed System fed the nominal launch rays with
    clip=True; with compensate="focus" also the shift against refocus() on
    Analysis's 13-ray bundle"""
    from rayopt.utils import pupil_distribution
    import rayopt_b200
    from rayopt_b200.tolerance import launch_bundles
    sys_ = build(R, name)
    params = [(j, k) for j, k, _ in TOL[name]]
    deltas = rayopt_b200.sensitivity_deltas([t for _, _, t in TOL[name]])
    heights = (0., .7)
    rtol = 1e-12 if exact else 1e-10
    for comp in (None, "focus"):
        s = copy.deepcopy(sys_)
        out = rayopt_b200.tolerance(s, params, deltas, heights=heights, nrays=300,
                                    compensate=comp, engine=eng, exact=exact)
        W = len(s.wavelengths)
        bundles, _ = launch_bundles(copy.deepcopy(sys_), heights, s.wavelengths, 300, "hexapolar",
                                    eng)
        launch = [(y.download(), u.download()) for y, u in bundles]
        nom = copy.deepcopy(sys_)
        fref, yp, fw = pupil_distribution("radau", 13)
        z, p = nom.pupil((0, 0.), l=s.wavelengths[0])
        fy, fu = nom.aim((0, 0.), yp, z, p, filter=False)
        for y, u in bundles:
            y.free(), u.free()
        for v, row in enumerate(deltas):
            ref = copy.deepcopy(sys_)
            for (j, kind), dv in zip(params, row):
                if dv:
                    from test_tolerance_host import apply
                    apply(ref, j, kind, dv)
            if comp == "focus":                                # the nominal lens's 13 rays
                g = R.GeometricTrace(ref)
                g.rays_given(fy, fu, s.wavelengths[0], fw, fref)
                g.propagate(clip=False)
                d0 = ref[-1].distance
                g.refocus()
                shift = ref[-1].distance - d0
                assert abs(out["focus"][v] - shift) <= 1e-10*abs(shift) + 1e-15, (v, out["focus"][v],
                                                                                 shift)
            for h in range(len(heights)):
                for w, l in enumerate(s.wavelengths):
                    y0, u0 = launch[h*W + w]
                    g = R.GeometricTrace(ref)
                    g.rays_given(y0, u0, l)
                    g.propagate(clip=True)
                    y = g.y[-1]
                    fin = np.isfinite(y[:, :2]).all(1)
                    assert out["transmitted"][v, h, w] == fin.mean(), (v, h, w)
                    want = tolerance_oracle.rms_finite_rows(y)
                    got = out["rms"][v, h, w]
                    assert abs(got - want) <= rtol*want, (comp, v, h, w, got, want)


def test_scale_and_chunking(eng, systems):
    """4096 variants x 9 bundles x 1e4 rays of the double Gauss: every ray is
    counted, two runs agree bit for bit and so does a run chunked into
    launches of 100 variants (the time is printed, not asserted)"""
    from rayopt_b200.tolerance import perturbed_tables
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

    def run(step):
        out = []
        for v0 in range(0, V, step):
            t = perturbed_tables(nominal, params, deltas[v0:v0 + step])
            n = len(t)
            it = items[v0*H*W:(v0 + n)*H*W].copy()
            it[:, 0] -= v0*W
            out.append(eng.trace_reduce_many(t.reshape(n*W, -1), bundles, it, clip=True))
        return np.concatenate(out)

    t0 = time.perf_counter()
    a = run(V)
    wall = time.perf_counter() - t0
    ms = eng.last_kernel_ms()
    b = run(V)
    c = run(100)
    assert a[:, 5].sum() == V*H*W*N
    assert a.tobytes() == b.tobytes() == c.tobytes()
    print("4096 x 9 x 1e4: kernel %.2f ms, call %.1f ms, %.3g ray-surfaces/s"
          % (ms, 1e3*wall, V*H*W*N*nominal.shape[1]/(ms*1e-3)))
