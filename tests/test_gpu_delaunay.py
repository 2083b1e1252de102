"""Delaunay triangulation on the device (rtx_delaunay, Engine.delaunay) against
exact rational predicates, scipy.spatial.Delaunay and the exact checker
(oracle/delaunay_oracle.py), its regridding against griddata, and the PSF
with the device triangulation against the host one."""
import os
import warnings
from fractions import Fraction

import numpy as np
import pytest
from scipy.interpolate import griddata
from scipy.spatial import Delaunay

import delaunay_oracle as dto
import psf_oracle
import ref_shim
from conftest import GOLDEN

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from rayopt_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def disc(m, seed):
    rng = np.random.default_rng(seed)
    r, phi = np.sqrt(rng.random(m)), 2*np.pi*rng.random(m)
    return np.stack([r*np.cos(phi), r*np.sin(phi)], -1)


def exit_pupil(name):
    d = np.load(os.path.join(GOLDEN, "vs_reference", name + ".npz"))
    x, y, t = d["x"], d["y"], d["t"]
    ok = np.isfinite(x) & np.isfinite(y) & np.isfinite(t)
    return np.stack([x[ok], y[ok]], -1), t[ok]


def triples(s):
    return {tuple(sorted(t)) for t in np.asarray(s).tolist()}


def triangulate(eng, p):
    tri = eng.delaunay(p)
    try:
        return tri.download()
    finally:
        tri.free()


# ---- 1. predicates -----------------------------------------------------------
def _sign(v):
    return (v > 0) - (v < 0)


def exact_signs(q):
    out = []
    for a, b, c, d in q.reshape(-1, 4, 2).tolist():
        F = [tuple(Fraction(v) for v in p) for p in (a, b, c, d)]
        o = (F[0][0] - F[2][0])*(F[1][1] - F[2][1]) - (F[0][1] - F[2][1])*(F[1][0] - F[2][0])
        m = [(p[0] - F[3][0], p[1] - F[3][1]) for p in F[:3]]
        lift = [x*x + y*y for x, y in m]
        i = (lift[0]*(m[1][0]*m[2][1] - m[2][0]*m[1][1]) + lift[1]*(m[2][0]*m[0][1] - m[0][0]*m[2][1])
             + lift[2]*(m[0][0]*m[1][1] - m[1][0]*m[0][1]))
        out.append((_sign(o), _sign(i)))
    return np.array(out)


def near_degenerate(n, seed, scale):
    """quadruples with c within ulps of the line ab and d within ulps of the
    circle abc, scaled by `scale`"""
    rng = np.random.default_rng(seed)
    q = np.empty((n, 4, 2))
    for k in range(n):
        a, b = rng.random(2), rng.random(2)
        c = a + rng.random()*(b - a)
        c = np.nextafter(c, c + rng.integers(-1, 2, 2))
        th = 2*np.pi*rng.random(4)
        r, ctr = rng.random() + .1, rng.random(2)
        circ = ctr + r*np.stack([np.cos(th), np.sin(th)], -1)
        circ[3] = np.nextafter(circ[3], circ[3] + rng.integers(-1, 2, 2))
        q[k] = [a, b, c, circ[3]] if k % 2 else circ
    return q*scale


def test_predicates_exact(eng):
    qs = [near_degenerate(400, 1, 1.), near_degenerate(200, 2, 2.**190),
          near_degenerate(200, 3, 2.**-150), disc(4000, 4).reshape(-1, 4, 2)]
    # integer lattice: exact zeros on lines and circles
    rng = np.random.default_rng(5)
    lat = rng.integers(-3, 4, (400, 4, 2)).astype(float)
    lat[:, 2] = lat[:, 0] + 2*(lat[:, 1] - lat[:, 0])
    qs.append(lat)
    sq = np.array([[0, 0], [1, 0], [1, 1], [0, 1]], float)
    qs.append(np.stack([sq*s + o for s, o in ((1, 0), (2.**-200, 0), (2.**200, 0), (3., 2.**-100))]))
    q = np.concatenate(qs)
    got = eng.selftest_predicates(q)
    want = exact_signs(q)
    assert np.array_equal(got, want), np.flatnonzero((got != want).any(1))[:10]
    assert (want == 0).sum() > 100 and (want != 0).sum() > 1000


# ---- 2. general position: scipy's triangles exactly -----------------------------
def check_regrid(eng, p, t, n, tri_dev, what):
    h = np.fabs(p).max()
    xs, ys, gh = psf_oracle.grid(n, h)
    want = griddata((p[:, 0], p[:, 1]), t, (xs, ys), method="linear", fill_value=np.nan)
    got = eng.grid_linear(p, t, tri_dev, n, gh)
    both = np.isfinite(got) & np.isfinite(want)
    scale = np.fabs(t).max()
    assert np.all(np.abs(got[both] - want[both]) <= 1e-13*scale), what
    flip = np.isnan(got) != np.isnan(want)
    if flip.any():
        from test_gpu_psf import hull_distance
        d = hull_distance(Delaunay(p), xs[flip], ys[flip])
        assert np.all(d <= 1e-9*h), what
    return got, want


GENERAL = [3, 4, 5, 100, 10**4, 10**5, 10**6]


@pytest.mark.parametrize("m", GENERAL)
def test_general_position_disc(eng, m):
    p = disc(m, m)
    tri = eng.delaunay(p)
    try:
        s, nb, tr = tri.download()
        ref = Delaunay(p)
        assert tri.T == len(ref.simplices)
        assert triples(s) == triples(ref.simplices)
        if m <= 10**5:
            dto.check(p, s, nb, ccw=True)
        assert not np.isnan(tr).any()
        if m >= 100:
            t = np.cos(4*p[:, 0])*p[:, 1] + p[:, 0]**2
            check_regrid(eng, p, t, int(4*m**.5) if m <= 10**5 else 1000, tri, "disc %d" % m)
    finally:
        tri.free()
    print("disc %d: T=%d, %.2f ms" % (m, len(s), eng.last_kernel_ms()))


@pytest.mark.parametrize("name", ["psf_cooke_f07", "psf_double_gauss_f07"])
def test_general_position_exit_pupil(eng, name):
    p, t = exit_pupil(name)
    tri = eng.delaunay(p)
    try:
        s, nb, _ = tri.download()
        assert triples(s) == triples(Delaunay(p).simplices)
        dto.check(p, s, nb, ccw=True)
        d = np.load(os.path.join(GOLDEN, "vs_reference", name + ".npz"))
        got, want = check_regrid(eng, p, t, d["o"].shape[0], tri, name)
    finally:
        tri.free()


# ---- 3. degenerate sets: exact checks, differences only in cocircular quads ----------
# Exactly cocircular ties come from the grids and the duplicates; the traced
# on-axis pupils (psf_cooke_f0, psf_mirror) are cocircular only up to rounding
# and have no exactly cocircular quadrilateral, so there the device matches
# scipy triangle for triangle.
def square_grid(k):
    return np.stack(np.meshgrid(np.arange(k, dtype=float), np.arange(k, dtype=float)), -1).reshape(-1, 2)


def triangular_grid(k):
    """rows offset by half a step (exactly representable, so that the slanted
    sides are exactly collinear)"""
    i, j = np.meshgrid(np.arange(k, dtype=float), np.arange(k, dtype=float))
    return np.stack([i + 0.5*j, j], -1).reshape(-1, 2)


def with_extreme_copies(p):
    """p plus copies of its lexicographic maximum (twice), minimum and a middle point"""
    order = np.lexsort((p[:, 1], p[:, 0]))
    return np.concatenate([p, p[[order[-1], order[0], order[len(p)//2], order[-1]]]])


def first_copies(p):
    """the lowest index of every distinct point: the vertices a triangulation keeps"""
    return set(np.unique(np.asarray(p) + 0.0, axis=0, return_index=True)[1].tolist())


def degenerate_sets():
    rng = np.random.default_rng(9)
    g = square_grid(40)/39
    line = np.stack([np.linspace(0, 1, 50), np.zeros(50)], -1)
    hull_line = np.concatenate([disc(500, 3)*0.4 + 0.5, np.stack([np.linspace(0, 1, 30), np.zeros(30)], -1),
                                np.stack([np.zeros(30), np.linspace(0, 1, 30)], -1)])
    return {
        "psf_cooke_f0": exit_pupil("psf_cooke_f0")[0],
        "psf_mirror": exit_pupil("psf_mirror")[0],
        "square_grid": g,
        "triangular_grid": triangular_grid(30),
        "duplicates": np.concatenate([g, g[rng.integers(0, len(g), 300)], [[0.5, -0.0], [0.5, 0.0]]]),
        "extreme_duplicates": with_extreme_copies(g),
        "square_with_copy": np.array([[0, 0], [1, 0], [0, 1], [1, 1], [1, 1]], float),
        "collinear_hull": hull_line,
        "line_plus_point": np.concatenate([line, [[0.3, 0.2]]]),
        "line_plus_point_and_dup": np.concatenate([line, line[::5], [[0.3, -0.2]]]),
    }


@pytest.mark.parametrize("name", list(degenerate_sets()))
def test_degenerate_sets(eng, name):
    p = degenerate_sets()[name]
    s, nb, tr = triangulate(eng, p)
    st = dto.check(p, s, nb, ccw=True)
    assert not np.isnan(tr).any()
    assert set(np.unique(s).tolist()) == first_copies(p), "a duplicate kept instead of the lowest index"
    ref = Delaunay(p)
    dev_q, ref_q = dto.cocircular_differences(p, s, ref.simplices)
    # every differing triangle lies in an exactly cocircular quadrilateral
    cs, cr = dto.canonical(p, s), dto.canonical(p, ref.simplices)
    assert triples(cs) - triples(cr) <= dev_q
    assert triples(cr) - triples(cs) <= ref_q
    # regridding: nodes that differ by more than rounding are covered by such quadrilaterals
    t = np.sin(3*p[:, 0]) + p[:, 1]**2
    h = np.fabs(p).max()
    n = 200
    xs, ys, gh = psf_oracle.grid(n, h)
    tri = eng.delaunay(p)
    try:
        got, win = eng.grid_linear(p, t, tri, n, gh, winner=True)
    finally:
        tri.free()
    want = griddata((p[:, 0], p[:, 1]), t, (xs, ys), method="linear", fill_value=np.nan)
    ref_win = psf_oracle.winner(ref, xs, ys)
    both = np.isfinite(got) & np.isfinite(want)
    bad = both & (np.abs(got - want) > 1e-13*np.fabs(t).max())
    for k in np.flatnonzero(bad.ravel()):
        assert tuple(sorted(cs[win.ravel()[k]])) in dev_q, name
        assert tuple(sorted(cr[ref_win.ravel()[k]])) in ref_q, name
    print("%s: T=%d, cocircular edges %d, differing triangles %d, nodes off by more than rounding %d"
          % (name, st["T"], st["cocircular"], len(dev_q), bad.sum()))


# ---- 4. refusals ------------------------------------------------------------------
def test_refusals(eng):
    from rayopt_b200._lib import RTX_E_NOMEM, RtxError
    import ctypes as C
    p = disc(1000, 1)
    triangulate(eng, p)                 # the workspace for 1000 points is kept in the context
    eng.sync()
    before = eng.free_bytes()
    T = C.c_int64()
    d = eng.to_device(p)
    out = eng.empty((2000, 3), np.int32)
    try:
        eng.sync()
        before = eng.free_bytes()
        lib, ctx = eng.lib, eng.ctx
        assert lib.rtx_delaunay(ctx, 0, 2, d.ptr, C.byref(T), out.ptr, None, None) == -1
        assert lib.rtx_delaunay(ctx, 1, 1000, d.ptr, C.byref(T), out.ptr, None, None) == -2
        # a workspace larger than free HBM: refused before anything is allocated
        m = (1 << 30) - 1
        assert eng.delaunay_bytes(m) > eng.total_bytes
        assert lib.rtx_delaunay(ctx, 0, m, d.ptr, C.byref(T), out.ptr, None, None) == RTX_E_NOMEM
        assert eng.free_bytes() == before
        # NaN, infinity, outside the predicates' domain, all collinear
        for bad in (np.nan, np.inf, 2.**201, 2.**-201):
            q = p.copy()
            q[17, 1] = bad
            d.upload(q)
            assert lib.rtx_delaunay(ctx, 0, 1000, d.ptr, C.byref(T), out.ptr, None, None) == -1, bad
        k = np.arange(1000.)
        q = np.stack([k, 2*k + 1], -1)          # exactly collinear
        q[::3] = q[5]
        d.upload(q)
        assert lib.rtx_delaunay(ctx, 0, 1000, d.ptr, C.byref(T), out.ptr, None, None) == -1
        assert eng.free_bytes() == before
        with pytest.raises(RtxError):
            eng.delaunay(q)
    finally:
        d.free()
        out.free()


# ---- 5. determinism -----------------------------------------------------------------
def test_deterministic_1e6(eng):
    from rayopt_b200.engine import Engine
    p = disc(10**6, 77)
    p[::1000] = p[1::1000]                     # duplicates
    a = triangulate(eng, p)
    b = triangulate(eng, p)
    e2 = Engine(0)
    try:
        c = triangulate(e2, p)
    finally:
        e2.close()
    for x, y, z in zip(a, b, c):
        assert x.tobytes() == y.tobytes() == z.tobytes()
    g = square_grid(300)
    assert all(x.tobytes() == y.tobytes() for x, y in zip(triangulate(eng, g), triangulate(eng, g)))


# ---- 6. end to end -------------------------------------------------------------------
needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="no reference tree staged")


@pytest.fixture(scope="module")
def R():
    warnings.simplefilter("ignore")
    np.seterr(all="ignore")
    return ref_shim.load()


E2E = [("cooke", .7, 1000), ("double_gauss", .7, 1000), ("mirror", .7, 1000),
       ("cooke", 0., 1000), ("mirror", 0., 1000), ("cooke", .7, 100000)]


@needs_ref
@pytest.mark.parametrize("name,field,nrays", E2E)
def test_psf_device_triangulation(R, eng, name, field, nrays):
    from rayopt_b200 import ResidentTrace
    from test_gpu_psf import build
    got = ResidentTrace(build(R, name), engine=eng)
    got.rays_point((0, field), nrays=nrays, distribution="hexapolar", clip=False)
    radius = got.system[-1].distance
    x, y, t = got.opd_rays(radius)
    ok = np.isfinite(x) & np.isfinite(y) & np.isfinite(t)
    p = np.stack([x[ok], y[ok]], -1)
    s, nb, _ = triangulate(eng, p)
    dto.check(p, s, nb, ccw=True)
    same = triples(s) == triples(Delaunay(p).simplices)
    if field:
        assert same, "off-axis bundle: the triangulations must be the same"
    _, _, host = got.psf_device()
    host_stats = got.psf_stats
    pd, qd, dev = got.psf_device(triangulation="device")
    err = np.abs(dev - host).max()/host.max()
    # a differing triangulation of cocircular points: the bound compare_e2e allows
    assert err <= (1e-12 if same else 1e-2), (name, field, err)
    # psf_profiles with the device triangulation: the encircled energy, the
    # line-sum MTFs and their axes of that PSF (Analysis.opds's reduction,
    # about the device's centroid)
    prof = got.psf_profiles(triangulation="device")
    import profile_oracle
    want = profile_oracle.profiles(pd, qd, dev, x0=prof["x0"], y0=prof["y0"])
    assert prof["center"] == want["center"] and prof["dx"] == want["dx"]
    assert np.abs(prof["ee"] - want["ee"]).max() <= 1e-12*dev.sum()
    np.testing.assert_array_equal(prof["xe"], want["xe"])
    np.testing.assert_array_equal(prof["of"], want["of"])
    for a, b in zip(prof["mtf"], want["mtf"]):
        assert a.shape == b.shape and np.abs(a - b).max() <= 1e-12*b.max()
    print("%s f%.1f %d: same triangulation %s, |dpsf|/max %.1e (host stats %s)"
          % (name, field, nrays, same, err, host_stats["count"]))
    got.free()
