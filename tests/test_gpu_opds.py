"""The exit-pupil points compacted in HBM (rtx_opd_points), the range of a
grid (rtx_grid_range), the device path they give ResidentMixin's opd_device /
psf_device / psf_profiles, and rayopt_b200.opds (Analysis.opds,
rayopt/analysis.py:285-352): exact against numpy, bit for bit against the
host composition they replace and against the resident trace, and end to end
against the reference where its tree is staged."""
import copy
import warnings

import numpy as np
import pytest
from scipy.spatial import Delaunay

import profile_oracle
import psf_oracle
import ref_shim

pytestmark = pytest.mark.gpu

SENTINEL = 0xA5
BAND = 1 << 16            # bytes of guard band after each output


@pytest.fixture(scope="module")
def eng():
    from rayopt_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def bits(a):
    a = np.ascontiguousarray(a, np.float64)
    return a.view(np.uint64)


def same_bits(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return a.shape == b.shape and np.array_equal(bits(a), bits(b))


def numpy_points(a, p, ref, k):
    """ResidentMixin.opd_rays's reference subtraction and GeometricTrace.opd's
    finite filter (rayopt/geometric_trace.py:125-135) on the host"""
    t = -(a - a[ref])/k
    p = p.copy()
    p -= p[ref]
    x, y = p[:, 0], p[:, 1]
    ok = np.isfinite(x) & np.isfinite(y) & np.isfinite(t)
    x, y, t = x[ok], y[ok], t[ok]
    h = np.fabs((x, y)).max() if t.size else 0.
    return np.stack([x, y], axis=-1), t, int(t.size), h


def opd_inputs(N, seed, ref):
    """A (N,), P (N,3) like rtx_trace_opd's, with NaN and +-inf placed
    separately in x, y, t and z, and -0.0 results: P[j].x = -0.0 against
    P[ref].x = +0.0, and A[j] = A[ref] (t = -0.0)"""
    rng = np.random.default_rng(seed)
    a = rng.normal(0, 1e3, N)
    p = rng.normal(0, 10., (N, 3))
    p[ref, 0] = 0.
    specials = (np.nan, np.inf, -np.inf)
    if N > 8:
        idx = rng.permutation(np.setdiff1d(np.arange(N), [ref]))
        groups = np.array_split(idx[:max(13, N//20)], 13)
        for g, v in zip(groups[:3], specials):
            p[g, 0] = v                               # x
        for g, v in zip(groups[3:6], specials):
            p[g, 1] = v                               # y
        for g, v in zip(groups[6:9], specials):
            a[g] = v                                  # t
        for g, v in zip(groups[9:12], specials):
            p[g, 2] = v                               # z: the ray is kept
        p[groups[12], 0] = -0.
        a[groups[12][::2]] = a[ref]
    return a, p


def call_points(eng, a, p, ref, k):
    """rtx_opd_points through the C ABI with guard bands after pts and vals;
    returns (pts, vals, M, h) and asserts the bands, A and P untouched"""
    import ctypes as C
    from rayopt_b200._lib import check
    N = len(a)
    A, P = eng.to_device(a), eng.to_device(p)
    pts = eng.empty((N*16 + BAND,), np.uint8)
    vals = eng.empty((N*8 + BAND,), np.uint8)
    try:
        eng.memset(pts, SENTINEL)
        eng.memset(vals, SENTINEL)
        M, h = C.c_int64(-1), C.c_double(-1.)
        check(eng.lib.rtx_opd_points(eng.ctx, 0, N, A.ptr, P.ptr, ref, k, pts.ptr, vals.ptr,
                                     C.byref(M), C.byref(h)))
        M = M.value
        pb, vb = pts.download(), vals.download()
        assert (pb[16*M:] == SENTINEL).all(), "written at or after pts[M]"
        assert (vb[8*M:] == SENTINEL).all(), "written at or after vals[M]"
        assert A.download().tobytes() == a.tobytes() and P.download().tobytes() == p.tobytes()
        return pb[:16*M].view(np.float64).reshape(M, 2), vb[:8*M].view(np.float64), M, h.value
    finally:
        for d in (A, P, pts, vals):
            d.free()


SIZES = [1, 31, 1024, 1025, 10**6 + 7, 3*10**7]


@pytest.mark.parametrize("N", SIZES)
def test_opd_points_equal_numpy(eng, N):
    k = 0.5876e-3
    refs = sorted({0, N//2, N - 1}) if N < 10**7 else [N//2]
    for ref in refs:
        a, p = opd_inputs(N, N + ref, ref)
        got = call_points(eng, a, p, ref, k)
        want = numpy_points(a, p, ref, k)
        assert got[2] == want[2], (N, ref, got[2], want[2])
        assert same_bits(got[0], want[0]) and same_bits(got[1], want[1]), (N, ref)
        assert same_bits(got[3], want[3]), (N, ref, got[3], want[3])
        if N > 8:                                         # the -0.0 results survive
            x, t = got[0][:, 0], got[1]
            assert (np.signbit(x) & (x == 0)).any() and (np.signbit(t) & (t == 0)).any()
        print("N=%d ref=%d: M=%d, kernels %.3f ms" % (N, ref, got[2], eng.last_kernel_ms()))


@pytest.mark.parametrize("what", ["a", "x", "y"])
def test_opd_points_nonfinite_reference_ray(eng, what):
    N, ref = 1025, 17
    a, p = opd_inputs(N, 3, ref)
    for v in (np.nan, np.inf, -np.inf):
        b, q = a.copy(), p.copy()
        if what == "a":
            b[ref] = v
        else:
            q[ref, "xy".index(what)] = v
        pts, vals, M, h = call_points(eng, b, q, ref, 1.)
        assert M == 0 and h == 0. and pts.shape == (0, 2) and vals.shape == (0,)
        assert numpy_points(b, q, ref, 1.)[2] == 0


def test_opd_points_engine_wrapper(eng):
    N, ref = 5000, 123
    a, p = opd_inputs(N, 9, ref)
    A, P = eng.to_device(a), eng.to_device(p)
    try:
        pts, vals, M, h = eng.opd_points(A, P, ref, 2.5e-4)
        want = numpy_points(a, p, ref, 2.5e-4)
        assert M == want[2] and pts.shape == (M, 2) and vals.shape == (M,)
        assert same_bits(pts.download(), want[0]) and same_bits(vals.download(), want[1])
        assert h == want[3]
        pts.free(), vals.free()
    finally:
        A.free(), P.free()


def test_opd_points_refusals(eng):
    """every refusal returns its code before any device work"""
    import ctypes as C
    lib = eng.lib
    N = 64
    A, P = eng.to_device(np.zeros(N)), eng.to_device(np.zeros((N, 3)))
    pts, vals = eng.empty((N, 2)), eng.empty((N,))
    M, h = C.c_int64(), C.c_double()
    try:
        def call(ctx=eng.ctx, dtype=0, n=N, a=A.ptr, p=P.ptr, ref=0, k=1., o=pts.ptr, v=vals.ptr,
                 m=True, hh=True):
            return lib.rtx_opd_points(ctx, dtype, n, a, p, ref, k, o, v,
                                      C.byref(M) if m else None, C.byref(h) if hh else None)
        assert call() == 0
        eng.sync()
        before, launches = eng.free_bytes(), eng.launch_count()
        assert call(ctx=None) == -1
        assert call(a=None) == -1 and call(p=None) == -1 and call(o=None) == -1
        assert call(v=None) == -1 and call(m=False) == -1 and call(hh=False) == -1
        assert call(n=0) == -1 and call(n=-1) == -1 and call(n=1 << 31) == -1
        assert call(ref=-1) == -1 and call(ref=N) == -1
        for k in (0., -0., np.nan, np.inf, -np.inf):
            assert call(k=k) == -1, k
        assert call(dtype=1) == -2 and call(dtype=2) == -1
        assert eng.free_bytes() == before and eng.launch_count() == launches
    finally:
        for d in (A, P, pts, vals):
            d.free()


def test_grid_range(eng):
    import ctypes as C
    rng = np.random.default_rng(4)
    grids = []
    g = rng.normal(0, 1, (300, 300))
    g[rng.random(g.shape) < .3] = np.nan
    grids.append(g)
    g2 = g.copy()
    g2[5, 5], g2[7, 9], g2[0, 0] = np.inf, -np.inf, np.inf
    grids.append(g2)
    grids.append(np.full((40, 40), np.nan))
    grids.append(np.array([np.nan, -np.inf, np.inf, 2.5, np.nan]))
    grids.append(np.array([-0., 0., -0.]))
    grids.append(np.array([7.]))
    grids.append(rng.normal(0, 1, 10**7 + 3))
    for o in grids:
        d = eng.to_device(o)
        try:
            count, lo, hi = eng.grid_range(d)
        finally:
            d.free()
        fin = o[np.isfinite(o)]
        assert count == fin.size
        if fin.size:
            assert lo == fin.min() and hi == fin.max()
            assert lo == np.nanmin(np.where(np.isfinite(o), o, np.nan))
            assert hi == np.nanmax(np.where(np.isfinite(o), o, np.nan))
        else:
            assert np.isnan(lo) and np.isnan(hi)
    d = eng.to_device(np.array([-0., 0.]))
    try:
        _, lo, hi = eng.grid_range(d)
        assert np.signbit(lo) and not np.signbit(hi)      # -0 counts below +0
        c, lo_, hi_ = C.c_int64(), C.c_double(), C.c_double()
        call = lambda **kw: eng.lib.rtx_grid_range(
            kw.get("ctx", eng.ctx), kw.get("dtype", 0), kw.get("n", 2), kw.get("o", d.ptr),
            C.byref(c) if kw.get("c", True) else None, C.byref(lo_), C.byref(hi_))
        assert call() == 0
        assert call(ctx=None) == -1 and call(o=None) == -1 and call(n=0) == -1
        assert call(c=False) == -1 and call(dtype=1) == -2 and call(dtype=2) == -1
    finally:
        d.free()


# ---- the device path against the host composition it replaces ---------------
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


def old_opd_grid(g, radius, triangulation, download):
    """the regridding before the points stayed in HBM: opd_rays (every ray
    downloaded), numpy's filter, upload, triangulation, rtx_grid_linear"""
    eng = g.engine
    x, y, t = g.opd_rays(radius)
    ok = np.isfinite(x) & np.isfinite(y) & np.isfinite(t)
    x, y, t = x[ok], y[ok], t[ok]
    n = int(4*g.nrays**.5)
    h = np.fabs((x, y)).max()
    xs, ys = np.mgrid[-1:1:1j*n, -1:1:1j*n]*h
    pts = np.stack([x, y], axis=-1)
    if triangulation == "host":
        return xs, ys, eng.grid_linear(pts, t, Delaunay(pts), n, xs[:, 0].copy(), download=download)
    dpts = eng.to_device(pts)
    tri = eng.delaunay(dpts)
    o = eng.grid_linear(dpts, t, tri, n, xs[:, 0].copy(), download=download)
    tri.free()
    dpts.free()
    return xs, ys, o


CASES = [(name, field, nrays) for name in ("cooke", "double_gauss", "mirror")
         for field in (0., .7) for nrays in (1000, 100000)]


@needs_ref
@pytest.mark.parametrize("exact", [False, True])
@pytest.mark.parametrize("name,field,nrays", CASES)
def test_device_points_change_no_bits(R, eng, name, field, nrays, exact):
    from rayopt_b200 import ResidentTrace
    g = ResidentTrace(build(R, name), engine=eng, exact=exact)
    g.rays_point((0, field), nrays=nrays, distribution="hexapolar", clip=False)
    radius = g.system[-1].distance
    for tri in ("host", "device"):
        tag = (name, field, nrays, exact, tri)
        xs, ys, want = old_opd_grid(g, None, tri, True)
        xg, yg, got = g.opd_device(triangulation=tri)
        assert same_bits(xg, xs) and same_bits(yg, ys) and same_bits(got, want), tag
        xs, _, o = old_opd_grid(g, radius, tri, False)
        out, raw = eng.psf(o, 4)
        o.free()
        psf_old = out.download()
        out.free()
        p, q, psf = g.psf_device(triangulation=tri)
        stats = dict(g.psf_stats)
        assert same_bits(psf, psf_old), tag
        f = np.fft.fftfreq(4*xs.shape[0], (xs[1, 0] - xs[0, 0])*(1/(g.l/g.system.scale))/radius)
        assert same_bits(p[:, 0], f) and eng.psf_stats(raw, f) == stats, tag
        r = g.psf_profiles(triangulation=tri)
        want = profile_oracle.profiles(p, q, psf, x0=stats["cp"], y0=stats["cq"])
        assert r["stats"] == stats and r["center"] == want["center"] and r["dx"] == want["dx"]
        d = eng.to_device(psf)
        bins, l0, l1 = eng.psf_profiles(d, r["center"])
        d.free()
        assert same_bits(r["ee"], np.cumsum(bins)), tag
        size = psf.size
        for m, lsf in zip(r["mtf"], (l0, l1)):
            assert same_bits(m, np.absolute(np.fft.ifft(lsf*size**.5))[:lsf.size//2]), tag
    g.free()


# ---- rayopt_b200.opds against the resident trace, height by height ---------
def resident_height(R, eng, s, h, wl, nrays, exact):
    """what opds computes for one height, through ResidentTrace; None when no
    ray makes it through"""
    from rayopt_b200 import ResidentTrace
    g = ResidentTrace(s, engine=eng, exact=exact)
    g.rays_point((0, h), wl, nrays=nrays, distribution="hexapolar", clip=True)
    try:
        _, _, o = g.opd_device(triangulation="device")
    except ValueError:
        g.free()
        return None
    og = o[np.isfinite(o)]
    r = g.psf_profiles(triangulation="device")
    _, _, psf = g.psf_device(triangulation="device")
    g.free()
    r.update(ptp=np.ptp(og), max_abs=np.fabs(og).max(), count=og.size, opd=o, psf=psf)
    return r


def assert_same_height(got, want, tag):
    assert (got is None) == (want is None), tag
    if got is None:
        return
    for k in ("ptp", "max_abs", "x0", "y0", "dx", "center", "xe", "ee", "of", "mtf", "opd", "psf"):
        assert same_bits(got[k], want[k]), (tag, k)
    assert got["count"] == want["count"] and got["stats"] == want["stats"], tag


@needs_ref
@pytest.mark.parametrize("exact", [False, True])
@pytest.mark.parametrize("nrays", [1000, 100000])
@pytest.mark.parametrize("name", ["cooke", "double_gauss", "mirror"])
def test_opds_equal_resident_trace(R, eng, name, nrays, exact):
    import rayopt_b200
    s, s2 = build(R, name), build(R, name)
    wl = s.wavelengths[0]
    heights = (0., .707, 1.)
    out = rayopt_b200.opds(s, heights, wl, nrays, download=True, engine=eng, exact=exact)
    assert out["heights"] == list(heights) and out["wavelength"] == wl
    # System.pupil depends on the calls before it: the resident trace aims
    # the heights on a fresh copy in Analysis's order, last to first, as opds does
    want = [resident_height(R, eng, s2, h, wl, nrays, exact) for h in heights[::-1]][::-1]
    for h, a, b in zip(heights, out["results"], want):
        assert_same_height(a, b, (name, nrays, exact, h))
    last = [b for b in want if b is not None][-1]
    assert out["mm"] == last["max_abs"]
    assert out["rm"] == np.searchsorted(last["ee"], .9)*1.5*last["dx"]
    par = s.paraxial
    assert out["airy"] == par.airy_radius[1]/par.wavelength*wl
    # without download: the same reductions, no grids
    lean = rayopt_b200.opds(build(R, name), heights, wl, nrays, engine=eng, exact=exact)
    for a, b in zip(lean["results"], out["results"]):
        assert "opd" not in a and "psf" not in a
        assert same_bits(a["ee"], b["ee"]) and a["ptp"] == b["ptp"]


# ---- against the oracle and the reference's own opd() and psf() ------------
@needs_ref
@pytest.mark.parametrize("name,nrays", [("cooke", 1000), ("double_gauss", 1000), ("mirror", 1000),
                                        ("cooke", 100000)])
def test_opds_against_reference(R, eng, name, nrays):
    """triangulation="host" (scipy's Delaunay, as griddata).  On the device's
    own rays (the resident trace's opd_rays) the OPD grid equals the oracle's
    griddata to 1e-13 of max |t| with the same NaN mask, the PSF the oracle's
    to 1e-12 of its peak, and the encircled energy and MTFs those of the
    oracle on that PSF to 1e-12 (test_gpu_psf.py, test_gpu_psf_profiles.py).

    Against Analysis.opds's own loop (GeometricTrace.rays_point, opd() and
    psf(), the heights last to first on one System), with test_gpu_psf.py's
    tolerances: the grids to 1e-9 waves and the PSFs to 1e-6 of the peak
    where the exit-pupil points are triangulated as the reference does them,
    1e-2 where cocircular rings are split the other way; at most 1e-3 of the
    nodes finite in one grid only; the PTPs as the grids; the encircled
    energy and MTFs within the PSFs' own difference (sum |dpsf|) plus 1e-12,
    and the centroid as in test_gpu_psf_profiles.py."""
    import rayopt_b200
    from rayopt_b200 import ResidentTrace
    heights = (0., .707, 1.)
    s, s_res, s_ref = build(R, name), build(R, name), build(R, name)
    wl = s.wavelengths[0]
    out = rayopt_b200.opds(s, heights, wl, nrays, triangulation="host", download=True, engine=eng)
    for h, r in reversed(list(zip(heights, out["results"]))):
        tag = (name, nrays, h)
        t = R.GeometricTrace(s_ref)
        t.rays_point((0, h), wl, nrays=nrays, distribution="hexapolar", clip=True)
        g = ResidentTrace(s_res, engine=eng)
        g.rays_point((0, h), wl, nrays=nrays, distribution="hexapolar", clip=True)
        try:
            _, _, o = t.opd()
        except ValueError:
            assert r is None, tag
            g.free()
            continue
        og = r["opd"]
        assert r["ptp"] == np.ptp(og[np.isfinite(og)]) and r["count"] == np.isfinite(og).sum()
        assert r["max_abs"] == np.fabs(og[np.isfinite(og)]).max()
        # the oracle on the device's own rays
        x, y, tt = g.opd_rays()
        _, _, oo = psf_oracle.opd_grid(x, y, tt, g.nrays)
        radius = s[-1].distance
        xp, _, op = psf_oracle.opd_grid(*g.opd_rays(radius), g.nrays)
        g.free()
        assert np.array_equal(np.isnan(og), np.isnan(oo)), tag
        fin = np.isfinite(oo)
        assert np.abs(og[fin] - oo[fin]).max() <= 1e-13*np.fabs(tt[np.isfinite(tt)]).max(), tag
        _, _, pso = psf_oracle.psf(xp, op, 4, wl/s.scale, radius)
        assert np.abs(r["psf"] - pso).max() <= 1e-12*pso.max(), tag
        ee = np.cumsum(profile_oracle.polar_sum_azimuthal(np.fft.fftshift(r["psf"]), r["center"]))
        assert r["ee"].shape == ee.shape and np.abs(r["ee"] - ee).max() <= 1e-12, tag
        for m, lsf in zip(r["mtf"], profile_oracle.line_sums(r["psf"])):
            want = np.absolute(np.fft.ifft(lsf*lsf.size))[:lsf.size//2]
            assert m.shape == want.shape and np.abs(m - want).max() <= 1e-12, tag
        # the reference's own opd() and psf()
        xh, yh, th = t.opd(resample=False)
        ok = np.isfinite(x) & np.isfinite(y) & np.isfinite(tt)
        okh = np.isfinite(xh) & np.isfinite(yh) & np.isfinite(th)
        same_tri = np.array_equal(ok, okh) and np.array_equal(
            psf_oracle.triangulate(x[ok], y[ok]).simplices,
            psf_oracle.triangulate(xh[okh], yh[okh]).simplices)
        tol = 1e-9 if same_tri else 1e-2
        both = np.isfinite(og) & np.isfinite(o)
        dopd = np.abs(og[both] - o[both]).max()
        assert dopd <= tol, (tag, dopd, same_tri)
        flips = int((np.isnan(og) != np.isnan(o)).sum())
        count = np.isfinite(o).sum()
        assert flips <= 1e-3*og.size, (tag, flips)
        ptp = np.ptp(o[np.isfinite(o)])
        assert abs(r["ptp"] - ptp) <= tol + (1e-2*ptp if flips else 0.), (tag, r["ptp"], ptp)
        p, q, psf = t.psf()
        err = np.abs(r["psf"] - psf).max()/psf.max()
        assert err <= (1e-6 if same_tri else 1e-2) + 4*flips/count, (tag, err, flips)
        dpsf = np.abs(r["psf"] - psf).sum()
        xr, yr, sr = map(np.fft.fftshift, (p, q, psf))
        x0, y0 = (sr*xr).sum(), (sr*yr).sum()
        dx = (xr - x0)[1, 0] - (xr - x0)[0, 0]
        dc = max(abs(r["x0"]/r["dx"] - x0/dx), abs(r["y0"]/r["dx"] - y0/dx))
        assert dc <= max(1e-9, dpsf*psf.shape[0]/2), (tag, dc)
        ee = np.cumsum(profile_oracle.polar_sum_azimuthal(np.fft.fftshift(psf), r["center"]))
        assert r["ee"].shape == ee.shape and np.abs(r["ee"] - ee).max() <= 1e-12 + dpsf, tag
        for m, lsf in zip(r["mtf"], profile_oracle.line_sums(psf)):
            want = np.absolute(np.fft.ifft(lsf*lsf.size))[:lsf.size//2]
            assert m.shape == want.shape and np.abs(m - want).max() <= 1e-12 + dpsf, tag
        print("%s h=%.3f %d: ptp %.9g vs reference %.9g, opd %.1e waves, |dpsf|/max %.1e, "
              "hull flips %d, same triangulation %s"
              % (name, h, nrays, r["ptp"], ptp, dopd, err, flips, same_tri))


# ---- vignetting and memory -------------------------------------------------
@needs_ref
def test_opds_vignetted_field_and_memory(R, eng):
    import rayopt_b200
    s = build(R, "cooke")
    v = copy.deepcopy(s)
    v[1].radius = 1e-9          # the first surface stops every ray off the axis
    out = rayopt_b200.opds(v, (.707, 1.), nrays=1000, engine=eng)
    assert out["results"] == [None, None]
    assert out["mm"] is None and out["rm"] is None
    for sys_, heights in ((s, (0., .707, 1.)), (v, (.707, 1.))):
        rayopt_b200.opds(sys_, heights, nrays=10000, engine=eng)        # warm-up
        eng.sync()
        before = eng.free_bytes()
        rayopt_b200.opds(sys_, heights, nrays=10000, engine=eng)
        eng.sync()
        assert eng.free_bytes() == before
