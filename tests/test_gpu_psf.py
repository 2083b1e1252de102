"""The diffraction PSF on the device (rtx_grid_linear, rtx_psf;
ResidentMixin.opd_device / psf_device) against scipy's griddata, numpy's FFT,
the oracle (oracle/psf_oracle.py) and, where its tree is staged, the
reference's own GeometricTrace.opd / psf (rayopt/geometric_trace.py:101-169)."""
import os
import warnings

import numpy as np
import pytest
from scipy.interpolate import griddata
from scipy.spatial import Delaunay

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


def hull_distance(tri, px, py):
    """distance of the points (px, py) to the convex hull's boundary"""
    a = tri.points[tri.convex_hull[:, 0]]
    b = tri.points[tri.convex_hull[:, 1]]
    p = np.stack([px, py], axis=-1)[:, None, :]
    ab = b - a
    s = np.clip(((p - a)*ab).sum(-1)/(ab*ab).sum(-1), 0, 1)
    return np.sqrt((np.square(a + s[..., None]*ab - p)).sum(-1)).min(1)


def check_regrid(eng, x, y, t, n, what):
    """device regridding vs griddata: bit-identical where the simplices agree,
    1e-13 max|t| on shared edges, NaN masks equal away from the hull"""
    h = np.fabs((x, y)).max()
    xs, ys, gh = psf_oracle.grid(n, h)
    pts = np.stack([x, y], axis=-1)
    tri = Delaunay(pts)
    got, win = eng.grid_linear(pts, t, tri, n, gh, winner=True)
    want = griddata((x, y), t, (xs, ys), method="linear", fill_value=np.nan)
    ref_win = psf_oracle.winner(tri, xs, ys)
    both = np.isfinite(got) & np.isfinite(want)
    same = both & (win == ref_win)
    assert np.array_equal(got[same], want[same]), what
    other = both & ~same
    scale = np.fabs(t).max()
    assert np.all(np.abs(got[other] - want[other]) <= 1e-13*scale), what
    flip = np.isnan(got) != np.isnan(want)
    if flip.any():
        d = hull_distance(tri, xs[flip], ys[flip])
        assert np.all(d <= 1e-9*h), (what, d.max()/h)
    assert flip.sum() <= 1e-3*n*n, (what, flip.sum())
    print("%s: n=%d nodes %d, winner agrees %d, shared-edge %d, hull flips %d, kernel %.3f ms"
          % (what, n, n*n, same.sum(), other.sum(), flip.sum(), eng.last_kernel_ms()))
    return got


@pytest.mark.parametrize("m", [20000, 100000])
def test_regrid_random_points(eng, m):
    rng = np.random.default_rng(m)
    r, phi = np.sqrt(rng.random(m)), 2*np.pi*rng.random(m)
    x, y = r*np.cos(phi), r*np.sin(phi)
    check_regrid(eng, x, y, np.cos(4*x)*y + x*x, int(4*m**.5), "random %d" % m)


@pytest.mark.parametrize("name", ["psf_cooke_f0", "psf_cooke_f07"])
def test_regrid_traced_exit_pupil(eng, name):
    d = np.load(os.path.join(GOLDEN, "vs_reference", name + ".npz"))
    x, y, t = d["x"], d["y"], d["t"]
    ok = np.isfinite(x) & np.isfinite(y) & np.isfinite(t)
    got = check_regrid(eng, x[ok], y[ok], t[ok], d["o"].shape[0], name)
    assert np.array_equal(np.isnan(got), np.isnan(d["o"]))


def pupil_opd(n, seed):
    """a smooth OPD on an (n, n) grid, NaN outside the unit disc"""
    rng = np.random.default_rng(seed)
    xs, ys, _ = psf_oracle.grid(n, 1.)
    o = 0.3*(xs*xs + ys*ys) + 0.1*xs*ys + rng.normal(0, .01, xs.shape)
    o[xs*xs + ys*ys > 1] = np.nan
    return xs, o


@pytest.mark.parametrize("pad", [1, 3, 4])
@pytest.mark.parametrize("n", [126, 127, 251, 400])
def test_psf_vs_numpy(eng, n, pad):
    xs, o = pupil_opd(n, n + pad)
    od = eng.to_device(o)
    try:
        out, raw = eng.psf(od, pad)
    finally:
        od.free()
    psf = out.download()
    out.free()
    _, _, want = psf_oracle.psf(xs, o, pad, 1e-3, 100.)
    err = np.abs(psf - want).max()/want.max()
    assert err <= 1e-12, err
    assert int(raw[0]) == np.isfinite(o).sum()
    f = psf_oracle.frequencies(xs, n*pad, 1e-3, 100.)
    p, q = np.broadcast_arrays(f[:, None], f)
    st, ref = eng.psf_stats(raw, f), psf_oracle.stats(p, q, want)
    assert abs(st["sum"] - ref["sum"]) <= 1e-12*ref["sum"]
    assert abs(st["max"] - ref["max"]) <= 1e-12*ref["max"]
    fs = ref["sum"]*np.fabs(f).max()
    for k in ("cp", "cq"):
        assert abs(st[k] - ref[k]) <= 1e-12*fs, k
    print("n=%d pad=%d: max |dpsf|/max psf %.2e" % (n, pad, err))


@pytest.mark.parametrize("name", ["psf_cooke_f0", "psf_cooke_f07", "psf_double_gauss_f07",
                                  "psf_mirror"])
def test_device_pipeline_vs_reference_psf(eng, name):
    """the stored per-ray OPD of the reference through rtx_grid_linear and
    rtx_psf reproduces the reference's opd() grid (to rounding on shared
    edges of the cocircular hexapolar points) and psf()"""
    d = np.load(os.path.join(GOLDEN, "vs_reference", name + ".npz"))
    x, y, t = d["x"], d["y"], d["t"]
    ok = np.isfinite(x) & np.isfinite(y) & np.isfinite(t)
    x, y, t = x[ok], y[ok], t[ok]
    pts = np.stack([x, y], axis=-1)
    n = d["o"].shape[0]
    o = eng.grid_linear(pts, t, Delaunay(pts), n, d["gh"], download=False)
    try:
        og, want = o.download(), d["o"]
        assert np.array_equal(np.isnan(og), np.isnan(want))
        fin = np.isfinite(want)
        assert np.abs(og[fin] - want[fin]).max() <= 1e-13*np.fabs(t).max()
        out, raw = eng.psf(o, 4)
    finally:
        o.free()
    psf = out.download()
    out.free()
    assert np.abs(psf - d["psf"]).max() <= 1e-12*d["psf"].max()


# ---- end to end on traced bundles (needs the reference's System) -----------
needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="no reference tree staged")


def build(R, name):
    import yaml
    import systems_yaml
    s = R.System(**yaml.safe_load(systems_yaml.SYSTEMS[name]))
    s.update()
    s.paraxial.refocus()
    return s


@pytest.fixture(scope="module")
def R():
    warnings.simplefilter("ignore")
    np.seterr(all="ignore")
    return ref_shim.load()


def compare_e2e(got, ref, tag):
    """device opd_device / psf_device against the oracle on the device's own
    per-ray OPD (tight) and against the reference's opd / psf.  The per-ray
    OPD comes from the device epilogue (rtx_trace_opd), which agrees with the
    reference to 1e-9 waves, so the grids agree to rounding and the PSFs to
    what 1e-9 waves of phase moves, unless the triangulation differs"""
    radius = got.system[-1].distance
    xr, yr, orf = ref.opd(radius=radius)
    xg, yg, og = got.opd_device(radius=radius)
    np.testing.assert_allclose(xg, xr, rtol=1e-12, atol=0)
    np.testing.assert_allclose(yg, yr, rtol=1e-12, atol=0)
    # the device grid against the oracle regridding of the device's own rays
    x, y, t = got.opd_rays(radius)
    _, _, oo = psf_oracle.opd_grid(x, y, t, got.nrays)
    assert np.array_equal(np.isnan(og), np.isnan(oo)), tag
    fin = np.isfinite(oo)
    assert np.abs(og[fin] - oo[fin]).max() <= 1e-13*np.fabs(t[np.isfinite(t)]).max(), tag
    # against the reference: with the same triangulation to 1e-9 waves; the
    # cocircular points of an on-axis hexapolar bundle can be triangulated
    # differently after rounding-level changes of the rays, and the linear
    # interpolant then differs across the flipped quadrilaterals
    ok = np.isfinite(x) & np.isfinite(y) & np.isfinite(t)
    xh, yh, th = ref.opd(resample=False, radius=radius)
    okh = np.isfinite(xh) & np.isfinite(yh) & np.isfinite(th)
    same_tri = np.array_equal(ok, okh) and np.array_equal(
        psf_oracle.triangulate(x[ok], y[ok]).simplices,
        psf_oracle.triangulate(xh[okh], yh[okh]).simplices)
    fin = np.isfinite(og) & np.isfinite(orf)
    dopd = np.abs(og[fin] - orf[fin]).max()
    assert dopd <= (1e-9 if same_tri else 1e-2), (tag, dopd, same_tri)   # waves
    flips = int((np.isnan(og) != np.isnan(orf)).sum())
    count = np.isfinite(orf).sum()
    assert flips <= 1e-3*og.size, (tag, flips)
    pr, qr, psr = ref.psf()
    pg, qg, psg = got.psf_device()
    np.testing.assert_allclose(pg, pr, rtol=1e-12, atol=0)
    np.testing.assert_allclose(qg, qr, rtol=1e-12, atol=0)
    # the oracle on the device's own grid: only the FFT differs
    _, _, pso = psf_oracle.psf(xg, og, 4, got.l/got.system.scale, got.system[-1].distance)
    dev = np.abs(psg - pso).max()/pso.max()
    assert dev <= 1e-12, (tag, dev)
    err = np.abs(psg - psr).max()/psr.max()
    # a node on the hull in one grid and not the other moves 1/#finite of the pupil
    tol = (1e-6 if same_tri else 1e-2) + 4*flips/count
    assert err <= tol, (tag, err, flips)
    st = got.psf_stats
    assert st["count"] == np.isfinite(og).sum()
    assert abs(st["sum"] - pso.sum()) <= 1e-12*pso.sum()
    assert abs(st["max"] - pso.max()) <= 1e-12*pso.max()
    print("%s: psf %s, |dpsf|/max %.1e vs oracle on the device grid, %.1e vs reference "
          "(opd %.1e waves, same triangulation %s), hull flips %d"
          % (tag, psg.shape, dev, err, dopd, same_tri, flips))


E2E = [("cooke", 0., 1000), ("cooke", .7, 1000), ("double_gauss", 0., 1000),
       ("double_gauss", .7, 1000), ("mirror", 0., 1000), ("mirror", .7, 1000),
       ("cooke", .7, 100000), ("double_gauss", 0., 100000), ("mirror", 0., 100000)]


@needs_ref
@pytest.mark.parametrize("name,field,nrays", E2E)
def test_psf_device_resident_trace(R, eng, name, field, nrays):
    from rayopt_b200 import ResidentTrace
    s1, s2 = build(R, name), build(R, name)
    ref, got = R.GeometricTrace(s1), ResidentTrace(s2, engine=eng)
    for g in (ref, got):
        g.rays_point((0, field), nrays=nrays, distribution="hexapolar", clip=False)
    compare_e2e(got, ref, "%s f%.1f %d" % (name, field, nrays))
    got.free()


@needs_ref
def test_psf_device_bound_reference_class(R, eng):
    from rayopt_b200 import bind
    s1, s2 = build(R, "double_gauss"), build(R, "double_gauss")
    GT = bind(R.GeometricTrace, engine=eng, resident=True)
    ref, got = R.GeometricTrace(s1), GT(s2)
    for g in (ref, got):
        g.rays_point((0, .7), nrays=1000, distribution="hexapolar", clip=False)
    compare_e2e(got, ref, "bound double_gauss")
    p, q, dev = got.psf_device(download=False)
    _, _, host = got.psf_device()
    assert np.array_equal(dev.download(), host)
    dev.free()
    got.free()


def test_large_bundle_psf(eng):
    """1e6 exit-pupil points, resample 4, pad 4: the 16000^2 PSF's peak, sum,
    centroid and low-frequency corners against the oracle on the same grid"""
    m = 10**6
    rng = np.random.default_rng(7)
    r, phi = np.sqrt(rng.random(m)), 2*np.pi*rng.random(m)
    x, y = r*np.cos(phi), r*np.sin(phi)
    t = 0.4*(x*x + y*y) + 0.2*x*y*y
    n = int(4*m**.5)
    h = np.fabs((x, y)).max()
    xs, ys, gh = psf_oracle.grid(n, h)
    pts = np.stack([x, y], axis=-1)
    o = eng.grid_linear(pts, t, Delaunay(pts), n, gh, download=False)
    try:
        oh = o.download()
        out, raw = eng.psf(o, 4)
    finally:
        o.free()
    assert out.shape == (16000, 16000)
    psf = out.download()
    out.free()
    _, _, want = psf_oracle.psf(xs, oh, 4, 1e-3, 100.)
    f = psf_oracle.frequencies(xs, 16000, 1e-3, 100.)
    st = eng.psf_stats(raw, f)
    scale = want.max()
    assert abs(st["max"] - scale) <= 1e-12*scale
    assert abs(st["sum"] - want.sum()) <= 1e-12*want.sum()
    cp = (want*f[:, None]).sum()
    cq = (want*f[None, :]).sum()
    fs = want.sum()*np.fabs(f).max()
    assert abs(st["cp"] - cp) <= 1e-12*fs and abs(st["cq"] - cq) <= 1e-12*fs
    for sl in (np.s_[:64, :64], np.s_[-64:, :64], np.s_[:64, -64:], np.s_[-64:, -64:]):
        assert np.abs(psf[sl] - want[sl]).max() <= 1e-12*scale
    assert int(raw[0]) == np.isfinite(oh).sum()


def test_memory_refusal(eng):
    """a PSF larger than free HBM is refused before anything is allocated"""
    from rayopt_b200._lib import RTX_E_NOMEM, RtxError
    o = eng.to_device(pupil_opd(1000, 0)[1])
    try:
        eng.sync()
        before = eng.free_bytes()
        with pytest.raises(RtxError, match="out of memory"):
            eng.psf(o, 1000)                     # (1e6)^2 nodes
        # the library's own check, before any allocation
        rc = eng.lib.rtx_psf(eng.ctx, 0, 1000, o.ptr, 200, o.ptr, None)
        assert rc == RTX_E_NOMEM
        assert eng.free_bytes() == before
        # FP32 is not supported
        assert eng.lib.rtx_psf(eng.ctx, 1, 1000, o.ptr, 1, o.ptr, None) == -2
        assert eng.lib.rtx_grid_linear(eng.ctx, 1, 0, None, None, 0, None, None, 4, o.ptr,
                                       o.ptr, None) == -2
    finally:
        o.free()
