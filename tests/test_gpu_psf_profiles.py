"""Encircled-energy bins and line sums of a device PSF (rtx_psf_profiles,
Engine.psf_profiles, ResidentMixin.psf_profiles) against the oracle
(oracle/profile_oracle.py): exact on dyadic inputs, within the stated bound of
the exact sums on real PSFs, deterministic, and end to end against
Analysis.opds's curves (rayopt/analysis.py:319-346) where the reference's
tree is staged."""
import math
import os
import warnings

import numpy as np
import pytest
from scipy.spatial import Delaunay

import profile_oracle
import psf_oracle
import ref_shim
from conftest import GOLDEN

pytestmark = pytest.mark.gpu

U = 2.**-53


@pytest.fixture(scope="module")
def eng():
    from rayopt_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def device_profiles(eng, psf, center):
    d = eng.to_device(psf)
    try:
        return eng.psf_profiles(d, center)
    finally:
        d.free()


def oracle_profiles(psf, center):
    return (profile_oracle.polar_sum_azimuthal(np.fft.fftshift(psf), center),
            *profile_oracle.line_sums(psf))


def centres(nx, ny):
    return [(nx/2 + .3712, ny/2 - .2841),     # Analysis-like: nx/2 + x0/dx
            (nx//2, ny//2), (1, 2),           # integer: pixels on bin boundaries
            (nx/2 + .5, ny/2 - .5),           # half-integer
            (-5.5, ny + 3.), (nx + 17.25, -9)]  # outside the array


@pytest.mark.parametrize("shape", [(1, 1), (3, 3), (7, 5), (126, 126), (381, 381), (512, 384)])
def test_exact_binning_dyadic(eng, shape):
    """integers times 2^-20 with a total below 2^30: every sum is exact in any
    order, so the device equals the oracle bit for bit"""
    rng = np.random.default_rng(shape[0]*1000 + shape[1])
    psf = rng.integers(0, 1 << 10, shape)*2.**-20
    for center in centres(*shape):
        got, want = device_profiles(eng, psf, center), oracle_profiles(psf, center)
        for g, w, what in zip(got, want, ("ee", "lsf0", "lsf1")):
            assert g.shape == w.shape and np.array_equal(g, w), (shape, center, what)


def test_docstring_cases_through_ifftshift(eng):
    m = np.arange(1., 10.).reshape((3, 3))
    stored = np.fft.ifftshift(m)
    assert np.array_equal(device_profiles(eng, stored, (1, 1))[0], [5., 40.])
    assert np.array_equal(device_profiles(eng, stored, (.5, .5))[0], [12., 24., 9.])


def exact_sums(psf, center):
    """math.fsum of every bin, column and row (stored order)"""
    s = np.fft.fftshift(psf)
    i, j = np.ogrid[:s.shape[0], :s.shape[1]]
    i, j = i - center[0], j - center[1]
    k = np.sqrt(j*j + i*i).astype(int).ravel()
    order = np.argsort(k, kind="stable")
    flat = s.ravel()[order]
    edges = np.searchsorted(k[order], np.arange(k.max() + 2))
    ee = np.array([math.fsum(flat[a:b]) for a, b in zip(edges[:-1], edges[1:])])
    lsf0 = np.array([math.fsum(c) for c in psf.T])
    lsf1 = np.array([math.fsum(r) for r in psf])
    return ee, lsf0, lsf1


def check_accuracy(eng, p, q, psf, what):
    """each sum within 2^-40 exact + 2^-90 sum psf of math.fsum; the
    cumulative EE and the MTF within 1e-12 of the oracle's"""
    want = profile_oracle.profiles(p, q, psf)
    got = device_profiles(eng, psf, want["center"])
    total = math.fsum(psf.ravel())
    for g, e, name in zip(got, exact_sums(psf, want["center"]), ("ee", "lsf0", "lsf1")):
        assert g.shape == e.shape, (what, name)
        err = np.abs(g - e)
        assert np.all(err <= 2.**-40*e + 2.**-90*total), (what, name, (err/np.maximum(e, 1e-300)).max())
    ee = np.cumsum(got[0])
    assert np.abs(ee - want["ee"]).max() <= 1e-12, what
    size = psf.size
    for lsf, m in zip(got[1:], want["mtf"]):
        mtf = np.absolute(np.fft.ifft(lsf*size**.5))[:lsf.size//2]
        assert np.abs(mtf - m).max() <= 1e-12, what
    print("%s: %s, %d bins, kernel %.3f ms" % (what, psf.shape, got[0].size, eng.last_kernel_ms()))


@pytest.mark.parametrize("name", ["psf_cooke_f0", "psf_cooke_f07", "psf_double_gauss_f07",
                                  "psf_mirror"])
def test_accuracy_stored_reference_psf(eng, name):
    d = np.load(os.path.join(GOLDEN, "vs_reference", name + ".npz"))
    p, q = np.broadcast_arrays(d["f"][:, None], d["f"])
    check_accuracy(eng, p, q, d["psf"], name)


def pupil_opd(n, seed):
    """a smooth OPD on an (n, n) grid, NaN outside the unit disc (as in
    test_gpu_psf.py)"""
    rng = np.random.default_rng(seed)
    xs, ys, _ = psf_oracle.grid(n, 1.)
    o = 0.3*(xs*xs + ys*ys) + 0.1*xs*ys + rng.normal(0, .01, xs.shape)
    o[xs*xs + ys*ys > 1] = np.nan
    return xs, o


@pytest.mark.parametrize("pad", [1, 3, 4])
@pytest.mark.parametrize("n", [126, 251, 400])
def test_accuracy_synthetic_pupils(eng, n, pad):
    xs, o = pupil_opd(n, n + pad)
    od = eng.to_device(o)
    try:
        out, _ = eng.psf(od, pad)
    finally:
        od.free()
    psf = out.download()
    out.free()
    f = psf_oracle.frequencies(xs, n*pad, 1e-3, 100.)
    p, q = np.broadcast_arrays(f[:, None], f)
    check_accuracy(eng, p, q, psf, "n=%d pad=%d" % (n, pad))


def test_deterministic_across_calls_and_engines(eng):
    from rayopt_b200.engine import Engine
    d = np.load(os.path.join(GOLDEN, "vs_reference", "psf_double_gauss_f07.npz"))
    psf = d["psf"]
    center = (psf.shape[0]/2 + .37, psf.shape[1]/2 - 1.61)
    a = device_profiles(eng, psf, center)
    b = device_profiles(eng, psf, center)
    e2 = Engine(0)
    try:
        c = device_profiles(e2, psf, center)
    finally:
        e2.close()
    for x, y, z in zip(a, b, c):
        assert x.tobytes() == y.tobytes() == z.tobytes()


def test_large_bundle_profiles(eng):
    """the 16000^2 PSF of 1e6 pupil points (as test_gpu_psf.test_large_bundle_psf)
    against the oracle on the downloaded PSF; the call holds no memory of its
    own beyond the context's scratch"""
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
        out, raw = eng.psf(o, 4)
    finally:
        o.free()
    try:
        assert out.shape == (16000, 16000)
        f = psf_oracle.frequencies(xs, 16000, 1e-3, 100.)
        st = eng.psf_stats(raw, f)
        fs = np.fft.fftshift(f)
        dx = (fs[1] - st["cp"]) - (fs[0] - st["cp"])
        center = (8000 + st["cp"]/dx, 8000 + st["cq"]/dx)
        first = eng.psf_profiles(out, center)
        eng.sync()
        before = eng.free_bytes()
        got = eng.psf_profiles(out, center)
        ms = eng.last_kernel_ms()
        assert eng.free_bytes() == before
        psf = out.download()
    finally:
        out.free()
    for a, b in zip(first, got):
        assert a.tobytes() == b.tobytes()
    want = oracle_profiles(psf, center)
    total = psf.sum()
    L = -(-250*250//132)
    for g, w, name, count in zip(got, want, ("ee", "lsf0", "lsf1"),
                                 (8*np.arange(1, len(want[0]) + 1) + 8, 16000, 16000)):
        assert g.shape == w.shape, name
        # oracle (sequential bincount, numpy's sums) and device error bounds
        tol = 1.01*(count + L + 200)*U*w + 2.**-90*total
        assert np.all(np.abs(g - w) <= tol), name
    print("16000^2: %d bins, kernel %.3f ms, %.0f GB/s read" % (got[0].size, ms,
                                                             psf.nbytes/ms/1e6))


def test_refusals(eng):
    """every refusal returns its code and allocates nothing; Engine raises"""
    from rayopt_b200._lib import RtxError
    lib = eng.lib
    psf = np.random.default_rng(1).random((40, 30))
    d = eng.to_device(psf)
    try:
        c0, c1 = 20.25, 14.5
        nb = eng.profile_nbins(psf.shape, (c0, c1))
        ee, l0, l1 = np.empty(nb), np.empty(30), np.empty(40)
        from rayopt_b200._lib import ptr

        def call(ctx=eng.ctx, dtype=0, nx=40, ny=30, p=d.ptr, a=c0, b=c1, nbins=nb, out=True):
            return lib.rtx_psf_profiles(ctx, dtype, nx, ny, p, a, b, nbins,
                                        ptr(ee) if out else None, ptr(l0) if out else None,
                                        ptr(l1) if out else None)
        assert call() == 0
        assert call(out=False) == 0
        eng.sync()
        before = eng.free_bytes()
        assert call(ctx=None) == -1
        assert call(p=None) == -1
        assert call(nx=0) == -1 and call(ny=0) == -1 and call(nx=-3) == -1
        for bad in (np.nan, np.inf, -np.inf):
            assert call(a=bad) == -1 and call(b=bad) == -1
        assert call(nbins=nb - 1) == -1 and call(nbins=nb + 1) == -1 and call(nbins=0) == -1
        assert call(dtype=1) == -2
        assert eng.free_bytes() == before
        for v in (-1e-300, -1., np.nan, np.inf):
            bad = psf.copy()
            bad[7, 3] = v
            d.upload(bad)
            assert call() == -1, v
            assert eng.free_bytes() == before
        with pytest.raises(RtxError, match="bad argument"):
            eng.psf_profiles(d, (c0, c1))
        d.upload(psf)
        with pytest.raises(RtxError, match="bad argument"):
            eng.psf_profiles(d, (np.nan, 1.))
        assert call() == 0
    finally:
        d.free()


# ---- end to end on traced bundles (needs the reference's System) -----------
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


E2E = [(name, field, nrays) for name in ("cooke", "double_gauss", "mirror")
       for field in (0., .7) for nrays in (1000, 100000)]


@needs_ref
@pytest.mark.parametrize("name,field,nrays", E2E)
def test_psf_profiles_resident_trace(R, eng, name, field, nrays):
    from rayopt_b200 import ResidentTrace
    s1, s2 = build(R, name), build(R, name)
    ref, got = R.GeometricTrace(s1), ResidentTrace(s2, engine=eng)
    for g in (ref, got):
        g.rays_point((0, field), nrays=nrays, distribution="hexapolar", clip=False)
    r = got.psf_profiles()
    p, q, psf = got.psf_device()
    want = profile_oracle.profiles(p, q, psf, x0=r["x0"], y0=r["y0"])
    assert want["center"] == r["center"] and want["dx"] == r["dx"]
    assert np.array_equal(r["xe"], want["xe"]) and np.array_equal(r["of"], want["of"])
    assert np.abs(r["ee"] - want["ee"]).max() <= 1e-12
    for a, b in zip(r["mtf"], want["mtf"]):
        assert a.shape == b.shape and np.abs(a - b).max() <= 1e-12
    assert abs(r["ee"][-1] - psf.sum()) <= 1e-12
    # the device's centroid against the reference's own psf(): to 1e-9 pixel
    # where the two PSFs agree to rounding.  The cocircular rings of an
    # on-axis hexapolar bundle can be triangulated differently after
    # rounding-level changes of the rays (test_gpu_psf.compare_e2e), and then
    # the centroids differ by up to sum |dpsf| times the largest offset, n/2
    # pixels
    radius = got.system[-1].distance
    x, y, t = got.opd_rays(radius)
    xh, yh, th = ref.opd(resample=False, radius=radius)
    ok = np.isfinite(x) & np.isfinite(y) & np.isfinite(t)
    okh = np.isfinite(xh) & np.isfinite(yh) & np.isfinite(th)
    same_tri = np.array_equal(ok, okh) and np.array_equal(
        psf_oracle.triangulate(x[ok], y[ok]).simplices,
        psf_oracle.triangulate(xh[okh], yh[okh]).simplices)
    pr, qr, psr = ref.psf()
    xr, yr, sr = map(np.fft.fftshift, (pr, qr, psr))
    x0, y0 = (sr*xr).sum(), (sr*yr).sum()
    dx = (xr - x0)[1, 0] - (xr - x0)[0, 0]
    dc = (abs(r["x0"]/r["dx"] - x0/dx), abs(r["y0"]/r["dx"] - y0/dx))
    tol = max(1e-9, np.abs(psf - psr).sum()*psf.shape[0]/2)
    print("%s f%.1f %d: psf %s, %d bins, centre %s, |dcentre| vs reference %.1e %.1e px "
          "(same triangulation %s, tolerance %.1e)"
          % (name, field, nrays, psf.shape, r["ee"].size, r["center"], *dc, same_tri, tol))
    assert max(dc) <= tol, (dc, same_tri)
    got.free()
