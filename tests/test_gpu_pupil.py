"""The direct-sum diffraction PSF on the device (rtx_pupil_sum,
rtx_pupil_intensity, ResidentMixin.psf_direct, rayopt_b200.psfs) against the
long-double oracle (tests/pupil_oracle.py) within the error bound of
include/rtx.h -- a bound asserted to be <= 1e-11 in Strehl units in every
comparison, so that a loose bound cannot pass -- against the FFT PSF, and end
to end on the reference's Cooke triplet and folded mirror.  Needs a GPU."""
import warnings

import numpy as np
import pytest

import pupil_oracle as po
import ref_shim
from rayopt_b200._lib import RtxError
from rayopt_b200.engine import pupil_bound, pupil_spec

pytestmark = pytest.mark.gpu

LAM, R = 5e-4, 50.
PITCH = .61*LAM/.2/8                      # an eighth of the Airy radius at NA 0.2


@pytest.fixture(scope="module")
def eng():
    from rayopt_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def rays(N, seed, bad=False):
    """N rays on a sphere of radius R over a pupil of NA 0.2 with about a
    wave of aberration; with `bad`, NaN and inf in A, P and w"""
    rng = np.random.default_rng(seed)
    r = 10*np.sqrt(rng.random(N))
    th = 2*np.pi*rng.random(N)
    x, y = r*np.cos(th), r*np.sin(th)
    P = np.stack([x, y, -np.sqrt(R*R - x*x - y*y)], -1)
    A = 123.25 + 3e-4*(r/10)**4 + 1e-4*rng.standard_normal(N)
    w = rng.random(N) + .5
    if bad and N >= 8:
        at = rng.choice(N, 6, replace=False)
        A[at[0]], A[at[1]] = np.nan, np.inf
        P[at[2], 0], P[at[3], 2] = np.nan, -np.inf
        w[at[4]], w[at[5]] = np.nan, np.inf
    return A, P, w


def spec_for(nx, ny, K, a0=123.25, center=(0., 0.)):
    z = np.linspace(-.02, .03, K)
    return pupil_spec(z, (nx, ny), center[0] - (nx//2)*PITCH, PITCH,
                      center[1] - (ny//2)*PITCH, PITCH*1.25, a0, LAM, 1/LAM, R)


def axes(spec):
    s = spec[0]
    nx, ny, K = int(s["nx"]), int(s["ny"]), int(s["planes"])
    p = s["p0"] + np.arange(nx)*s["dp"]
    q = s["q0"] + np.arange(ny)*s["dq"]
    return p, q, s["z"][:K].copy()


GUARD = 37
SENTINEL = 7.25 - 3.5j


def device_sum(eng, A, P, w, spec, U0=None, N=None):
    """pupil_sum into a guarded U (initial value U0); returns (U, count,
    sum w) and checks the guard bands"""
    s = spec[0]
    K, nx, ny = int(s["planes"]), int(s["nx"]), int(s["ny"])
    n = K*nx*ny
    host = np.full(n + 2*GUARD, SENTINEL)
    host[GUARD:GUARD + n] = 0 if U0 is None else U0.ravel()
    buf = eng.to_device(host)
    dA, dP = eng.to_device(np.r_[A, 0.]), eng.to_device(np.r_[P.ravel(), 0, 0, 0].reshape(-1, 3))
    dw = None if w is None else eng.to_device(np.r_[w, 0.])
    try:
        cnt, sw = eng.pupil_sum(dA, dP, spec, buf.rows(GUARD, GUARD + n), w=dw,
                                N=len(A) if N is None else N)
        out = buf.download()
    finally:
        for a in (buf, dA, dP, dw):
            if a is not None:
                a.free()
    assert (out[:GUARD] == SENTINEL).all() and (out[GUARD + n:] == SENTINEL).all()
    return out[GUARD:GUARD + n].reshape(K, nx, ny), cnt, sw


def check_oracle(U, cnt, sw, A, P, w, spec, chunks=1):
    s = spec[0]
    p, q, z = axes(spec)
    Uo, n, swo, _ = po.pupil_sum(A, P, w, s["a0"], LAM, 1/LAM, R, p, q, z)
    assert cnt == n
    assert abs(sw - swo) <= 1e-13*max(abs(swo), 1)
    phi = po.phi_bound(A, P, w, s["a0"], LAM, 1/LAM, R, s["p0"], s["dp"], len(p), s["q0"],
                       s["dq"], len(q), z)
    ok = np.isfinite(A) & np.isfinite(P).all(1) & np.isfinite(np.ones(len(A)) if w is None else w)
    sabs = float(np.abs(np.ones(len(A)) if w is None else w)[ok].sum())
    bound = pupil_bound(len(A), phi, sabs, chunks)
    if n:
        assert 2*bound/swo <= 1e-11, 2*bound/swo           # Strehl units
    err = np.maximum(np.abs(U.real - Uo.real.astype(float)), np.abs(U.imag - Uo.imag.astype(float)))
    assert err.max(initial=0) <= bound, (err.max()/bound, bound)
    return Uo


CASES = [(0, 8, 8, 1, False), (1, 37, 23, 1, True), (31, 64, 64, 1, False),
         (33, 64, 32, 2, True), (2048, 37, 23, 3, False), (2049, 130, 70, 5, True),
         (4097, 37, 23, 16, True), (70001, 64, 64, 9, False), (10**6, 9, 7, 1, True),
         (10**6, 17, 9, 2, False)]


@pytest.mark.parametrize("N,nx,ny,K,weighted", CASES)
def test_sum_against_oracle(eng, N, nx, ny, K, weighted):
    A, P, w = rays(N, N + nx, bad=N > 100)
    w = w if weighted else None
    spec = spec_for(nx, ny, K)
    U, cnt, sw = device_sum(eng, A, P, w, spec)
    if N == 0:
        assert cnt == 0 and sw == 0 and (U == 0).all()
        return
    check_oracle(U, cnt, sw, A, P, w, spec)


def test_bits_across_calls_contexts_and_grids(eng):
    """the same rays and record give the same bits in every call and
    context; a grid that is a corner of another gives that corner's bits"""
    from rayopt_b200.engine import Engine
    A, P, w = rays(9000, 5, bad=True)
    spec = spec_for(64, 64, 1)
    U1, *_ = device_sum(eng, A, P, w, spec)
    U2, *_ = device_sum(eng, A, P, w, spec)
    e2 = Engine(0)
    try:
        U3, *_ = device_sum(e2, A, P, w, spec)
    finally:
        e2.close()
    assert np.array_equal(U1, U2) and np.array_equal(U1, U3)
    s = spec[0]
    small = pupil_spec(s["z"][:1], (37, 23), s["p0"], s["dp"], s["q0"], s["dq"], s["a0"], LAM,
                       1/LAM, R)
    U4, *_ = device_sum(eng, A, P, w, small)
    assert np.array_equal(U4[0], U1[0, :37, :23])


def test_chunks_and_accumulation(eng):
    """calls add: a bundle summed in two chunks is within the bound of one
    call, and a second call of the same rays doubles U exactly"""
    A, P, w = rays(50000, 6, bad=True)
    spec = spec_for(40, 24, 2)
    U, cnt, sw = device_sum(eng, A, P, w, spec)
    Ua, ca, sa = device_sum(eng, A[:20000], P[:20000], w[:20000], spec)
    Ub, cb, sb = device_sum(eng, A[20000:], P[20000:], w[20000:], spec, U0=Ua)
    assert ca + cb == cnt
    check_oracle(Ub, ca + cb, sa + sb, A, P, w, spec, chunks=2)
    U2, *_ = device_sum(eng, A, P, w, spec, U0=U)
    assert np.array_equal(U2, 2*U)


def test_intensity_and_stats(eng):
    A, P, w = rays(20000, 7)
    spec = spec_for(70, 50, 3)
    U, cnt, sw = device_sum(eng, A, P, w, spec)
    old = np.random.default_rng(1).random(U.shape)
    dU, dpsf = eng.to_device(U), eng.to_device(old)
    try:
        st = eng.pupil_intensity(spec, dU, dpsf, 1/sw**2)
        psf = dpsf.download()
    finally:
        dU.free(), dpsf.free()
    want = old + np.abs(U)**2/sw**2
    assert np.abs(psf - want).max() <= 4e-16*want.max()
    p, q, _ = axes(spec)
    for k in range(3):
        f = psf[k]
        assert abs(st[k, 0] - f.sum()) <= 1e-13*f.sum()
        assert st[k, 1] == f.max() and st[k, 2] == np.argmax(f)
        assert abs(st[k, 3] - (f*p[:, None]).sum()) <= 1e-13*(f*np.abs(p)[:, None]).sum()
        assert abs(st[k, 4] - (f*q[None, :]).sum()) <= 1e-13*(f*np.abs(q)[None, :]).sum()


def test_intensity_first_maximum_on_ties(eng):
    """equal maxima in pixel groups that meet out of index order in the
    block's tree (512 and 1024), and an all-zero plane: the first index"""
    spec = spec_for(64, 64, 2)
    old = np.zeros((2, 64, 64))
    old[0].flat[[1024, 512, 3000]] = 1.
    dU, dpsf = eng.to_device(np.zeros((2, 64, 64), np.complex128)), eng.to_device(old)
    try:
        st = eng.pupil_intensity(spec, dU, dpsf, 1.)
    finally:
        dU.free(), dpsf.free()
    assert st[0, 1] == 1 and st[0, 2] == 512
    assert st[1, 1] == 0 and st[1, 2] == 0


def test_fft_identity_on_regridded_nodes(eng):
    """rtx_psf's PSF of an rtx_grid_linear OPD is |U|^2/(m nx ny) of the
    nodes as rays on the FFT's frequency grid (fftshifted)"""
    from scipy.spatial import Delaunay
    rng = np.random.default_rng(3)
    h, n, pad, lam, rad = 4., 24, 2, 5.5e-4, 80.
    r, th = h*np.sqrt(rng.random(3000)), 2*np.pi*rng.random(3000)
    pts = np.stack([r*np.cos(th), r*np.sin(th)], -1)
    t = .4*(pts[:, 0]/h)**2 - .3*(pts[:, 1]/h)**3
    xs, ys = np.mgrid[-1:1:1j*n, -1:1:1j*n]*h
    o_dev = eng.grid_linear(pts, t, Delaunay(pts), n, xs[:, 0].copy(), download=False)
    o = o_dev.download()
    fft_dev, raw = eng.psf(o_dev, pad)
    fft = fft_dev.download()
    fft_dev.free(), o_dev.free()
    import psf_oracle
    _, _, fft_np = psf_oracle.psf(xs, o, pad, lam, rad)
    e_fft = np.abs(fft - fft_np).max()                  # cuFFT against numpy's FFT
    nx = pad*n
    df = 1/(nx*(xs[1, 0] - xs[0, 0])/lam/rad)
    spec = pupil_spec([0.], (nx, nx), -(nx//2)*df, df, -(nx//2)*df, df, 0., lam, 1/lam, rad)
    A, Pn = po.nodes_as_rays(xs, ys, o, lam)
    U, m, sw = device_sum(eng, A, Pn, None, spec)
    assert m == np.isfinite(o).sum()
    got = np.abs(U[0])**2/(m*nx*nx)
    p, q, _ = axes(spec)
    phi = po.phi_bound(A, Pn, None, 0., lam, 1/lam, rad, p[0], df, nx, q[0], df, nx, [0.])
    e_sum = pupil_bound(m, phi, m)
    tol = (2*m*e_sum + e_sum**2)/(m*nx*nx) + e_fft + 1e-15*fft.max()
    assert np.abs(got - np.fft.fftshift(fft)).max() <= tol


def test_refusals_launch_nothing(eng):
    from rayopt_b200._lib import check
    import ctypes as C
    A, P, w = rays(100, 8)
    dA, dP = eng.to_device(A), eng.to_device(P)
    U = eng.to_device(np.full(64*2, SENTINEL))
    psf = eng.to_device(np.zeros(64*2))
    good = spec_for(8, 8, 2)
    bad = []
    for k, v in (("planes", 0), ("planes", 17), ("nx", 0), ("ny", 4097), ("reserved", 1),
                 ("wavelength", 0.), ("radius", np.nan), ("a0", np.inf), ("kappa", np.nan),
                 ("p0", np.nan), ("dp", np.inf), ("q0", -np.inf), ("dq", np.nan)):
        s = good.copy()
        s[k] = v
        bad.append(s)
    s = good.copy()
    s["z"][0, 1] = np.nan
    bad.append(s)
    n0 = eng.launch_count()
    cnt, sw = C.c_int64(-5), C.c_double(-5)
    pp = lambda a: a.ctypes.data_as(C.c_void_p)
    try:
        for s in bad:
            assert eng.lib.rtx_pupil_sum(eng.ctx, 100, dA.ptr, dP.ptr, None, pp(s), U.ptr,
                                         C.byref(cnt), C.byref(sw)) == -1
            assert eng.lib.rtx_pupil_intensity(eng.ctx, pp(s), U.ptr, 1., psf.ptr, None) == -1
        gp = pp(good)
        for args in ((None, 100, dA.ptr, dP.ptr, None, gp, U.ptr, C.byref(cnt), C.byref(sw)),
                     (eng.ctx, -1, dA.ptr, dP.ptr, None, gp, U.ptr, C.byref(cnt), C.byref(sw)),
                     (eng.ctx, 100, None, dP.ptr, None, gp, U.ptr, C.byref(cnt), C.byref(sw)),
                     (eng.ctx, 100, dA.ptr, None, None, gp, U.ptr, C.byref(cnt), C.byref(sw)),
                     (eng.ctx, 100, dA.ptr, dP.ptr, None, None, U.ptr, C.byref(cnt), C.byref(sw)),
                     (eng.ctx, 100, dA.ptr, dP.ptr, None, gp, None, C.byref(cnt), C.byref(sw)),
                     (eng.ctx, 100, dA.ptr, dP.ptr, None, gp, U.ptr, None, C.byref(sw)),
                     (eng.ctx, 100, dA.ptr, dP.ptr, None, gp, U.ptr, C.byref(cnt), None)):
            assert eng.lib.rtx_pupil_sum(*args) == -1
        assert eng.lib.rtx_pupil_intensity(eng.ctx, gp, U.ptr, np.nan, psf.ptr, None) == -1
        assert eng.lib.rtx_pupil_intensity(eng.ctx, gp, None, 1., psf.ptr, None) == -1
        assert eng.lib.rtx_pupil_intensity(eng.ctx, gp, U.ptr, 1., None, None) == -1
        assert eng.launch_count() == n0
        assert (U.download() == SENTINEL).all() and (psf.download() == 0).all()
        # N = 0 adds nothing and launches nothing
        check(eng.lib.rtx_pupil_sum(eng.ctx, 0, None, None, None, gp, U.ptr, C.byref(cnt),
                                    C.byref(sw)))
        assert cnt.value == 0 and sw.value == 0 and eng.launch_count() == n0
        with pytest.raises(ValueError):
            pupil_spec(np.zeros(17), (8, 8), 0, 1, 0, 1, 0, 1, 1, 1)
    finally:
        for a in (dA, dP, U, psf):
            a.free()


# ---- end to end on the reference's systems ---------------------------------
needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="reference tree not present")


def _system(R, name):
    import yaml
    import systems_yaml
    s = R.System(**yaml.safe_load(systems_yaml.SYSTEMS[name]))
    s.update()
    s.paraxial.refocus()
    return s


@needs_ref
@pytest.mark.parametrize("field", [0., .7])
def test_psf_direct_against_oracle_and_psf_device(eng, field):
    """psf_direct on the Cooke triplet: the whole grid against the oracle of
    the trace's own per-ray OPD (tight), and its Strehl at the chief point
    against psf_device's FFT PSF at p = q = 0 in Strehl units (psf nx ny /
    #finite nodes), within the agreement the oracle shows between the two
    quadratures on the reference's own rays"""
    from rayopt_b200 import ResidentTrace
    from test_pupil_oracle import COOKE_STREHL_TOL
    R_ = ref_shim.load()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        s = _system(R_, "cooke")
        t = ResidentTrace(s, engine=eng)
        t.rays_point((0, field), nrays=10000, distribution="hexapolar", clip=False)
        p, q, fft = t.psf_device()
        regrid = fft[0, 0]*fft.size/t.psf_stats["count"]
        pp, qq, psf = t.psf_direct(pixels=(33, 33))
        st, nrays = t.psf_direct_stats, t.nrays
        x, y, w = t.opd_rays(s[-1].distance)
        lam = t.l/s.scale
        kappa = t.n[t.length - 2]/lam                    # n of the image space
        t.free()
    assert psf.shape == (1, 33, 33) and st["count"] + st["left_out"] == nrays
    ok = np.isfinite(x) & np.isfinite(y) & np.isfinite(w)
    P = np.stack([x[ok], y[ok], np.zeros(ok.sum())], -1)
    U, n, sw, _ = po.pupil_sum(-lam*w[ok], P, None, 0., lam, kappa, s[-1].distance, pp[:, 0],
                               qq[0], [0.])
    assert n == st["count"]
    assert np.abs(psf[0] - (np.abs(U[0])**2/sw**2).astype(float)).max() <= 1e-9
    assert abs(st["strehl"][0] - regrid) <= COOKE_STREHL_TOL, (st["strehl"], regrid)
    # the grid's centre pixel is the chief point, exactly
    assert pp[16, 16] == 0 and qq[16, 16] == 0
    assert abs(psf[0, 16, 16] - st["strehl"][0]) <= 1e-12


@needs_ref
def test_psf_direct_centroid_against_psf_device(eng):
    """the PSF centroid of psf_direct against psf_device's at field 0.7,
    within the agreement the oracle shows between the two quadratures"""
    from rayopt_b200 import ResidentTrace
    from test_pupil_oracle import COOKE_CENTROID_TOL
    R_ = ref_shim.load()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        s = _system(R_, "cooke")
        t = ResidentTrace(s, engine=eng)
        t.rays_point((0, .7), nrays=40000, distribution="hexapolar", clip=False)
        par = s.paraxial
        airy = par.airy_radius[1]/par.wavelength*t.l
        p, q, out = t.psf_device(download=False)
        out.free()
        fs = t.psf_stats
        regrid = np.array([fs["cp"], fs["cq"]])/fs["sum"]
        t.psf_direct(pixels=(200, 200), pitch=airy/2)
        direct = t.psf_direct_stats["centroid"][0]
        t.free()
    assert abs(regrid[1]) > .3*airy                      # coma moves it: not a trivial 0
    assert np.abs(direct - regrid).max() <= COOKE_CENTROID_TOL*airy, (direct/airy, regrid/airy)


@needs_ref
@pytest.mark.parametrize("name,dz", [("cooke", 0.), ("mirror", 3.), ("mirror", -3.)])
def test_peak_plane_near_refocus(eng, name, dz):
    """through focus on axis the intensity peaks within FOCUS_TOL of the
    plane refocus() finds, in the image frame's +z; the folded mirror, its
    image moved by dz Rayleigh ranges, checks the sign in a reflected image
    space"""
    from rayopt_b200 import ResidentTrace
    from test_pupil_oracle import FOCUS_TOL
    R_ = ref_shim.load()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        s = _system(R_, name)
        rr = s.paraxial.rayleigh_range[1]
        s[-1].distance += dz*rr
        t = ResidentTrace(s, engine=eng)
        t.rays_point((0, 0.), nrays=10000, distribution="hexapolar", clip=False)
        shift = t.refocus_fused()
        s[-1].distance -= shift                          # back to the traced image
        z = np.linspace(-6, 6, 25)*rr
        strehl = []
        for part in (z[:13], z[13:]):
            t.psf_direct(pixels=(1, 1), defocus=part)
            strehl.append(t.psf_direct_stats["strehl"])
        t.free()
    peak = z[np.argmax(np.concatenate(strehl))]
    assert abs(peak - shift) <= FOCUS_TOL*rr, (name, dz, peak/rr, shift/rr)


@needs_ref
@pytest.mark.parametrize("name", ["cooke", "mirror"])
def test_through_focus_centroid_follows_spot(eng, name):
    """far from focus the PSF is the geometric shadow: its centroid follows
    the spot centroid (folded mirror: the signs in a reflected image space)"""
    from rayopt_b200 import ResidentTrace
    R_ = ref_shim.load()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        s = _system(R_, name)
        t = ResidentTrace(s, engine=eng)
        t.rays_point((0, .7), nrays=40000, distribution="hexapolar", clip=False)
        par = s.paraxial
        airy = par.airy_radius[1]/par.wavelength*t.l
        y, i = np.asarray(t.y[-1]), np.asarray(t.i[-1])
        c, u = y[t.ref, :2], i[t.ref, :2]/i[t.ref, 2]
        ok = np.isfinite(y).all(1) & np.isfinite(i).all(1)
        for zk in np.array([-1., 1.])*10*par.rayleigh_range[1]:
            # the grid follows the chief ray to the plane; the PSF must be there
            _, _, psf = t.psf_direct(pixels=(160, 160), pitch=airy/2, center=zk*u, defocus=[zk])
            st = t.psf_direct_stats
            spot = (y[ok, :2] - c + zk*i[ok, :2]/i[ok, 2:]).mean(0)
            # a circular pupil's PSF integrates to (lambda/NA)^2/pi in Strehl
            # units: at least half of it is on the grid
            assert st["sum"][0]*(airy/2)**2 > .5*(airy/.61)**2/np.pi, (name, zk)
            assert np.abs(st["centroid"][0] - spot).max() <= airy, \
                (name, zk, st["centroid"][0], spot)
        t.free()


@needs_ref
def test_psfs_poly_and_lateral_colour(eng):
    """the polychromatic PSF is the weighted mean of the per-wavelength PSFs
    on one grid, and each wavelength's PSF sits at its chief ray's lateral
    colour offset: it equals psf_direct of that wavelength's own trace on the
    same sample points (grid centre at minus the offset), and not on the
    mirrored ones; its peak is the in-frame peak moved by the offset"""
    from rayopt_b200 import ResidentTrace, psfs
    R_ = ref_shim.load()
    n = 192                                   # 24 Airy radii: the full field's PSF fits
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        s = _system(R_, "cooke")
        W = len(s.wavelengths)
        wts = np.arange(1., W + 1)
        par = s.paraxial
        pitch = par.airy_radius[1]/8
        out = psfs(s, heights=(0., 1.), nrays=20000, pixels=(n, n), pitch=pitch,
                   spectral_weights=wts, engine=eng, per_wavelength=True)
        frames = []
        for w, wl in enumerate(s.wavelengths):
            off = out["chief_offset"][1, w]
            t = ResidentTrace(s, engine=eng)
            t.rays_point((0, 1.), wl, nrays=20000, distribution="hexapolar", clip=True)
            # the in-frame reference samples the points of the common grid
            # shifted by whole pixels m: its peak index plus m is the peak's
            m = np.rint(off/pitch)
            got = [t.psf_direct(pixels=(n, n), pitch=pitch, center=c)[2][0]
                   for c in (-off, off, m*pitch - off)]
            frames.append(got)
            t.free()
    assert out["poly"].shape == (2, 1, n, n) and out["psf"].shape == (2, W, 1, n, n)
    want = np.einsum("w,hwkab->hkab", wts, out["psf"])/wts.sum()
    assert np.abs(out["poly"] - want).max() <= 1e-14*want.max()
    assert (out["count"] > 0).all()
    assert np.abs(out["chief_offset"][0]).max() <= 1e-12     # no lateral colour on axis
    offs = out["chief_offset"][1]/pitch
    assert np.abs(offs).max() >= 3, offs                      # pixels: a sign flip shows
    for w in range(W):
        mine, mirrored, centred = frames[w]
        f = out["psf"][1, w, 0]
        assert np.abs(f - mine).max() <= 1e-6*f.max(), w
        if np.abs(offs[w]).max() >= 1:
            assert np.abs(f - mirrored).max() >= .1*f.max(), w
        # peaks: the common grid's is the in-frame one moved by the lateral
        # colour, to within a pixel
        a, b = np.unravel_index(np.argmax(f), f.shape)
        a0, b0 = np.unravel_index(np.argmax(centred), centred.shape)
        assert min(a, b, a0, b0) >= 8 and max(a, b, a0, b0) < n - 8, (w, a, b, a0, b0)
        d = np.array([a - a0, b - b0]) - offs[w]
        assert np.abs(d).max() <= 1, (w, d)
