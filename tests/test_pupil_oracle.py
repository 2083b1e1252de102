"""The long-double direct-sum oracle of rtx_pupil_sum (tests/pupil_oracle.py)
against mpmath, the FFT PSF of a regridded pupil, the shift theorem, and the
closed-form Airy, annular and defocus patterns; and, on the reference's own
Cooke triplet rays, against the reference's psf() -- the agreement the
device's end-to-end checks rely on."""
import warnings

import numpy as np
import pytest

import psf_oracle
import pupil_oracle as po
import ref_shim


def random_rays(n, seed, R=50.):
    rng = np.random.default_rng(seed)
    r = 10*np.sqrt(rng.random(n))
    th = 2*np.pi*rng.random(n)
    x, y = r*np.cos(th), r*np.sin(th)
    P = np.stack([x, y, -np.sqrt(R*R - x*x - y*y)], -1)
    A = 100 + 3e-4*rng.standard_normal(n)
    return A, P, rng.random(n) + .5


def test_against_mpmath():
    mpmath = pytest.importorskip("mpmath")
    mpmath.mp.dps = 40
    A, P, w = random_rays(7, 1)
    a0, lam, kappa, R = A[0], 5e-4, 1/5e-4, 50.
    p, q, z = np.array([-.01, 0, .013]), np.array([.002, -.02]), np.array([0., .05])
    U, n, sw, _ = po.pupil_sum(A, P, w, a0, lam, kappa, R, p, q, z)
    assert n == 7 and abs(sw - w.sum()) < 1e-14
    for k in range(2):
        for a in range(3):
            for b in range(2):
                s = mpmath.mpc(0)
                for j in range(7):
                    ph = ((mpmath.mpf(A[j]) - mpmath.mpf(a0))/mpmath.mpf(lam)
                          + mpmath.mpf(kappa)*(-mpmath.mpf(P[j, 0])*mpmath.mpf(p[a])
                                               - mpmath.mpf(P[j, 1])*mpmath.mpf(q[b])
                                               - mpmath.mpf(P[j, 2])*mpmath.mpf(z[k]))/mpmath.mpf(R))
                    s += mpmath.mpf(w[j])*mpmath.exp(2j*mpmath.pi*ph)
                assert abs(complex(s) - complex(U[k, a, b])) < 1e-12, (k, a, b)


def test_skips_and_counts_non_finite_rays():
    A, P, w = random_rays(20, 2)
    A[3], P[5, 1], w[7] = np.nan, np.inf, np.nan
    U, n, sw, _ = po.pupil_sum(A, P, w, A[0], 5e-4, 2e3, 50., [0.], [0.], [0.])
    ok = np.ones(20, bool)
    ok[[3, 5, 7]] = False
    U2, n2, _, _ = po.pupil_sum(A[ok], P[ok], w[ok], A[0], 5e-4, 2e3, 50., [0.], [0.], [0.])
    assert n == n2 == 17 and U[0, 0, 0] == U2[0, 0, 0] and abs(sw - w[ok].sum()) < 1e-13


@pytest.mark.parametrize("n,pad", [(16, 2), (21, 4)])
def test_fft_identity(n, pad):
    """rtx_psf's PSF of a regridded pupil is |U|^2/(m nx ny) of the nodes as
    rays on the FFT's own frequency grid (m finite nodes)"""
    rng = np.random.default_rng(n)
    h, lam, R = 4., 5.5e-4, 80.
    xs, ys, _ = psf_oracle.grid(n, h)
    o = .3*(xs/h)**2 - .2*(ys/h)**3 + .05*rng.standard_normal(xs.shape)
    o[xs*xs + ys*ys > h*h] = np.nan
    p, q, want = psf_oracle.psf(xs, o, pad, lam, R)
    A, P = po.nodes_as_rays(xs, ys, o, lam, a0=12.5)
    U, m, _, _ = po.pupil_sum(A, P, None, 12.5, lam, 1/lam, R, p[:, 0], q[0], [0.])
    got = (np.abs(U[0])**2/(m*p.size)).astype(float)
    assert np.abs(got - want).max() <= 1e-12*want.max()


def test_shift_theorem():
    A, P, w = random_rays(50, 3)
    lam, kappa, R, s = 5e-4, 1/5e-4, 50., .0123
    p, q = np.linspace(-.05, .05, 7), np.linspace(-.04, .04, 5)
    U, *_ = po.pupil_sum(A, P, w, A[0], lam, kappa, R, p + s, q, [0.])
    As = A + lam*kappa*s*(-P[:, 0]/R)
    V, *_ = po.pupil_sum(As, P, w, A[0], lam, kappa, R, p, q, [0.])
    assert np.abs(U - V).max() < 1e-10*w.sum()


def disc_rays(h, m, eps=0.):
    """the nodes of an (m, m) square grid inside a disc of radius h (and
    outside eps h): a uniformly sampled pupil on a plane at z = -R"""
    x = (np.arange(m) - (m - 1)/2)*(2*h/m)
    xs, ys = np.meshgrid(x, x, indexing="ij")
    r2 = xs*xs + ys*ys
    keep = (r2 <= h*h) & (r2 >= (eps*h)**2)
    return xs[keep], ys[keep]


@pytest.mark.parametrize("eps", [0., .4])
def test_airy_and_annulus(eps):
    """a flat wavefront over a disc gives the Airy pattern, over an annulus
    the annular pattern (the regridded FFT path fills the hole)"""
    h, R, lam = 5., 100., 5e-4
    x, y = disc_rays(h, 400, eps)
    P = np.stack([x, y, -R*np.ones_like(x)], -1)
    A = np.zeros(len(x))
    r = np.linspace(0, 4*.61*lam*R/h, 41)           # four Airy radii
    U, n, sw, _ = po.pupil_sum(A, P, None, 0., lam, 1/lam, R, r, [0.], [0.])
    got = (np.abs(U[0, :, 0])**2/sw**2).astype(float)
    v = 2*np.pi*h*r/(lam*R)
    want = po.annulus(v, eps) if eps else po.airy(v)
    assert np.abs(got - want).max() < 2e-3, np.abs(got - want).max()


def test_defocus_symmetric_on_axis():
    """a perfect spherical wave: the on-axis intensity is even in z and
    falls as the disc's |sinc(kappa z h^2 / (2 R^2))|^2"""
    h, R, lam = 5., 100., 5e-4
    x, y = disc_rays(h, 300)
    P = np.stack([x, y, -np.sqrt(R*R - x*x - y*y)], -1)
    A = np.zeros(len(x))
    z = np.linspace(-.5, .5, 11)
    U, n, sw, _ = po.pupil_sum(A, P, None, 0., lam, 1/lam, R, [0.], [0.], z)
    I = (np.abs(U[:, 0, 0])**2/sw**2).astype(float)
    assert np.abs(I - I[::-1]).max() < 1e-12
    assert np.abs(I - np.sinc(z*h*h/(2*R*R*lam))**2).max() < 5e-3


# ---- the reference's Cooke triplet: direct sum against its psf() --------
needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="no reference tree staged")

# Measured: the oracle's direct sum over the reference's opd(resample=False)
# rays against the reference's psf() (regridded, 4x resampled, 4x padded) at
# the chief point, in Strehl units, Cooke triplet at its paraxial focus
# (Strehl 0.02-0.04), hexapolar rays with equal weights:
#   field 0:   0.0184 vs 0.0402 (1e3 rays), 0.0321 vs 0.0385 (1e4), 0.0352 vs 0.0383 (4e4)
#   field 0.7: 0.0146 vs 0.0207 (1e3 rays), 0.0172 vs 0.0181 (1e4), 0.0174 vs 0.0176 (4e4)
# The two are different quadratures of the same pupil integral and meet as
# the ray count grows; at 1e4 rays they differ by at most 6.5e-3.
# The same difference on the folded mirror defocused by one Rayleigh range
# (Strehl 0.32): 1.3e-2 at 1e4 rays, 6.0e-3 at 4e4, at fields 0 and 0.7.  It
# is the quadrature of equal-weight hexapolar rays (the rim ring counts as a
# full ring), not an error of either sum; the device's own sum is held to the
# oracle on its own rays far tighter (tests/test_gpu_pupil.py).
COOKE_STREHL_TOL = 1e-2     # at 1e4 rays

# Measured: the PSF centroid of the same two quadratures, Cooke triplet at
# field 0.7, the direct sum on a square grid of pitch airy/2 centred on the
# chief point, the regridded FFT PSF over its whole periodic grid:
#   1e4 rays: 0.46 / 0.21 / 0.059 Airy radii apart on 96 / 128 / 160 pixels
#   4e4 rays: 0.065 / 0.011 Airy radii apart on 160 / 200 pixels
# (the grid must hold the aberrated PSF's wings).  The device check uses
# 4e4 rays, 200 pixels and 0.05 Airy radii.
COOKE_CENTROID_TOL = .05    # Airy radii, at 4e4 rays on 200 x 200 pixels of airy/2

# Measured: the peak of the on-axis intensity through focus (planes 0.25
# Rayleigh ranges apart) against the least-squares focus of refocus():
# Cooke triplet -3.25 vs -3.24 Rayleigh ranges; folded mirror with its image
# moved by +3 / -3 Rayleigh ranges: -3.50 vs -3.00 and +2.50 vs +3.00.
FOCUS_TOL = .75             # Rayleigh ranges


def traced(R, name, field, nrays, dz=0.):
    """a reference System refocused, its image moved by dz Rayleigh ranges,
    and its GeometricTrace of hexapolar rays"""
    import yaml
    import systems_yaml
    warnings.simplefilter("ignore")
    np.seterr(all="ignore")
    s = R.System(**yaml.safe_load(systems_yaml.SYSTEMS[name]))
    s.update()
    s.paraxial.refocus()
    s[-1].distance += dz*s.paraxial.rayleigh_range[1]
    g = R.GeometricTrace(s)
    g.rays_point((0, field), nrays=nrays, distribution="hexapolar", clip=False)
    return s, g


def cooke(R, field, nrays):
    return traced(R, "cooke", field, nrays)


def ref_rays(s, g, field0=True):
    """(A - a0, P, lambda, R) of the reference's own opd(resample=False) rays
    on psf()'s sphere; P_z from the sphere, which holds on axis, where the
    chief ray's point is the sphere's vertex"""
    radius = s[-1].distance
    x, y, t = g.opd(resample=False, radius=radius)
    lam = g.l/s.scale
    ok = np.isfinite(x) & np.isfinite(y) & np.isfinite(t)
    x, y = x[ok], y[ok]
    pz = -np.sign(radius)*np.sqrt(radius*radius - x*x - y*y)
    return -lam*t[ok], np.stack([x, y, pz], -1), lam, radius


@needs_ref
@pytest.mark.parametrize("field", [0., .7])
def test_reference_cooke_chief_strehl(field):
    R = ref_shim.load()
    s, g = cooke(R, field, 10000)
    radius = s[-1].distance
    x, y, t = g.opd(resample=False, radius=radius)
    lam = g.l/s.scale
    ok = np.isfinite(x) & np.isfinite(y) & np.isfinite(t)
    P = np.stack([x[ok], y[ok], np.zeros(ok.sum())], -1)
    U, n, sw, _ = po.pupil_sum(-lam*t[ok], P, None, 0., lam, 1/lam, radius, [0.], [0.], [0.])
    direct = float(abs(U[0, 0, 0])**2/sw**2)
    p, q, psf = g.psf()
    xs, _, o = g.opd(radius=radius)
    m = np.isfinite(o).sum()
    regrid = psf[0, 0]*psf.size/m
    assert abs(direct - regrid) <= COOKE_STREHL_TOL, (direct, regrid)


@needs_ref
def test_reference_cooke_centroid():
    R = ref_shim.load()
    s, g = cooke(R, .7, 40000)
    A, P, lam, radius = ref_rays(s, g)
    par = s.paraxial
    airy = par.airy_radius[1]/par.wavelength*g.l
    ax = (np.arange(200) - 100)*airy/2
    U, n, sw, _ = po.pupil_sum(A, P, None, 0., lam, 1/lam, radius, ax, ax, [0.])
    I = (np.abs(U[0])**2).astype(float)
    direct = np.array([(I*ax[:, None]).sum(), (I*ax[None, :]).sum()])/I.sum()
    p, q, psf = g.psf()
    regrid = np.array([(psf*p).sum(), (psf*q).sum()])/psf.sum()
    assert np.abs(direct - regrid).max() <= COOKE_CENTROID_TOL*airy, (direct/airy, regrid/airy)


@needs_ref
@pytest.mark.parametrize("name,dz", [("cooke", 0.), ("mirror", 3.), ("mirror", -3.)])
def test_reference_peak_plane_near_refocus(name, dz):
    """the on-axis intensity peaks within FOCUS_TOL of refocus()'s plane, in
    the image frame's +z (the folded mirror: a reflected image space)"""
    R = ref_shim.load()
    s, g = traced(R, name, 0., 10000, dz)
    A, P, lam, radius = ref_rays(s, g)
    rr = s.paraxial.rayleigh_range[1]
    z = np.linspace(-6, 6, 49)*rr
    U, *_ = po.pupil_sum(A, P, None, 0., lam, 1/lam, radius, [0.], [0.], z)
    peak = z[np.argmax(np.abs(U[:, 0, 0]))]
    d0 = s[-1].distance
    g.refocus()
    assert abs(peak - (s[-1].distance - d0)) <= FOCUS_TOL*rr, (peak/rr, (s[-1].distance - d0)/rr)

