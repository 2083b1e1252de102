"""Long-double oracle of rtx_pupil_sum (include/rtx.h): the Debye sum of the
pupil function over the rays,

    U_k(a, b) = sum_j w_j exp(2 pi i [(A_j - a0)/lambda
                                      + kappa (sx_j p_a + sy_j q_b + sz_j z_k)])

with s_j = -P_j/R, over the rays whose A, P and w are finite.  Every phase is
formed in long double and reduced modulo one turn before its cosine and sine,
so the oracle's own error is far below the device's bound."""
import numpy as np

LD = np.longdouble


def _phasor(turns):
    t = turns - np.round(turns)
    ang = 2*np.pi*t.astype(LD)
    return np.cos(ang) + 1j*np.sin(ang)


def terms(A, P, w, a0, lam, kappa, R):
    """(ok, sx, sy, sz, d, w) in long double: the summed rays' directions
    scaled by kappa, their reference phases (A - a0)/lambda and weights"""
    A = np.asarray(A, np.float64)
    P = np.asarray(P, np.float64).reshape(-1, 3)
    w = np.ones(len(A)) if w is None else np.asarray(w, np.float64)
    ok = np.isfinite(A) & np.isfinite(P).all(1) & np.isfinite(w)
    s = -P[ok].astype(LD)/LD(R)*LD(kappa)
    d = (A[ok].astype(LD) - LD(a0))/LD(lam)
    return ok, s[:, 0], s[:, 1], s[:, 2], d, w[ok].astype(LD)


def pupil_sum(A, P, w, a0, lam, kappa, R, p, q, z, chunk=1 << 15):
    """(U clongdouble (K, nx, ny), count, sum w, phi): the sum, the rays
    summed, their weight and the phase size Phi of the bound in rtx.h for
    the grid axes p (nx,), q (ny,) and planes z (K,)"""
    ok, kx, ky, kz, d, w = terms(A, P, w, a0, lam, kappa, R)
    p = np.asarray(p, np.float64).astype(LD)
    q = np.asarray(q, np.float64).astype(LD)
    z = np.atleast_1d(np.asarray(z, np.float64)).astype(LD)
    U = np.zeros((len(z), len(p), len(q)), np.clongdouble)
    for j0 in range(0, len(d), chunk):
        sl = slice(j0, j0 + chunk)
        X = _phasor(kx[sl, None]*p[None, :])                    # (n, nx)
        Y = _phasor(ky[sl, None]*q[None, :])                    # (n, ny)
        for k, zk in enumerate(z):
            c = w[sl]*_phasor(d[sl] + kz[sl]*zk)
            U[k] += (X*c[:, None]).T @ Y
    pm = np.abs(p).max() if len(p) else 0
    qm = np.abs(q).max() if len(q) else 0
    phi = float((np.abs(d) + np.abs(kx)*pm + np.abs(ky)*qm + np.abs(kz)*np.abs(z).max()).max()) \
        if len(d) else 0.
    return U, int(ok.sum()), float(w.sum()), phi


def phi_bound(A, P, w, a0, lam, kappa, R, p0, dp, nx, q0, dq, ny, z):
    """Phi exactly as include/rtx.h defines it (axis ends |p0| + (nx-1)|dp|)"""
    ok, kx, ky, kz, d, _ = terms(A, P, w, a0, lam, kappa, R)
    if not len(d):
        return 0.
    return float((np.abs(d) + np.abs(kx)*(abs(p0) + (nx - 1)*abs(dp))
                  + np.abs(ky)*(abs(q0) + (ny - 1)*abs(dq))
                  + np.abs(kz)*np.abs(np.asarray(z, float)).max()).max())


def nodes_as_rays(xs, ys, o, lam, a0=0.):
    """the finite nodes of a regridded OPD o (waves) as rays: P = (x, y, 0),
    A = a0 - lambda o, so that exp(2 pi i (A - a0)/lambda) = exp(-2 pi i o),
    the pupil function rtx_psf transforms"""
    good = np.isfinite(o)
    P = np.stack([xs[good], ys[good], np.zeros(good.sum())], axis=-1)
    return a0 - lam*o[good], P


def airy(v):
    """[2 J1(v)/v]^2"""
    from scipy.special import j1
    v = np.asarray(v, float)
    with np.errstate(invalid="ignore", divide="ignore"):
        r = np.where(v == 0, 1., 2*j1(v)/np.where(v == 0, 1, v))
    return r*r


def annulus(v, eps):
    """the annular aperture's intensity, obscuration ratio eps, 1 at v = 0"""
    from scipy.special import j1
    v = np.asarray(v, float)

    def a(x):
        with np.errstate(invalid="ignore", divide="ignore"):
            return np.where(x == 0, 1., 2*j1(x)/np.where(x == 0, 1, x))
    f = (a(v) - eps*eps*a(eps*v))/(1 - eps*eps)
    return f*f
