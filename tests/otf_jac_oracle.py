"""Extended-precision statement of the OTF sums and their lens-parameter
derivatives (rtx_otf_jacobian_sums, include/rtx.h), from per-ray image points
q (N, 2) and derivatives J (P, 2, N).

TEST INFRASTRUCTURE ONLY: the product never imports it.

d = fl(q - c) in float64, as the kernel forms it.  Each phase nu_j d is formed
in long double (the product of two doubles rounded once), reduced mod 1
exactly, cos and sin of 2 pi frac are taken in long double, and the terms
exp(-2 pi i nu d) and -2 pi i nu J exp(-2 pi i nu d) are summed pairwise in
long double (otf_oracle's approach).  `oracle_error` bounds the result's own
error.
"""
import numpy as np

from otf_oracle import EPS_LD, LD, TWO_PI


def enter(q, J, c=None):
    """(d (N, 2) float64, in (N,) the rays that enter, bad (N,) the rays with
    a finite q and a non-finite derivative)"""
    q = np.asarray(q, np.float64)
    c = np.zeros(2) if c is None else np.asarray(c, np.float64).reshape(2)
    with np.errstate(invalid="ignore", over="ignore"):
        d = q[:, :2] - c
    qf = np.isfinite(d).all(1)
    J = np.zeros((0, 2, len(q))) if J is None else np.asarray(J, np.float64)[..., :len(q)]
    tf = np.isfinite(J).all((0, 1))
    return d, qf & tf, qf & ~tf


def sums(q, J, freqs, c=None):
    """dict: n, bad; S re, im (2, F) and dS re, im (P, 2, F) as long double
    arrays; phi = max |nu_j d_a| over the rays that enter (0 when none);
    absJ (P, 2, F) = sum 2 pi |nu_j J| over them (the unit of dS's bound)"""
    d, inn, bad = enter(q, J, c)
    nu = np.asarray(freqs, np.float64).reshape(-1)
    F = len(nu)
    J = np.zeros((0, 2, len(d))) if J is None else np.asarray(J, np.float64)[..., :len(d)]
    P = J.shape[0]
    Sre, Sim = np.zeros((2, F), LD), np.zeros((2, F), LD)
    dre, dim = np.zeros((P, 2, F), LD), np.zeros((P, 2, F), LD)
    absJ = np.zeros((P, 2, F))
    n = int(inn.sum())
    phi = 0.
    if n:
        dk, Jk = d[inn], J[:, :, inn]
        phi = float(np.abs(nu).max()*np.abs(dk).max())
        k = TWO_PI*nu.astype(LD)                                  # 2 pi nu, (F,)
        for a in range(2):
            ph = nu[:, None].astype(LD)*dk[None, :, a].astype(LD)  # (F, n)
            t = TWO_PI*(ph - np.rint(ph))
            cs, sn = np.cos(t), np.sin(t)
            Sre[a], Sim[a] = cs.sum(1), -sn.sum(1)
            for p in range(P):
                jv = Jk[p, a].astype(LD)[None, :]
                # -2 pi i nu J (cos - i sin) = -2 pi nu J sin - i 2 pi nu J cos
                dre[p, a] = -k*(jv*sn).sum(1)
                dim[p, a] = -k*(jv*cs).sum(1)
                absJ[p, a] = np.float64(2*np.pi)*np.abs(nu)*np.abs(Jk[p, a]).sum()
    return dict(n=n, bad=int(bad.sum()), Sre=Sre, Sim=Sim, dre=dre, dim=dim, phi=phi,
                absJ=absJ)


def oracle_error(n, phi):
    """a bound on the oracle's own error per component in units of n (for S)
    or of sum 2 pi |nu J| (for dS): the phase product and 2 pi's rounding,
    cosl / sinl, and the pairwise sum"""
    depth = np.ceil(np.log2(max(n, 2))) + 1
    return float(EPS_LD)*(8*phi + 8 + depth)


def device_bound(N, phi, chunks=1):
    """include/rtx.h's bound factors (S, dS) in units of n and of
    sum 2 pi |nu J|, for N rays in one call (plus chunks - 1 for calls added
    in order)"""
    slot = 4096                                     # RTX_OTF_JAC_SLOT
    D = slot//8 + 8 + -(-int(N)//slot) + chunks - 1
    eps = 2.**-52
    return (D + 4*phi + 3)*eps, (D + 4*phi + 5)*eps


def mtf_grad(S, dS, n):
    """the MTF |S|/n and its derivative Re(conj(S) dS)/(|S| n), NaN where
    |S| = 0; S (..., 2, F), dS (..., P, 2, F) complex"""
    a = np.abs(S)
    with np.errstate(invalid="ignore", divide="ignore"):
        g = (np.conj(S)[..., None, :, :]*dS).real/a[..., None, :, :]/n
        g = np.where(a[..., None, :, :] > 0, g, np.nan)
        return a/n, g
