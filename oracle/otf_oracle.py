"""Extended-precision statement of the geometric OTF sums (rtx_otf_rows,
include/rtx.h).

TEST INFRASTRUCTURE ONLY (like spot_oracle.py): the product never imports it.

The points are spot_oracle.points' (the kernel's FP64 expression).  Each
phase nu_j q (nu_j = arange(F)*dnu in float64) is formed in long double
(64-bit significand: the product of two doubles rounded once, relative error
2^-64), reduced mod 1 exactly, cos and sin of 2 pi frac are taken in long
double and the terms are summed pairwise (numpy's reduction of a contiguous
axis) in long double.  Per term the error is about 2 pi |nu q| 2^-64 + a few
2^-64; `oracle_error` bounds it with the summation.
"""
import numpy as np

import spot_oracle

LD = np.longdouble
assert np.finfo(LD).nmant + 1 >= 64, "the oracle needs a long double with a 64-bit significand"
TWO_PI = 8*np.arctan(LD(1))
EPS_LD = LD(2)**-63


def freqs(dnu, nfreq):
    """nu_j = j*dnu, one rounded float64 product each"""
    return np.arange(int(nfreq))*np.float64(dnu)


def otf(y, inc, c, z, dnu, nfreq, offsets=None, block=32):
    """(S complex (K, 2, F) as two long double arrays re, im; count (K,);
    phi (K,) = max |nu_j q| over the counted rays (0 when none))"""
    q = spot_oracle.points(y, inc, c, z, offsets)               # (K, N, 2) float64
    nu = freqs(dnu, nfreq)
    K, F = q.shape[0], len(nu)
    re, im = np.zeros((K, 2, F), LD), np.zeros((K, 2, F), LD)
    count, phi = np.zeros(K, np.int64), np.zeros(K)
    for k in range(K):
        fin = np.isfinite(q[k, :, 0]) & np.isfinite(q[k, :, 1])
        count[k] = np.count_nonzero(fin)
        if not count[k]:
            continue
        qk = q[k, fin]
        phi[k] = np.abs(nu).max()*np.abs(qk).max()
        for a in range(2):
            qa = qk[:, a].astype(LD)
            for j0 in range(0, F, block):
                ph = nu[j0:j0 + block, None].astype(LD)*qa[None, :]   # (B, n) contiguous rows
                ph = ph - np.rint(ph)
                t = TWO_PI*ph
                re[k, a, j0:j0 + block] = np.cos(t).sum(axis=1)
                im[k, a, j0:j0 + block] = -np.sin(t).sum(axis=1)
    return re, im, count, phi


def oracle_error(count, phi):
    """a bound on the oracle's own error per component, (K,): the phase
    product and 2 pi's rounding, cosl / sinl, and the pairwise sum"""
    n = np.asarray(count, np.float64)
    depth = np.ceil(np.log2(np.maximum(n, 2))) + 1
    return float(EPS_LD)*(8*np.asarray(phi) + 8 + depth)*n
