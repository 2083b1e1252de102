"""Extended-precision statement of rtx_trace_otf_many's sums (include/rtx.h)
from a ray's stored state at the last surface: y, i (N, 3) (a keep-LAST row
of rtx_trace for the item's table and bundle).

TEST INFRASTRUCTURE ONLY: the product never imports it.

q_k = d + z_k u with d = y_xy - c and u = i_xy / i_z is formed in float64
numpy, every operation rounded separately as the kernel does; a ray counts at
plane k iff both components of q_k are finite.  The sums of
exp(-2 pi i nu q_k[a]) are then otf_jac_oracle's (long double).
"""
import numpy as np

import otf_jac_oracle as oj


def points(y, inc, c, z):
    """(K, N, 2) float64 q_k of every ray"""
    y = np.asarray(y, np.float64)
    inc = np.asarray(inc, np.float64)
    c = np.zeros(2) if c is None else np.asarray(c, np.float64).reshape(2)
    with np.errstate(all="ignore"):
        d = y[:, :2] - c
        u = inc[:, :2]/inc[:, 2:3]
        return np.stack([d + zk*u for zk in np.asarray(z, np.float64)])


def sums(y, inc, c, z, freqs):
    """(S re, S im) long double (K, 2, F), count (K,) int64, phi (K,) =
    max |nu_j q_k[a]| over the counted rays"""
    q = points(y, inc, c, z)
    K, F = len(q), len(np.atleast_1d(freqs))
    re = np.zeros((K, 2, F), oj.LD)
    im = np.zeros((K, 2, F), oj.LD)
    count = np.zeros(K, np.int64)
    phi = np.zeros(K)
    for k in range(K):
        r = oj.sums(q[k], None, freqs)
        re[k], im[k], count[k], phi[k] = r["Sre"], r["Sim"], r["n"], r["phi"]
    return re, im, count, phi


def device_bound(N, phi):
    """include/rtx.h's bound factor per component, in units of count[k]"""
    return (20 + -(-int(N)//512) + 4*np.asarray(phi) + 3)*2.**-52


def oracle_error(count, phi):
    """otf_jac_oracle's bound on the oracle's own error per plane, in units
    of count[k]"""
    return np.array([oj.oracle_error(n, p) for n, p in
                     zip(np.atleast_1d(count), np.atleast_1d(phi))])
