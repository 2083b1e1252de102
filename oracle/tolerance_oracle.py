"""numpy restatement of rtx_trace_reduce_many and of the tolerance rms.

TEST INFRASTRUCTURE ONLY (like np_oracle.py and epi_oracle.py): the product
never imports it.  Each item's launch rays are traced with np_oracle through
the item's table and its 20 moments summed exactly (epi_oracle.exact_sum),
with the sums of the terms' magnitudes that scale the kernel's rounding
bound (ceil(N/512) + 64) eps sum|term|.
"""
import numpy as np

import epi_oracle
import np_oracle


def disc(n, seed):
    """uniform pupil coordinates in the unit disc"""
    rng = np.random.default_rng(seed)
    r = np.sqrt(rng.random(n))
    phi = 2*np.pi*rng.random(n)
    return np.c_[r*np.cos(phi), r*np.sin(phi)]


def item_sums(table, rot0, y0, u0, clip, center):
    """(sums, abs_sums) of one item's 20 moments (w = 1): the numpy trace of
    its launch rays y0, u0 through `table` and the exact sums of
    epi_oracle.reduce_terms at the last surface about `center` (4,) or None"""
    if len(y0) == 0:
        return np.zeros(epi_oracle.NMOM), np.zeros(epi_oracle.NMOM)
    Y, _, I, _ = np_oracle.trace(table, y0, u0, clip=clip, rot0=rot0)
    return epi_oracle.reduce_sums(Y[-1], I[-1], None, center)


def many_sums(tables, rot0, bundles, items, centers, clip):
    """item_sums of every item (table index, bundle index) of
    rtx_trace_reduce_many: (nitems, 20) sums and magnitudes; `bundles` a list
    of host (y0, u0)"""
    s, a = [], []
    for i, (t, b) in enumerate(np.asarray(items).reshape(-1, 2)):
        y0, u0 = bundles[b]
        si, ai = item_sums(tables[t], rot0, y0, u0, clip,
                           None if centers is None else centers[i])
        s.append(si)
        a.append(ai)
    return np.array(s).reshape(-1, epi_oracle.NMOM), np.array(a).reshape(-1, epi_oracle.NMOM)


def rms_finite(m):
    """rms about the mean of the rays with a finite image x, y (w = 1):
    sqrt((m3 - (m1^2 + m2^2)/m0)/m0); NaN without such a ray"""
    m = np.asarray(m, np.float64)
    if m[0] == 0:
        return float("nan")
    return float(np.sqrt(max((m[3] - (m[1]*m[1] + m[2]*m[2])/m[0])/m[0], 0.)))


def rms_finite_rows(y_last):
    """the same rms from a trace's last rows (N, 3): the spread of the rays
    with finite x and y about their mean"""
    y = np.asarray(y_last, np.float64)[:, :2]
    y = y[np.isfinite(y).all(1)]
    if not len(y):
        return float("nan")
    return float(np.sqrt(np.square(y - y.mean(0)).sum(1).mean()))
