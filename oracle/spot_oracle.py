"""numpy statement of the through-focus spot images (rtx_trace_spot,
rtx_spot_rows; include/rtx.h).

TEST INFRASTRUCTURE ONLY (like epi_oracle.py): the product never imports it.

* `points`     Analysis.spots' points (rayopt/analysis.py:266-280) from stored
               rows: ``(y_xy - c + z_k tanarcsin(i)) - o_k`` in float64, each
               operation rounded on its own as numpy evaluates it;
* `bin_index`  the binning rule: edges ``np.linspace(lo, hi, n + 1)``, bin
               ``searchsorted(edges, x, "right") - 1`` with ``x == hi`` in the
               last bin, -1 outside ``[lo, hi]`` and for NaN / inf -- what
               np.histogram2d and np.histogram do (tests/test_spot_oracle.py
               pins it to them);
* `spot`       counts, tallies (binned, non-finite) and extents (max |q_x|,
               max |q_y|, max r over the finite points) of a bundle.
"""
import numpy as np


def points(y, inc, c, z, offsets=None):
    """(K, N, 2) float64 points of the rows y, inc (N, 3) about the centre c
    at the defocus distances z (K,), minus the per-plane offsets (K, 2)"""
    y = np.asarray(y, np.float64)
    inc = np.asarray(inc, np.float64)
    z = np.atleast_1d(np.asarray(z, np.float64))
    o = np.zeros((len(z), 2)) if offsets is None else np.asarray(offsets, np.float64)
    with np.errstate(all="ignore"):
        d = y[:, :2] - np.asarray(c, np.float64)[:2]
        u = inc[:, :2]/inc[:, 2:]                           # tanarcsin, utils.py:42-48
        return np.stack([(d + zk*u) - ok for zk, ok in zip(z, o)])


def edges(lo, hi, n):
    return np.linspace(lo, hi, n + 1)


def bin_index(x, lo, hi, n):
    """the bin of each x (-1: not counted)"""
    x = np.asarray(x, np.float64)
    e = edges(lo, hi, n)
    j = np.searchsorted(e, x, side="right") - 1
    j[x == hi] = n - 1
    ok = (x >= lo) & (x <= hi)                              # False for NaN
    return np.where(ok, j, -1)


def histogram(qx, qy, bins, range):
    """np.histogram2d(qx, qy, bins, range) by the rule above, uint64"""
    (nx, ny), ((xl, xh), (yl, yh)) = bins, range
    jx, jy = bin_index(qx, xl, xh, nx), bin_index(qy, yl, yh, ny)
    ok = (jx >= 0) & (jy >= 0)
    return np.bincount(jx[ok]*ny + jy[ok], minlength=nx*ny).reshape(nx, ny).astype(np.uint64)


def histogram1d(r, n, range):
    """np.histogram(r, n, range) by the rule above, uint64"""
    j = bin_index(r, range[0], range[1], n)
    return np.bincount(j[j >= 0], minlength=n).astype(np.uint64)


def radii(q):
    with np.errstate(all="ignore"):
        return np.sqrt(q[..., 0]*q[..., 0] + q[..., 1]*q[..., 1])


def spot(y, inc, c, z, bins, range, radial=False, offsets=None):
    """(counts (K, nx, ny) or (K, nx) uint64, tally (K, 2) uint64, extent
    (K, 3) float64) of rows y, inc; `range` ((x_lo, x_hi), (y_lo, y_hi)), or
    ((r_lo, r_hi),) when radial"""
    q = points(y, inc, c, z, offsets)
    K = q.shape[0]
    r = radii(q)
    counts, tally, extent = [], np.zeros((K, 2), np.uint64), np.zeros((K, 3))
    for k in np.arange(K):
        fin = np.isfinite(q[k, :, 0]) & np.isfinite(q[k, :, 1])
        if radial:
            h = histogram1d(r[k], bins[0], range[0])
        else:
            h = histogram(q[k, :, 0], q[k, :, 1], bins, range)
        counts.append(h)
        tally[k] = h.sum(dtype=np.uint64), np.count_nonzero(~fin)
        if fin.any():
            extent[k] = (np.abs(q[k, fin, 0]).max(), np.abs(q[k, fin, 1]).max(), r[k, fin].max())
    return np.stack(counts), tally, extent
