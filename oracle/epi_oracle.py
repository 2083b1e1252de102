"""numpy restatement of the fused trace epilogues and the moment reductions.

TEST INFRASTRUCTURE ONLY (like np_oracle.py): the product never imports it.

It restates the contracts of include/rtx.h for the numbers users read off a
trace, given the rows a trace stores:

* `reduce_terms`  the per-ray terms of the 20 moments of rtx_trace_reduce, of
  the 8 of rtx_moments and of the 8 of rtx_focus_moments;
* `exact_sum`     their sums, exact to far below the kernels' rounding, and
  the sums of |term| that set the kernels' error bounds;
* `opd_epilogue`  A and P of rtx_trace_opd in the DEVICE's operation order
  (rtx_device.cuh, epi_kernel's EPI_OPD branch): every product and sum rounded
  on its own, so that the kernel's output can be compared bit for bit;
* `opd_reference_order`  the same quantity in the reference's order
  (rayopt/geometric_trace.py:101-131), which pins the restatement to the
  reference (tests/test_epi_oracle.py).

Everything is evaluated in float64, also for float32 rows: the kernels widen
each float32 value to double before they use it, and round the OPD outputs
back to float32 at the end.
"""
import math

import numpy as np

NMOM = 20

# above this many rays exact_sum switches from math.fsum to a chunked
# extended-precision pairwise sum
FSUM_MAX = 200000
CHUNK = 1 << 20


def _tanarcsin(inc):
    """rayopt/utils.py:42-48, as the kernels evaluate it: i_xy / i_z in double"""
    i = np.asarray(inc, np.float64)
    with np.errstate(all="ignore"):
        return i[:, :2]/i[:, 2:3]


def reduce_terms(y, inc, w=None, center=None, magnitude=False):
    """(N, 20) per-ray terms of rtx_trace_reduce's moments of one surface:
    intercepts y (N,3), incidence directions inc (N,3), weights w (N,) or None
    (= 1), centre (y_x, y_y, u_x, u_y) or None (= 0).  Gating as in the
    header: m[0..7] over the rays with finite dx and dy (m[5] counts every
    ray), m[8..19] over the rays with a finite slope.  Rays outside a gate
    contribute 0.  `magnitude`: the scale each term's own rounding is relative
    to instead -- |term|, and w (|dx ux| + |dy uy|) for the dot product of
    m[18], whose parts may cancel."""
    y = np.asarray(y, np.float64)
    N = y.shape[0]
    c = np.zeros(4) if center is None else np.asarray(center, np.float64).reshape(4)
    ww = np.ones(N) if w is None else np.asarray(w, np.float64)
    out = np.zeros((N, NMOM))
    with np.errstate(all="ignore"):
        dx, dy = y[:, 0] - c[0], y[:, 1] - c[1]
        s = _tanarcsin(inc)
        ux, uy = s[:, 0] - c[2], s[:, 1] - c[3]
        f = np.isfinite(dx) & np.isfinite(dy)
        g = np.isfinite(ux) & np.isfinite(uy)
        out[:, 5] = 1.0
        for k, v in ((0, ww), (1, ww*dx), (2, ww*dy), (3, ww*(dx*dx + dy*dy)), (4, 1.0),
                     (6, dx), (7, dy)):
            out[f, k] = np.broadcast_to(v, (N,))[f]
        dot = np.abs(dx*ux) + np.abs(dy*uy) if magnitude else dx*ux + dy*uy
        for k, v in ((8, 1.0), (9, dx), (10, dy), (11, ux), (12, uy), (13, ww), (14, ww*dx),
                     (15, ww*dy), (16, ww*ux), (17, ww*uy), (18, ww*dot),
                     (19, ww*(ux*ux + uy*uy))):
            out[g, k] = np.broadcast_to(v, (N,))[g]
    return np.abs(out) if magnitude else out


def moments_terms(y, w=None, center=None):
    """(N, 8) per-ray terms of rtx_moments: m[0..7] of rtx_trace_reduce
    without the slope moments (center = (y_x, y_y) or None)"""
    c = None if center is None else np.r_[np.asarray(center, np.float64).reshape(2), 0., 0.]
    y = np.asarray(y, np.float64)
    return reduce_terms(y, np.zeros_like(y), w, c)[:, :8]


def focus_terms(y, inc, w=None, center=None):
    """(N, 8) per-ray terms of rtx_focus_moments about (y_x, y_y, u_x, u_y):
    #good, #total, sum dy (2), sum du (2), sum w dy.du, sum w du.du over the
    rays with a finite slope"""
    t = reduce_terms(y, inc, w, center)
    out = np.empty((t.shape[0], 8))
    out[:, 0] = t[:, 8]
    out[:, 1] = t[:, 5]
    out[:, 2:6] = t[:, 9:13]
    out[:, 6:8] = t[:, 18:20]
    return out


def exact_sum(terms):
    """(sums, abs_sums) of the columns of `terms` (N, k).

    Up to FSUM_MAX rows: math.fsum, the correctly rounded sum.  Above: numpy's
    pairwise sum in np.longdouble (x87 extended, 64-bit significand) of each
    column over chunks of CHUNK rows (each chunk transposed, so that the sum
    runs along a contiguous axis, where numpy sums pairwise), the chunk sums
    added in longdouble too.  Its error is below (log2(CHUNK) + N/CHUNK)
    2**-64 sum|term|, about 1e-18 sum|term| at 2e7 rays, five orders below the
    kernels' bound.  NaN or infinite terms propagate (the kernels add them
    too)."""
    terms = np.asarray(terms, np.float64)
    if terms.ndim == 1:
        terms = terms[:, None]
    N, k = terms.shape
    if N <= FSUM_MAX:
        s = np.array([math.fsum(terms[:, j]) if np.isfinite(terms[:, j]).all()
                      else terms[:, j].sum() for j in range(k)])
        a = np.array([math.fsum(np.abs(terms[:, j])) if np.isfinite(terms[:, j]).all()
                      else np.abs(terms[:, j]).sum() for j in range(k)])
        return s, a
    if np.finfo(np.longdouble).nmant < 63:
        raise RuntimeError("exact_sum needs an extended-precision np.longdouble for N > %d"
                           % FSUM_MAX)
    s = np.zeros(k, np.longdouble)
    a = np.zeros(k, np.longdouble)
    for i in range(0, N, CHUNK):
        s_, a_ = _pairwise(terms[i:i + CHUNK])
        s += s_
        a += a_
    return s.astype(np.float64), a.astype(np.float64)


def _pairwise(terms):
    """longdouble column sums of terms (n, k) and of |terms|, summed along a
    contiguous axis (numpy's pairwise summation)"""
    blk = np.ascontiguousarray(np.asarray(terms).T, np.longdouble)
    return blk.sum(1), np.abs(blk).sum(1)


def reduce_sums(y, inc, w=None, center=None, chunk=CHUNK):
    """the 20 moments of rtx_trace_reduce, exact (exact_sum), and the sums of
    the terms' magnitudes (reduce_terms(magnitude=True)) that scale the
    kernels' rounding; chunked, so that 2e7-ray bundles never hold N x 20
    terms at once"""
    N = np.asarray(y).shape[0]
    if N <= FSUM_MAX:
        return (exact_sum(reduce_terms(y, inc, w, center))[0],
                exact_sum(reduce_terms(y, inc, w, center, magnitude=True))[0])
    s = np.zeros(NMOM, np.longdouble)
    a = np.zeros(NMOM, np.longdouble)
    for i in range(0, N, chunk):
        args = (y[i:i + chunk], inc[i:i + chunk], None if w is None else w[i:i + chunk], center)
        s += _pairwise(reduce_terms(*args))[0]
        a += _pairwise(reduce_terms(*args, magnitude=True))[0]
    return s.astype(np.float64), a.astype(np.float64)


def opd_epilogue(y0, y_after, u_after, path_sum, spec):
    """A (N,) and P (N,3) of rtx_trace_opd in the device's operation order.

    y0: the launch rays (row 0 of the trace, before any rot0), y_after /
    u_after: the stored rows of surface `after` (its normal frame), path_sum:
    the per-ray sum of t over the marched surfaces in the trace dtype (what
    rtx_set_path_sum_output writes), spec: the members of `struct rtx_opd`.
    Each numpy operation below is one IEEE double operation, in the order the
    kernel writes them; the results are rounded to the dtype of y_after."""
    dt = np.asarray(y_after).dtype
    f = lambda a: np.asarray(a, np.float64)         # noqa: E731
    y0, y, u, A = f(y0), f(y_after), f(u_after), f(path_sum).copy()
    y0r, u0r = f(spec["y0_ref"]).reshape(3), f(spec["u0_ref"]).reshape(3)
    M, d = f(spec["M"]).reshape(9), f(spec["d"]).reshape(3)
    n0, n_after, radius = float(spec["n0"]), float(spec["n_after"]), float(spec["radius"])
    with np.errstate(all="ignore"):
        if spec["infinite"]:
            tj = (u0r[0]*(y0r[0] - y0[:, 0]) + u0r[1]*(y0r[1] - y0[:, 1])) \
                + u0r[2]*(y0r[2] - y0[:, 2])
            A = A - tj*n0
        q = [((y[:, 0]*M[k] + y[:, 1]*M[3 + k]) + y[:, 2]*M[6 + k]) + d[k] for k in range(3)]
        v = [(u[:, 0]*M[k] + u[:, 1]*M[3 + k]) + u[:, 2]*M[6 + k] for k in range(3)]
        q[2] = q[2] + radius
        c = 1.0/radius
        uyv = (v[0]*q[0] + v[1]*q[1]) + v[2]*q[2]
        yyv = (q[0]*q[0] + q[1]*q[1]) + q[2]*q[2]
        dd = c*uyv - v[2]
        ff = c*yyv - 2.0*q[2]
        gg = np.sqrt(dd*dd - c*ff)
        ti = -(dd + gg)/c
        A = A + ti*n_after
        P = np.stack([q[0] + ti*v[0], q[1] + ti*v[1], (q[2] + ti*v[2]) - radius], axis=-1)
    return A.astype(dt), P.astype(dt)


def opd_reference_order(T, ref, y0, u0, n0, n_after, y_after, u_after, Ra, Ri,
                        o_after, o_image, y_image_ref, radius, infinite, wavelength_scaled):
    """GeometricTrace.opd(resample=False) (rayopt/geometric_trace.py:101-131)
    restated expression by expression on the reference's stored rows:
    T the rows 0..after of t, y0 / u0 row 0, Ra / Ri the rot_normal of
    surfaces `after` / `image` (None = not rotated), o_* their origins,
    y_image_ref = y[image, ref], wavelength_scaled = l/scale.  Returns
    (x, y, t) exactly as the reference does."""
    with np.errstate(all="ignore"):
        t = (T - T[:, (ref,)]).sum(0)                               # :102
        if infinite:                                                # :103-109
            tj = np.dot(u0[ref], (y0[ref] - y0).T)
            t -= tj*n0
        y = y_after if Ra is None else np.dot(y_after, Ra)          # :116
        y = y + (o_after - o_image)                                 # :117
        y = (y if Ri is None else np.dot(y, Ri.T)) - y_image_ref    # :118
        u = u_after if Ra is None else np.dot(u_after, Ra)          # :119
        u = u if Ri is None else np.dot(u, Ri.T)
        y[:, 2] += radius                                           # :123
        ti = sphere_intercept(1./radius, y, u)                      # :124
        t += (ti - ti[ref])*n_after                                 # :125
        t = -t/wavelength_scaled                                    # :126
        py = y + ti[:, None]*u                                      # :129
        py[:, 2] -= radius
        py -= py[ref]
        x, y, z = py.T
    return x, y, t


def sphere_intercept(c, y, u):
    """Spheroid(curvature=c).intercept for the conic k = 0
    (rayopt/elements.py:477-501): the exit reference sphere of opd"""
    uy = (u*y).sum(1)
    uu = 1.
    yy = np.square(y).sum(1)
    d = c*uy - u[:, 2]
    e = c*uu
    f = c*yy - 2*y[:, 2]
    g = np.sqrt(np.square(d) - e*f)
    return -(d + g)/e
