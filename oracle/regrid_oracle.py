"""numpy restatement of the device regridding (rtx_grid_linear,
rayopt_b200/csrc/rtx_psf.cuh) and an exact rational checker of it.

* ``restate``: the claim and evaluation passes written out in numpy.  Every
  simplex with a usable transform visits the grid nodes of its bounding box
  (with a margin of nodes beyond it), computes the barycentric coordinates
  from the given transform with numpy's separately rounded operations in the
  kernel's order (c0, c1 accumulated from 0, c2 = (1 - c0) - c1) and claims
  the node when every c_k is in [-100 eps, 1 + 100 eps]; a node's winner is
  the lowest claiming index, its value ((0 + c0 v0) + c1 v1) + c2 v2 on the
  winner.  No scipy walk is involved, so this is the kernel's rule on its own
  terms and gives the device's bits.  ``reach`` reports how far beyond its box
  a claimed node lies (the kernel looks one node beyond).
* exact checks with ``fractions.Fraction``, meant for the few nodes near an
  edge: the barycentric coordinates of a node in a triangle, whether a node
  lies in the convex hull (the hull itself built with exact orientations), and
  the exact linear interpolant.
* ``delaunay_transform``: the explicit 2x2 inverse rtx_delaunay writes, in
  numpy, and the condition number of its determinant.
"""
from fractions import Fraction

import numpy as np

EPS = np.finfo(np.float64).eps
GRID_EPS = 100*EPS               # scipy's inside tolerance (rtx_psf.cuh)
GRID_WARP_NODES = 64             # boxes of more nodes go to the warp path


# ---- the restatement ---------------------------------------------------------
def barycentric(tr, x, y):
    """rtx_psf.cuh barycentric(): tr (..., 6) = {T00, T01, T10, T11, r0, r1}"""
    dx = x - tr[..., 4]
    dy = y - tr[..., 5]
    c0 = (0. + tr[..., 0]*dx) + tr[..., 1]*dy
    c1 = (0. + tr[..., 2]*dx) + tr[..., 3]*dy
    c2 = (1. - c0) - c1
    return c0, c1, c2


def inside(c):
    return (c >= -GRID_EPS) & (c <= 1. + GRID_EPS)


def node_boxes(pts, simplices, transform, gh, margin):
    """per simplex the node index ranges [i0, i1] x [j0, j1] of its bounding
    box widened by `margin` nodes on each side (clamped), the unwidened box
    (b0, b1) per axis, and whether the simplex can claim at all (a finite
    transform[0, 0] and vertex indices in range, as the kernel checks)"""
    pts = np.asarray(pts, np.float64)
    simplices = np.asarray(simplices, np.int64).reshape(-1, 3)
    tr = np.asarray(transform, np.float64).reshape(-1, 6)
    n = len(gh)
    s = -1. if gh[-1] < gh[0] else 1.
    key = s*np.asarray(gh, np.float64)
    ok = (tr[:, 0] == tr[:, 0]) & ((simplices >= 0) & (simplices < len(pts))).all(1)
    v = pts[np.where(ok[:, None], simplices, 0)]          # (T, 3, 2)
    out = []
    for ax in range(2):
        lo, hi = v[..., ax].min(1), v[..., ax].max(1)
        a, b = (lo, hi) if s > 0 else (-hi, -lo)
        first = np.searchsorted(key, a, "left")            # first node >= a
        last = np.searchsorted(key, b, "right") - 1        # last node <= b
        out.append((np.clip(first - margin, 0, n - 1), np.clip(last + margin, 0, n - 1),
                    first, last))
    return ok, out


def restate(pts, vals, simplices, transform, gh, margin=3, chunk=1 << 22):
    """the device's regridding on the grid node (i, j) = (gh[i], gh[j]).
    Returns dict(winner (n, n) int64, -1 where none claims; value (n, n);
    reach: the most nodes beyond its box at which a simplex claimed a node;
    box_nodes (T,): the nodes the kernel visits per simplex, its box plus one
    node each side, 0 for a simplex that cannot claim)"""
    gh = np.asarray(gh, np.float64)
    vals = np.asarray(vals, np.float64)
    simplices = np.asarray(simplices, np.int64).reshape(-1, 3)
    tr = np.asarray(transform, np.float64).reshape(-1, 6)
    n, T = len(gh), len(simplices)
    ok, ((i0, i1, fi, li), (j0, j1, fj, lj)) = node_boxes(pts, simplices, tr, gh, margin)
    wi, wj = np.where(ok, i1 - i0 + 1, 0), np.where(ok, j1 - j0 + 1, 0)
    cnt = wi*wj
    win = np.full(n*n, T, np.int64)
    reach = 0
    start = 0
    csum = np.cumsum(cnt)
    while start < T:
        stop = max(int(np.searchsorted(csum, (csum[start - 1] if start else 0) + chunk, "right")),
                   start + 1)
        stop = min(stop, T)
        sid = np.arange(start, stop)
        c = cnt[sid]
        s = np.repeat(sid, c)
        k = np.arange(len(s)) - np.repeat(np.cumsum(c) - c, c)
        i = i0[s] + k//wj[s]
        j = j0[s] + k % wj[s]
        c0, c1, c2 = barycentric(tr[s], gh[i], gh[j])
        hit = inside(c0) & inside(c1) & inside(c2)
        if hit.any():
            s, i, j = s[hit], i[hit], j[hit]
            np.minimum.at(win, i*n + j, s)
            out = np.maximum.reduce([fi[s] - i, i - li[s], fj[s] - j, j - lj[s],
                                     np.zeros_like(i)])
            reach = max(reach, int(out.max()))
        start = stop
    win[win == T] = -1
    value = np.full(n*n, np.nan)
    k = np.flatnonzero(win >= 0)
    w = win[k]
    c0, c1, c2 = barycentric(tr[w], gh[k//n], gh[k % n])
    sv = vals[simplices[w]]
    value[k] = ((0. + c0*sv[:, 0]) + c1*sv[:, 1]) + c2*sv[:, 2]
    _, ((b0, b1, _, _), (c0_, c1_, _, _)) = node_boxes(pts, simplices, tr, gh, 1)
    box = np.where(ok, (b1 - b0 + 1)*(c1_ - c0_ + 1), 0)
    return dict(winner=win.reshape(n, n), value=value.reshape(n, n), reach=reach, box_nodes=box)


# ---- exact checks ------------------------------------------------------------
def _F(p):
    return (Fraction(float(p[0])), Fraction(float(p[1])))


def orient(a, b, c):
    """exact sign of the orientation of the points a, b, c (Fractions)"""
    d = (a[0] - c[0])*(b[1] - c[1]) - (a[1] - c[1])*(b[0] - c[0])
    return (d > 0) - (d < 0)


def exact_barycentric(tri_pts, node):
    """exact barycentric coordinates (c0, c1, c2) of `node` in the triangle
    with vertices tri_pts (3, 2) (r = the last vertex, as in the transform);
    None for a zero-area triangle"""
    a, b, r = (_F(p) for p in tri_pts)
    x, y = _F(node)
    t00, t01, t10, t11 = a[0] - r[0], b[0] - r[0], a[1] - r[1], b[1] - r[1]
    det = t00*t11 - t01*t10
    if det == 0:
        return None
    dx, dy = x - r[0], y - r[1]
    c0 = (t11*dx - t01*dy)/det
    c1 = (t00*dy - t10*dx)/det
    return c0, c1, 1 - c0 - c1


def exact_hull(pts):
    """the convex hull of `pts` as a counter-clockwise list of exact vertices
    (collinear points dropped), by the monotone chain with exact orientations
    on the points that can be hull vertices: qhull's hull vertices and every
    point within rounding of qhull's hull"""
    from scipy.spatial import ConvexHull
    pts = np.asarray(pts, np.float64)
    h = ConvexHull(pts)
    a, b = pts[h.simplices[:, 0]], pts[h.simplices[:, 1]]
    scale = np.fabs(pts).max()
    near = np.zeros(len(pts), bool)
    near[h.vertices] = True
    for lo in range(0, len(pts), 4096):
        p = pts[lo:lo + 4096, None, :]
        ab = b - a
        s = np.clip(((p - a)*ab).sum(-1)/(ab*ab).sum(-1), 0, 1)
        d = np.sqrt(np.square(a + s[..., None]*ab - p).sum(-1)).min(1)
        near[lo:lo + 4096] |= d <= 1e-9*scale
    cand = sorted({(float(x), float(y)) for x, y in pts[near]})
    P = [_F(p) for p in cand]

    def chain(seq):
        out = []
        for p in seq:
            while len(out) >= 2 and orient(out[-2], out[-1], p) <= 0:
                out.pop()
            out.append(p)
        return out
    lower, upper = chain(P), chain(P[::-1])
    return lower[:-1] + upper[:-1]


def in_hull_exact(hull, node):
    """+1 strictly inside the exact hull, 0 on its boundary, -1 outside"""
    p = _F(node)
    s = [orient(hull[k], hull[(k + 1) % len(hull)], p) for k in range(len(hull))]
    if min(s) < 0:
        return -1
    return 0 if min(s) == 0 else 1


def hull_depth(hull, xs, ys, chunk=1 << 20):
    """float signed distance of the nodes (xs, ys) to the exact hull's edge
    lines, the least over the edges: the distance to the boundary for a node
    inside (> 0), and a lower bound of minus the distance to the hull for a
    node outside"""
    H = np.array([[float(x), float(y)] for x, y in hull])
    a, b = H, np.roll(H, -1, axis=0)
    ab = b - a
    L = np.hypot(ab[:, 0], ab[:, 1])
    x, y = np.ravel(xs), np.ravel(ys)
    out = np.empty(x.shape)
    step = max(1, chunk//len(H))
    for lo in range(0, len(x), step):
        px, py = x[lo:lo + step, None], y[lo:lo + step, None]
        d = (ab[:, 0]*(py - a[:, 1]) - ab[:, 1]*(px - a[:, 0]))/L
        out[lo:lo + len(d)] = d.min(1)
    return out.reshape(np.shape(xs))


def hull_distance(hull, xs, ys):
    """float distance of the nodes to the exact hull's boundary segments"""
    H = np.array([[float(x), float(y)] for x, y in hull])
    a, b = H, np.roll(H, -1, axis=0)
    p = np.stack([np.ravel(xs), np.ravel(ys)], -1)[:, None, :]
    ab = b - a
    s = np.clip(((p - a)*ab).sum(-1)/(ab*ab).sum(-1), 0, 1)
    return np.sqrt(np.square(a + s[..., None]*ab - p).sum(-1)).min(1)


def node_condition(tr, rho, xs, ys):
    """per node the error scale of its barycentric coordinates on the simplex
    with transform row tr (..., 6) and determinant condition rho:
    (rho + 2) (1 + max_k (|Tinv| |p - r|)_k)"""
    dx, dy = np.fabs(xs - tr[..., 4]), np.fabs(ys - tr[..., 5])
    q = np.maximum(np.fabs(tr[..., 0])*dx + np.fabs(tr[..., 1])*dy,
                   np.fabs(tr[..., 2])*dx + np.fabs(tr[..., 3])*dy)
    return (rho + 2.)*(1. + q)


def exact_check(pts, vals, simplices, transform, gh, winner, value, sample=2500, seed=0):
    """the regridding (winner, value) against exact arithmetic.  Returns
    dict(depth: hull_depth of every node, tol: 1e3 eps h, h; bary_low: the
    least exact barycentric coordinate of a node in its winner, over the
    nodes nearest an edge, and bary_excess: how far it falls below -100 eps
    in units of eps times the node's condition; value_ratio: the largest
    |value - exact interpolant| / (eps cond sum |v_k|) over the sampled
    nodes; checked: how many nodes were checked exactly)"""
    pts = np.asarray(pts, np.float64)
    vals = np.asarray(vals, np.float64)
    simplices = np.asarray(simplices, np.int64).reshape(-1, 3)
    tr = np.asarray(transform, np.float64).reshape(-1, 6)
    n = len(gh)
    h = float(np.fabs(pts).max())
    hull = exact_hull(pts)
    X, Y = np.meshgrid(gh, gh, indexing="ij")
    depth = hull_depth(hull, X, Y)
    res = dict(depth=depth, tol=1e3*EPS*h, h=h, hull=hull, bary_low=0., bary_excess=0.,
               value_ratio=0., checked=0)
    k = np.flatnonzero(winner.ravel() >= 0)
    if not len(k):
        return res
    w = winner.ravel()[k]
    c = np.stack(barycentric(tr[w], gh[k//n], gh[k % n]), -1)
    rng = np.random.default_rng(seed)
    near = k[np.argsort(np.fabs(c).min(1), kind="stable")[:sample]]   # nearest an edge
    pick = np.unique(np.concatenate([near, rng.choice(k, min(sample//4, len(k)), replace=False)]))
    _, rho = delaunay_transform(pts, simplices[winner.ravel()[pick]])
    cond = node_condition(tr[winner.ravel()[pick]], rho, gh[pick//n], gh[pick % n])
    low = excess = ratio = 0.
    for node, cd in zip(pick.tolist(), cond.tolist()):
        s = simplices[winner.ravel()[node]]
        p = (gh[node//n], gh[node % n])
        cx = exact_barycentric(pts[s], p)
        m = float(min(cx))
        low = min(low, m)
        excess = max(excess, (-m - GRID_EPS)/(EPS*cd))
        ex = sum(ck*Fraction(float(v)) for ck, v in zip(cx, vals[s]))
        err = abs(Fraction(float(value.ravel()[node])) - ex)
        ratio = max(ratio, float(err)/(EPS*cd*max(float(np.fabs(vals[s]).sum()), 1e-300)))
    res.update(bary_low=low, bary_excess=excess, value_ratio=ratio, checked=len(pick))
    return res


# ---- the device triangulation's transform -----------------------------------
def delaunay_transform(pts, simplices):
    """rtx_delaunay's transform (T, 3, 2) of the triangles `simplices`:
    T = [v0 - r, v1 - r] as columns, r = v2, Tinv by the explicit formula
    (adj T)/det with separately rounded operations, NaN rows for det == 0;
    and rho = (|t00 t11| + |t01 t10|)/|det|, the condition number of the
    determinant (inf for det == 0)"""
    p = np.asarray(pts, np.float64)[np.asarray(simplices, np.int64)]
    a, b, r = p[:, 0], p[:, 1], p[:, 2]
    t00, t01 = a[:, 0] - r[:, 0], b[:, 0] - r[:, 0]
    t10, t11 = a[:, 1] - r[:, 1], b[:, 1] - r[:, 1]
    with np.errstate(divide="ignore", invalid="ignore"):
        det = t00*t11 - t01*t10
        tr = np.stack([t11/det, -t01/det, -t10/det, t00/det, r[:, 0], r[:, 1]], -1)
        rho = (np.fabs(t00*t11) + np.fabs(t01*t10))/np.fabs(det)
    tr[det == 0] = np.nan
    return tr.reshape(-1, 3, 2), rho


def exact_inverse(pts, simplex):
    """the exact inverse of T = [v0 - r, v1 - r] (Fractions, row major)"""
    a, b, r = (_F(pts[k]) for k in simplex)
    t00, t01, t10, t11 = a[0] - r[0], b[0] - r[0], a[1] - r[1], b[1] - r[1]
    det = t00*t11 - t01*t10
    return t11/det, -t01/det, -t10/det, t00/det
