"""Exact checks of a 2-d Delaunay triangulation (CPU).

This does not restate the device algorithm (rtx_delaunay); it checks any
triangulation of a point set -- scipy's or the device's -- exactly: the
predicates are evaluated in floating point with Shewchuk's static error
bounds and, where the bound does not decide the sign, in exact rational
arithmetic (fractions.Fraction).

``check`` asserts that the simplices have non-zero area (and, with ``ccw``,
are counter-clockwise), that every edge is shared by at most two simplices and
``neighbors`` agrees, that the boundary is exactly the convex hull with its
collinear points, that every distinct point is a vertex, that T = 2V - h - 2
and that every interior edge is locally Delaunay (incircle <= 0), which for a
valid triangulation is global Delaunay.  ``cocircular_differences`` explains
where two Delaunay triangulations of one point set differ."""
from fractions import Fraction

import numpy as np

EPS = 2.0**-53
CCW_BOUND = (3 + 16*EPS)*EPS
ICC_BOUND = (10 + 96*EPS)*EPS


def _orient_exact(a, b, c):
    ax, ay, bx, by, cx, cy = (Fraction(float(v)) for v in (*a, *b, *c))
    d = (ax - cx)*(by - cy) - (ay - cy)*(bx - cx)
    return (d > 0) - (d < 0)


def _incircle_exact(a, b, c, d):
    dx, dy = Fraction(float(d[0])), Fraction(float(d[1]))
    m = [(Fraction(float(p[0])) - dx, Fraction(float(p[1])) - dy) for p in (a, b, c)]
    lift = [x*x + y*y for x, y in m]
    v = (lift[0]*(m[1][0]*m[2][1] - m[2][0]*m[1][1]) + lift[1]*(m[2][0]*m[0][1] - m[0][0]*m[2][1])
         + lift[2]*(m[0][0]*m[1][1] - m[1][0]*m[0][1]))
    return (v > 0) - (v < 0)


def orient(a, b, c):
    """sign of orient2d for arrays of points (n, 2): > 0 counter-clockwise"""
    a, b, c = (np.atleast_2d(np.asarray(p, np.float64)) for p in (a, b, c))
    with np.errstate(all="ignore"):
        left = (a[:, 0] - c[:, 0])*(b[:, 1] - c[:, 1])
        right = (a[:, 1] - c[:, 1])*(b[:, 0] - c[:, 0])
        det = left - right
        bound = CCW_BOUND*(np.abs(left) + np.abs(right)) + 2.0**-1000
    s = np.sign(det).astype(np.int64)
    s[~(np.abs(det) > bound)] = 0
    for k in np.flatnonzero(~(np.abs(det) > bound)):
        s[k] = _orient_exact(a[k], b[k], c[k])
    return s


def incircle(a, b, c, d):
    """sign of incircle for arrays of points: > 0 when d lies strictly inside
    the circle through the counter-clockwise a, b, c"""
    a, b, c, d = (np.atleast_2d(np.asarray(p, np.float64)) for p in (a, b, c, d))
    with np.errstate(all="ignore"):
        ad, bd, cd = a - d, b - d, c - d
        bc, cb = bd[:, 0]*cd[:, 1], cd[:, 0]*bd[:, 1]
        ca, ac = cd[:, 0]*ad[:, 1], ad[:, 0]*cd[:, 1]
        ab, ba = ad[:, 0]*bd[:, 1], bd[:, 0]*ad[:, 1]
        la, lb, lc = (p[:, 0]*p[:, 0] + p[:, 1]*p[:, 1] for p in (ad, bd, cd))
        det = la*(bc - cb) + lb*(ca - ac) + lc*(ab - ba)
        perm = (np.abs(bc) + np.abs(cb))*la + (np.abs(ca) + np.abs(ac))*lb + (np.abs(ab) + np.abs(ba))*lc
        bound = ICC_BOUND*perm + 2.0**-1000
    s = np.sign(det).astype(np.int64)
    unsure = ~(np.abs(det) > bound)
    s[unsure] = 0
    for k in np.flatnonzero(unsure):
        s[k] = _incircle_exact(a[k], b[k], c[k], d[k])
    return s


def hull_edges(points):
    """directed counter-clockwise boundary edges (i, j) of the convex hull,
    collinear boundary points included (monotone chain, exact orient);
    duplicates are represented by their lowest index"""
    p = np.asarray(points, np.float64) + 0.0            # -0.0 -> 0.0
    _, first = np.unique(p, axis=0, return_index=True)
    idx = first[np.lexsort((p[first, 1], p[first, 0]))]

    def chain(order):
        h = []
        for i in order:
            while len(h) >= 2 and orient(p[h[-2]], p[h[-1]], p[i])[0] < 0:
                h.pop()
            h.append(i)
        return h
    lower, upper = chain(idx), chain(idx[::-1])
    ring = lower[:-1] + upper[:-1]
    return {(ring[k], ring[(k + 1) % len(ring)]) for k in range(len(ring))}


def orient_simplices(points, simplices):
    """the simplices in counter-clockwise order, and their exact orient signs"""
    p = np.asarray(points, np.float64)
    s = np.array(simplices, np.int64)
    o = orient(p[s[:, 0]], p[s[:, 1]], p[s[:, 2]])
    cw = o < 0
    s[cw] = s[cw][:, [0, 2, 1]]
    return s, o


def check(points, simplices, neighbors=None, ccw=False):
    """assert that `simplices` (with `neighbors`, scipy's convention, if given)
    is a Delaunay triangulation of `points`; with `ccw` the simplices must
    also be counter-clockwise as given.  Returns a dict of counts."""
    p = np.asarray(points, np.float64)
    M = len(p)
    s, o = orient_simplices(p, simplices)
    T = len(s)
    assert np.all(o != 0), "%d simplices with zero area" % (o == 0).sum()
    if ccw:
        assert np.all(o > 0), "%d clockwise simplices" % (o < 0).sum()
    # edges: directed edge k of simplex t is (s[t, k+1], s[t, k+2]), opposite s[t, k]
    a = np.stack([s[:, 1], s[:, 2], s[:, 0]], 1).ravel()
    b = np.stack([s[:, 2], s[:, 0], s[:, 1]], 1).ravel()
    key, rkey = a*M + b, b*M + a
    order = np.argsort(key, kind="stable")
    ks = key[order]
    assert np.all(ks[1:] != ks[:-1]), "an edge is shared by more than two simplices"
    pos = np.searchsorted(ks, rkey)
    pos = np.minimum(pos, len(ks) - 1)
    twin = np.where(ks[pos] == rkey, order[pos], -1)      # directed-edge index of the twin
    inner = twin >= 0
    if neighbors is not None:
        nb = np.asarray(neighbors, np.int64)
        s0 = np.asarray(simplices, np.int64)
        # neighbours are given for the simplices as given: map the twin's simplex
        want = np.where(inner, twin//3, -1).reshape(T, 3)
        # column k of a clockwise simplex was swapped with column 3-k (k = 1, 2)
        cw = (s != s0).any(1)
        got = nb.copy()
        got[cw] = nb[cw][:, [0, 2, 1]]
        assert np.array_equal(got, want), "neighbors disagree with the simplices"
    # boundary = convex hull, collinear points included
    boundary = {(int(x), int(y)) for x, y in zip(a[~inner], b[~inner])}
    uniq, first, inv = np.unique(p + 0.0, axis=0, return_index=True, return_inverse=True)
    canon = first[inv.ravel()]                            # lowest index of each distinct point
    hull = hull_edges(p)
    boundary_c = {(int(canon[x]), int(canon[y])) for x, y in boundary}
    assert boundary_c == hull, "boundary is not the convex hull (%d vs %d edges)" % (
        len(boundary_c), len(hull))
    # every distinct point is a vertex, and only once
    verts = np.unique(s)
    assert len(np.unique(canon[verts])) == len(verts), "two vertices at one point"
    V = len(uniq)
    assert len(verts) == V, "%d distinct points but %d vertices" % (V, len(verts))
    h = len(hull)
    assert T == 2*V - h - 2, "T = %d but 2V - h - 2 = %d" % (T, 2*V - h - 2)
    # local Delaunay on interior edges (each once)
    e = np.flatnonzero(inner & (np.arange(3*T) < twin))
    t, u = e//3, twin[e]//3
    d = s[u, twin[e] % 3]
    ic = incircle(p[s[t, 0]], p[s[t, 1]], p[s[t, 2]], p[d])
    assert np.all(ic <= 0), "%d interior edges are not locally Delaunay" % (ic > 0).sum()
    return dict(T=T, V=V, h=h, interior_edges=len(e), cocircular=int((ic == 0).sum()),
                boundary=len(boundary))


def canonical(points, simplices):
    """the simplices with every vertex replaced by the lowest index of the
    points equal to it (triangulations may keep different duplicates)"""
    p = np.asarray(points, np.float64) + 0.0
    _, first, inv = np.unique(p, axis=0, return_index=True, return_inverse=True)
    return first[inv.ravel()][np.asarray(simplices)]


def cocircular_differences(points, simp_a, simp_b):
    """Explain the difference between two Delaunay triangulations of one point
    set: every edge of `simp_a` that `simp_b` lacks must be the diagonal of an
    exactly cocircular quadrilateral of `simp_a` (and likewise with the roles
    swapped).  Returns the sets of sorted vertex triples of the simplices of
    each that lie in such quadrilaterals (vertices as ``canonical`` numbers
    them); raises AssertionError otherwise."""
    p = np.asarray(points, np.float64)
    simp_a, simp_b = canonical(p, simp_a), canonical(p, simp_b)

    def edges(s):
        out = {}
        for t, tri in enumerate(np.asarray(s).tolist()):
            for k in range(3):
                e = tuple(sorted((tri[(k + 1) % 3], tri[(k + 2) % 3])))
                out.setdefault(e, []).append((t, tri[k]))
        return out

    result = []
    for x, y in ((simp_a, simp_b), (simp_b, simp_a)):
        ex, ey = edges(x), edges(y)
        sx, _ = orient_simplices(p, x)
        tris = set()
        for e, owners in ex.items():
            if e in ey:
                continue
            assert len(owners) == 2, "edge %s differs on the hull" % (e,)
            (t, c), (u, d) = owners
            assert incircle(p[sx[t, 0]], p[sx[t, 1]], p[sx[t, 2]], p[d])[0] == 0, \
                "edge %s differs but its quadrilateral is not cocircular" % (e,)
            tris.add(tuple(sorted(np.asarray(x)[t].tolist())))
            tris.add(tuple(sorted(np.asarray(x)[u].tolist())))
        result.append(tris)
    return result[0], result[1]
