"""The exact Delaunay checker (oracle/delaunay_oracle.py) on its own: it
accepts scipy's triangulations and rejects corrupted ones."""
import numpy as np
import pytest
from scipy.spatial import Delaunay

import delaunay_oracle as dto


def disc(m, seed):
    rng = np.random.default_rng(seed)
    r, phi = np.sqrt(rng.random(m)), 2*np.pi*rng.random(m)
    return np.stack([r*np.cos(phi), r*np.sin(phi)], -1)


def square_grid(k):
    return np.stack(np.meshgrid(np.arange(k, dtype=float), np.arange(k, dtype=float)), -1).reshape(-1, 2)


@pytest.mark.parametrize("m", [3, 4, 5, 100, 3000])
def test_accepts_scipy_general_position(m):
    p = disc(m, m)
    tri = Delaunay(p)
    st = dto.check(p, tri.simplices, tri.neighbors)
    assert st["T"] == len(tri.simplices) and st["cocircular"] == 0


def test_accepts_scipy_square_grid():
    """101^2 grid: every cell is a cocircular quadrilateral; scipy gives 20000
    simplices = 2V - h - 2 and no degenerate transform"""
    p = square_grid(101)
    tri = Delaunay(p)
    st = dto.check(p, tri.simplices, tri.neighbors)
    assert st["T"] == 20000 == 2*10201 - 400 - 2
    assert st["h"] == 400 and st["cocircular"] == 10000
    assert not np.isnan(tri.transform).any()


def test_predicates_exact():
    """points on a line or circle up to one ulp, decided by Fractions"""
    a, b = np.array([0.1, 0.3]), np.array([0.7, 0.9])
    c = a + 0.5*(b - a)
    assert dto.orient(a, b, c)[0] == dto._orient_exact(a, b, c)
    c2 = c.copy()
    c2[0] = np.nextafter(c2[0], 1)
    assert dto.orient(a, b, c2)[0] == dto._orient_exact(a, b, c2) != 0
    q = np.array([[0., 0.], [1., 0.], [1., 1.], [0., 1.]])
    assert dto.incircle(*q)[0] == 0
    q[3, 1] = np.nextafter(1., 2.)
    assert dto.incircle(*q)[0] == -1


def test_rejects_flipped_edge():
    p = disc(200, 1)
    tri = Delaunay(p)
    s, nb = tri.simplices.copy(), tri.neighbors
    # flip the shared edge of simplex 0 and an interior neighbour
    for k in range(3):
        u = nb[0, k]
        if u >= 0:
            break
    a, b = s[0, (k + 1) % 3], s[0, (k + 2) % 3]
    c = s[0, k]
    d = [v for v in s[u] if v not in (a, b)][0]
    s[0], s[u] = [c, a, d], [c, d, b]
    if dto.orient(p[[c]], p[[a]], p[[d]])[0] == 0 or dto.orient(p[[c]], p[[d]], p[[b]])[0] == 0:
        pytest.skip("degenerate flip")
    with pytest.raises(AssertionError, match="locally Delaunay|zero area|shared"):
        dto.check(p, s)


def test_rejects_dropped_triangle():
    p = disc(300, 2)
    s = Delaunay(p).simplices
    with pytest.raises(AssertionError):
        dto.check(p, s[1:])


def test_rejects_boundary_not_hull():
    """drop a hull vertex's triangles: the boundary is no longer the hull"""
    p = disc(300, 3)
    tri = Delaunay(p)
    v = tri.convex_hull[0, 0]
    keep = ~(tri.simplices == v).any(1)
    with pytest.raises(AssertionError, match="hull|vertices"):
        dto.check(p, tri.simplices[keep])


def test_rejects_clockwise_with_ccw_flag():
    p = disc(100, 4)
    s, _ = dto.orient_simplices(p, Delaunay(p).simplices)
    dto.check(p, s, ccw=True)
    s[5] = s[5, [0, 2, 1]]
    dto.check(p, s)
    with pytest.raises(AssertionError, match="clockwise"):
        dto.check(p, s, ccw=True)


def test_rejects_bad_neighbors():
    p = disc(100, 5)
    tri = Delaunay(p)
    nb = tri.neighbors.copy()
    nb[0] = np.roll(nb[0], 1)
    with pytest.raises(AssertionError, match="neighbors"):
        dto.check(p, tri.simplices, nb)


def test_cocircular_differences_grid():
    """the grid's two diagonals of one cell: explained; a non-cocircular
    difference is not"""
    p = square_grid(3)
    s = Delaunay(p).simplices
    other = s.copy()
    # re-triangulate the cell with the other diagonal
    st = {tuple(sorted(t)) for t in s.tolist()}
    a, b = dto.cocircular_differences(p, s, s)
    assert not a and not b
    cell = [0, 1, 3, 4]                       # (0,0) (1,0) (0,1) (1,1)
    inside = [k for k, t in enumerate(s.tolist()) if set(t) <= set(cell)]
    assert len(inside) == 2
    diag = set(s[inside[0]]) & set(s[inside[1]])
    o = sorted(set(cell) - diag)
    d = sorted(diag)
    other[inside[0]] = [o[0], o[1], d[0]]
    other[inside[1]] = [o[0], o[1], d[1]]
    dto.check(p, other)
    a, b = dto.cocircular_differences(p, s, other)
    assert len(a) == 2 and len(b) == 2 and st
    q = p.copy()
    q[4] = [1.0, 1.01]                        # the cell is no longer cocircular
    with pytest.raises(AssertionError):
        dto.cocircular_differences(q, Delaunay(q).simplices, other)
