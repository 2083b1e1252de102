"""rtx_grid_linear bit for bit against the numpy restatement of its claim and
evaluation passes (oracle/regrid_oracle.py) -- winner, value and NaN mask at
every node -- and against exact rational arithmetic: nodes deep inside the
convex hull are finite, nodes outside it are NaN, winners contain their nodes
and values are within a stated bound of the exact interpolant.  Also the
transform rtx_delaunay writes against the exact inverse of every triangle, and
the NaN mask of its regridding against griddata's."""
import types

import numpy as np
import pytest
from scipy.interpolate import griddata
from scipy.spatial import Delaunay

import psf_oracle
import regrid_oracle as ro
from test_gpu_delaunay import degenerate_sets
from test_regrid_oracle import (assert_exact, chord_pupil, check_inverse, disc, dyadic_grid,
                                slivers, smooth, traced_pupil, uneven_axis, warp_and_lane)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from rayopt_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def host_arrays(eng, tri):
    """(simplices, transform) of a scipy triangulation, a DeviceTriangulation
    or a namespace holding the two arrays"""
    if hasattr(tri, "download"):
        s, _, tr = tri.download()
        return s, tr
    return np.asarray(tri.simplices), np.asarray(tri.transform)


def check(eng, p, t, tri, gh, what, exact=True):
    """the device regridding equals the restatement bit for bit; with `exact`
    also the exact checks.  Returns (value, winner, restatement)"""
    gh = np.asarray(gh, np.float64)
    got, win = eng.grid_linear(p, t, tri, len(gh), gh, winner=True)
    s, tr = host_arrays(eng, tri)
    r = ro.restate(p, t, s, tr, gh)
    bad = win != r["winner"]
    assert not bad.any(), (what, "winner differs at %d nodes" % bad.sum(), np.argwhere(bad)[:5])
    nan = np.isnan(r["value"])
    assert np.array_equal(np.isnan(got), nan), what
    assert np.array_equal(got[~nan].view(np.int64), r["value"][~nan].view(np.int64)), what
    assert r["reach"] <= 1, (what, r["reach"])
    if exact:
        assert_exact(ro.exact_check(p, t, s, tr, gh, win, got), win, what)
    big = r["box_nodes"] > ro.GRID_WARP_NODES
    print("%s: n=%d, %d simplices (%d by a warp), %d finite nodes, kernel %.3f ms"
          % (what, len(gh), len(s), big.sum(), (~nan).sum(), eng.last_kernel_ms()))
    return got, win, r


def device_tri(eng, p):
    return eng.delaunay(p)


@pytest.mark.parametrize("m", [2000, 20000])
def test_random_disc(eng, m):
    p = disc(m, m)
    n = int(4*m**.5)
    check(eng, p, smooth(p), Delaunay(p), psf_oracle.grid(n, np.fabs(p).max())[2], "disc %d" % m)


@pytest.mark.parametrize("name", ["psf_cooke_f0", "psf_cooke_f07", "psf_double_gauss_f07",
                                  "psf_mirror"])
def test_traced_pupil(eng, name):
    p, t, n = traced_pupil(name)
    xs = np.mgrid[-1:1:1j*n, -1:1:1j*n][0]*np.fabs(p).max()     # lazy.regrid's grid
    check(eng, p, t, Delaunay(p), xs[:, 0].copy(), name)


@pytest.mark.parametrize("triangulation", ["host", "device"])
@pytest.mark.parametrize("name", ["chord", "slivers", "dyadic"])
def test_thin_and_exact_sets(eng, name, triangulation):
    """a pupil clipped by a chord (collinear hull points and thin triangles),
    slivers whose determinant cancels to 1e-9, and points exactly on grid
    nodes (nodes on vertices and shared edges)"""
    if name == "dyadic":
        p, gh = dyadic_grid()
    else:
        p = chord_pupil(4000, 2) if name == "chord" else slivers()
        gh = psf_oracle.grid(int(4*len(p)**.5), np.fabs(p).max())[2]
    tri = Delaunay(p) if triangulation == "host" else device_tri(eng, p)
    try:
        check(eng, p, smooth(p), tri, gh, "%s (%s)" % (name, triangulation))
    finally:
        if triangulation == "device":
            tri.free()


@pytest.mark.parametrize("triangulation", ["host", "device"])
@pytest.mark.parametrize("name", list(degenerate_sets()))
def test_degenerate_sets(eng, name, triangulation):
    """grids, duplicates and collinear hulls; with the device triangulation
    also its NaN mask against griddata's, equal away from the hull's boundary"""
    p = degenerate_sets()[name]
    t = np.sin(3*p[:, 0]) + p[:, 1]**2
    xs, ys, gh = psf_oracle.grid(200, np.fabs(p).max())
    tri = Delaunay(p) if triangulation == "host" else device_tri(eng, p)
    try:
        got, win, r = check(eng, p, t, tri, gh, "%s (%s)" % (name, triangulation))
    finally:
        if triangulation == "device":
            tri.free()
    want = griddata((p[:, 0], p[:, 1]), t, (xs, ys), method="linear", fill_value=np.nan)
    flip = np.isnan(got) != np.isnan(want)
    if flip.any():
        hull = ro.exact_hull(p)
        depth = ro.hull_depth(hull, xs[flip], ys[flip])
        assert np.all(np.fabs(depth) <= 1e3*ro.EPS*np.fabs(p).max()), (name, np.fabs(depth).max())
    print("%s (%s): NaN mask differs from griddata's at %d nodes, all on the hull"
          % (name, triangulation, flip.sum()))


def test_warp_and_lane_paths(eng):
    """one launch with simplices on both claim paths"""
    p = warp_and_lane()
    gh = psf_oracle.grid(400, np.fabs(p).max())[2]
    _, _, r = check(eng, p, smooth(p), Delaunay(p), gh, "warp and lane")
    box = r["box_nodes"]
    assert (box > ro.GRID_WARP_NODES).sum() >= 10 and (box[box > 0] <= ro.GRID_WARP_NODES).sum() >= 1000


@pytest.mark.parametrize("where", ["inner", "shifted", "off"])
def test_triangles_off_the_grid(eng, where):
    """a grid covering part of the points (triangles partly or wholly off the
    grid) or none of them (every node NaN)"""
    p = disc(3000, 11)
    t = smooth(p)
    gh = {"inner": np.linspace(-.5, .5, 150), "shifted": np.linspace(.4, 1.7, 171),
          "off": np.linspace(2., 3., 50)}[where]
    got, _, _ = check(eng, p, t, Delaunay(p), gh, "grid %s" % where)
    if where == "off":
        assert np.isnan(got).all()
    else:
        assert np.isfinite(got).any() and np.isnan(got).any() == (where == "shifted")


def test_nan_transform_rows(eng):
    """caller-supplied NaN transform rows never win: whole rows, a NaN in
    Tinv's last entry only, a NaN in r only"""
    p = disc(3000, 12)
    tri = Delaunay(p)
    tr = tri.transform.copy()
    tr[::5] = np.nan
    tr[1::7, 1, 1] = np.nan
    tr[2::11, 2, 0] = np.nan
    nan_rows = np.isnan(tr).any((1, 2))
    arg = types.SimpleNamespace(simplices=tri.simplices, transform=tr)
    gh = psf_oracle.grid(220, np.fabs(p).max())[2]
    got, win, _ = check(eng, p, smooth(p), arg, gh, "NaN rows", exact=False)
    assert not nan_rows[win[win >= 0]].any()
    assert np.isnan(got).sum() > np.isnan(eng.grid_linear(p, smooth(p), tri, 220, gh)).sum()


@pytest.mark.parametrize("n", [2, 3, 4099])
def test_grid_sizes(eng, n):
    p = disc(3000, 13)
    h = np.fabs(p).max()
    check(eng, p, smooth(p), Delaunay(p), psf_oracle.grid(n, h)[2], "n=%d" % n, exact=n < 4000)
    if n == 2:   # the four corners lie outside the disc
        assert np.isnan(eng.grid_linear(p, smooth(p), Delaunay(p), 2, [-h, h])).all()


AXES = ["mgrid", "uneven", "descending", "descending_uneven"]


def axis(kind, n, h):
    if kind == "mgrid":
        return (np.mgrid[-1:1:1j*n, -1:1:1j*n][0]*h)[:, 0].copy()
    g = uneven_axis(n, h) if "uneven" in kind else psf_oracle.grid(n, h)[2]
    return g[::-1].copy() if kind.startswith("descending") else g


@pytest.mark.parametrize("kind", AXES)
def test_grid_axes(eng, kind):
    """any strictly monotone axis: node (i, j) = (gh[i], gh[j]) and the
    restatement's values, NaN only off the hull"""
    p = disc(5000, 14)
    gh = axis(kind, 283, np.fabs(p).max())
    got, _, _ = check(eng, p, smooth(p), Delaunay(p), gh, "axis %s" % kind)
    xs, ys = np.meshgrid(gh, gh, indexing="ij")
    want = griddata((p[:, 0], p[:, 1]), smooth(p), (xs, ys), method="linear", fill_value=np.nan)
    both = np.isfinite(got) & np.isfinite(want)
    assert np.abs(got[both] - want[both]).max() <= 1e-13*np.fabs(smooth(p)).max()
    assert both.sum() >= np.isfinite(want).sum() - 10, kind


@pytest.mark.parametrize("kind", AXES)
def test_grid_axes_traced_pupil(eng, kind):
    p, t, n = traced_pupil("psf_cooke_f07")
    check(eng, p, t, Delaunay(p), axis(kind, n, np.fabs(p).max()), "cooke f07 axis %s" % kind)


def test_axis_refused(eng):
    p = disc(100, 1)
    for gh in ([0., 1., 1., 2.], [0., 2., 1., 3.], [0., np.nan, 2., 3.]):
        with pytest.raises(ValueError, match="monotone"):
            eng.grid_linear(p, smooth(p), Delaunay(p), 4, gh)


# ---- the transform rtx_delaunay writes --------------------------------------------
TRANSFORM_SETS = ["chord", "slivers", "dyadic", "disc", "psf_cooke_f07"] + list(degenerate_sets())


@pytest.mark.parametrize("name", TRANSFORM_SETS)
def test_device_transform(eng, name):
    """every triangle's transform: the restatement of the explicit inverse bit
    for bit, within (3 rho + 3) eps/2 of the exact inverse entry by entry, NaN
    only where the rounded determinant is 0"""
    if name in ("chord", "slivers", "dyadic", "disc", "psf_cooke_f07"):
        p = {"chord": lambda: chord_pupil(4000, 2), "slivers": slivers,
             "dyadic": lambda: dyadic_grid()[0], "disc": lambda: disc(10000, 3),
             "psf_cooke_f07": lambda: traced_pupil("psf_cooke_f07")[0]}[name]()
    else:
        p = degenerate_sets()[name]
    tri = eng.delaunay(p)
    try:
        s, _, tr = tri.download()
    finally:
        tri.free()
    want, _ = ro.delaunay_transform(p, s)
    assert np.array_equal(tr.view(np.int64), want.view(np.int64)), name
    worst, rho = check_inverse(p, s, tr)
    print("%s: %d triangles (%d with a rounded determinant of 0), largest finite rho %.1e, "
          "inverse error %.3f (rho + 1) eps" % (name, len(s), len(s) - len(rho), rho.max(), worst))
