"""The numpy restatement of the device regridding (oracle/regrid_oracle.py)
against scipy's griddata and exact rational arithmetic, without a GPU.  The
point sets are those tests/test_gpu_regrid_exact.py puts through
rtx_grid_linear, which must give the restatement's bits."""
import os
from fractions import Fraction

import numpy as np
import pytest
from scipy.interpolate import griddata
from scipy.spatial import Delaunay

import psf_oracle
import regrid_oracle as ro
from conftest import GOLDEN

# Bounds asserted on every regridding, in units of eps = 2^-52 times the node's
# condition (rho + 2)(1 + max_k (|Tinv| |p - r|)_k), rho the condition number
# of the triangle's determinant (regrid_oracle.node_condition).  Derived: the
# coordinates c_k are rounded from dx, dy, two products and two sums, the
# transform carries a relative error of about rho eps, so each c_k is off by a
# few eps times the condition, and the value ((0 + c0 v0) + c1 v1) + c2 v2 by
# that times sum |v_k|.  The restatement gives the device's bits, so what these
# host tests measure is what the device produces.
BARY_EXCESS = 2.      # a winner's exact coordinates are >= -100 eps - BARY_EXCESS eps cond
VALUE_RATIO = 2.      # |value - exact interpolant| <= VALUE_RATIO eps cond sum |v_k|


# ---- the point sets -------------------------------------------------------------
def disc(m, seed, r=1.):
    rng = np.random.default_rng(seed)
    rad, phi = r*np.sqrt(rng.random(m)), 2*np.pi*rng.random(m)
    return np.stack([rad*np.cos(phi), rad*np.sin(phi)], -1)


def smooth(p):
    return np.cos(4*p[:, 0])*p[:, 1] + p[:, 0]**2


def traced_pupil(name):
    """the reference's per-ray exit-pupil points and OPD (finite rays)"""
    d = np.load(os.path.join(GOLDEN, "vs_reference", name + ".npz"))
    x, y, t = d["x"], d["y"], d["t"]
    ok = np.isfinite(x) & np.isfinite(y) & np.isfinite(t)
    return np.stack([x[ok], y[ok]], -1), t[ok], d["o"].shape[0]


def chord_pupil(m, seed, c=0.55):
    """a disc clipped at y = c: points on the chord itself (collinear hull
    points) and a few within ulps of it make thin triangles along the cut"""
    rng = np.random.default_rng(seed)
    p = disc(m, seed)
    p = p[p[:, 1] < c]
    w = np.sqrt(1 - c*c)
    on = np.stack([np.linspace(-w, w, 41), np.full(41, c)], -1)
    off = np.stack([rng.uniform(-w, w, 12), np.full(12, c)], -1)
    off[:, 1] = np.nextafter(off[:, 1], np.where(np.arange(12) % 2, 0., 1.))   # just below / above
    off[1::2, 1] = np.nextafter(off[1::2, 1], 0.)
    return np.concatenate([p, on, off])


def dyadic_grid(n=65, stride=2, seed=3):
    """points exactly on the nodes of the (n, n) grid of half-width 1 (node
    coordinates are multiples of 2/(n - 1) = 1/32): every stride-th node of
    the border and a random half of the interior ones, so that grid nodes fall
    exactly on vertices and on shared edges"""
    gh = psf_oracle.grid(n, 1.)[2]
    assert np.array_equal(gh*(n - 1)/2, np.round(gh*(n - 1)/2))
    i, j = np.meshgrid(np.arange(0, n, stride), np.arange(0, n, stride), indexing="ij")
    i, j = i.ravel(), j.ravel()
    rng = np.random.default_rng(seed)
    border = (i == 0) | (j == 0) | (i == n - 1) | (j == n - 1)
    keep = border | (rng.random(len(i)) < 0.5)
    return np.stack([gh[i[keep]], gh[j[keep]]], -1), gh


def warp_and_lane(seed=5):
    """a few points spread over the disc (large triangles: boxes of more than
    GRID_WARP_NODES nodes) around a dense cluster (boxes of a few nodes)"""
    return np.concatenate([disc(24, seed), disc(3000, seed + 1, 0.2) + [0.3, -0.2]])


def slivers(seed=6):
    """points on a line, a few within 1e-9 of it and one far off, turned by
    0.3 rad: triangles whose determinant cancels to 1e-9 of its terms"""
    rng = np.random.default_rng(seed)
    line = np.stack([np.linspace(0., 1., 50), np.zeros(50)], -1)
    near = np.stack([rng.random(7), 1e-9*(1 + rng.random(7))], -1)
    p = np.concatenate([line, near, [[0.5, 1.]], disc(200, seed, 0.3) + [0.5, 0.6]])
    c, s = np.cos(0.3), np.sin(0.3)
    return p @ np.array([[c, s], [-s, c]])


def uneven_axis(n, h, seed=0):
    """an ascending axis on [-h, h] with random, widely varying gaps"""
    rng = np.random.default_rng(seed)
    g = np.cumsum(rng.random(n - 1)**3 + 1e-3)
    return -h + 2*h*np.concatenate([[0.], g/g[-1]])


def host_case(name):
    """(points, values, n, gh) of the host cases"""
    if name.startswith("psf_"):
        p, t, n = traced_pupil(name)
        return p, t, n, psf_oracle.grid(n, np.fabs(p).max())[2]
    if name == "disc":
        p = disc(5000, 1)
    elif name == "chord":
        p = chord_pupil(4000, 2)
    elif name == "dyadic":
        p, gh = dyadic_grid()
        return p, smooth(p), len(gh), gh
    elif name == "warp_and_lane":
        p = warp_and_lane()
    elif name == "slivers":
        p = slivers()
    n = int(4*len(p)**.5)
    return p, smooth(p), n, psf_oracle.grid(n, np.fabs(p).max())[2]


HOST_CASES = ["disc", "psf_cooke_f0", "psf_cooke_f07", "chord", "dyadic", "warp_and_lane", "slivers"]


# ---- the restatement is griddata where the winners agree -------------------------
@pytest.mark.parametrize("name", HOST_CASES)
def test_restatement_is_griddata(name):
    p, t, n, gh = host_case(name)
    tri = Delaunay(p)
    r = ro.restate(p, t, tri.simplices, tri.transform, gh)
    xs, ys = np.meshgrid(gh, gh, indexing="ij")
    want = griddata((p[:, 0], p[:, 1]), t, (xs, ys), method="linear", fill_value=np.nan)
    fw = psf_oracle.winner(tri, xs, ys)
    same = r["winner"] == fw
    assert np.array_equal(r["value"][same], want[same], equal_nan=True), name
    fin = np.isfinite(want)
    # another winner than scipy's walk only on a shared edge or vertex: the
    # same interpolant there to rounding; the NaN masks differ only on the hull
    other = ~same & fin & np.isfinite(r["value"])
    assert np.all(np.fabs(r["value"][other] - want[other]) <= 1e-13*np.fabs(t).max()), name
    assert r["reach"] <= 1, "a node claimed more than one node beyond its simplex's box"
    chk = ro.exact_check(p, t, tri.simplices, tri.transform, gh, r["winner"], r["value"])
    flip = np.isnan(r["value"]) != np.isnan(want)
    assert np.all(np.fabs(chk["depth"][flip]) <= chk["tol"]), name
    print("%s: n=%d, winner = find_simplex at %d of %d finite nodes, hull flips %d"
          % (name, n, (same & fin).sum(), fin.sum(), flip.sum()))


# ---- the restatement's winners against exact arithmetic --------------------------
@pytest.mark.parametrize("name", HOST_CASES)
def test_restatement_exact(name):
    """winners contain their nodes up to the 100-eps tolerance, exactly;
    nodes inside the exact hull by more than 1e3 eps h have a winner, nodes
    outside by more have none; values are within VALUE_RATIO of the exact
    interpolant"""
    p, t, n, gh = host_case(name)
    tri = Delaunay(p)
    r = ro.restate(p, t, tri.simplices, tri.transform, gh)
    chk = ro.exact_check(p, t, tri.simplices, tri.transform, gh, r["winner"], r["value"])
    assert_exact(chk, r["winner"], name)


def assert_exact(chk, winner, what):
    depth, tol = chk["depth"], chk["tol"]
    assert np.all(winner[depth > tol] >= 0), (what, "a node deep inside the hull has no winner")
    assert np.all(winner[depth < -tol] < 0), (what, "a node outside the hull has a winner")
    assert chk["bary_excess"] <= BARY_EXCESS, (what, chk["bary_excess"])
    assert chk["value_ratio"] <= VALUE_RATIO, (what, chk["value_ratio"])
    print("%s: %d nodes checked exactly, least exact coordinate %.2e, excess %.2f, "
          "value error %.2f eps cond sum|v|" % (what, chk["checked"], chk["bary_low"],
                                                chk["bary_excess"], chk["value_ratio"]))


def test_exact_hull_and_coordinates():
    """the exact helpers on a square with collinear points on its sides"""
    sq = np.array([[0, 0], [1, 0], [1, 1], [0, 1], [.5, 0], [1, .25], [.5, .5]], float)
    hull = ro.exact_hull(sq)
    assert sorted((float(x), float(y)) for x, y in hull) == [(0, 0), (0, 1), (1, 0), (1, 1)]
    assert ro.in_hull_exact(hull, (.5, .5)) == 1
    assert ro.in_hull_exact(hull, (1., .75)) == 0
    assert ro.in_hull_exact(hull, (np.nextafter(1., 2.), .5)) == -1
    c = ro.exact_barycentric(sq[[0, 1, 3]], (.25, .5))
    assert c == (Fraction(1, 4), Fraction(1, 4), Fraction(1, 2))
    d = ro.hull_depth(hull, np.array([.5, 2., .1]), np.array([.5, .5, .5]))
    np.testing.assert_allclose(d, [.5, -1., .1])


# ---- the explicit inverse rtx_delaunay writes -------------------------------------
TINV_BOUND = 2.5      # |Tinv - exact| <= TINV_BOUND (rho + 1) eps |exact|, entry by entry


def check_inverse(p, simplices, tr=None):
    """the explicit inverse (the restatement's, or the device's `tr`) against
    the exact rational inverse of every triangle.  Derived bound: the four
    differences are rounded (u = eps/2 each), det = t00 t11 - t01 t10 adds
    3u (|t00 t11| + |t01 t10|) = 3 u rho |det|, the quotient one more u, so each
    entry is within (3 rho + 3) u + O(u^2) <= 2.5 (rho + 1) eps of the exact one"""
    want, rho = ro.delaunay_transform(p, simplices)
    tr = want if tr is None else tr
    worst = 0.
    for s, row, rh in zip(np.asarray(simplices).tolist(), tr.reshape(-1, 6), rho):
        ex = ro.exact_inverse(p, s)          # raises for a triangle of zero area
        if np.isinf(rh):
            # the rounded determinant is 0 (vertices collinear to rounding):
            # a NaN row, which never claims a node, as scipy's transform is
            # NaN for a nearly singular simplex
            assert np.isnan(row).all()
            continue
        for got, e in zip(row[:4].tolist(), ex):
            if e == 0:
                assert got == 0
                continue
            worst = max(worst, float(abs(Fraction(got) - e)/abs(e))/(ro.EPS*(rh + 1)))
        assert row[4] == p[s[2], 0] and row[5] == p[s[2], 1]
    assert worst <= TINV_BOUND, worst
    return worst, rho[np.isfinite(rho)]


@pytest.mark.parametrize("name", ["chord", "slivers", "psf_cooke_f07", "dyadic"])
def test_explicit_inverse_bound(name):
    p = host_case(name)[0]
    tri = Delaunay(p)
    ok = ~np.isnan(tri.transform[:, 0, 0])
    worst, rho = check_inverse(p, tri.simplices[ok])
    print("%s: %d triangles, largest finite rho %.1e, inverse error %.3f (rho + 1) eps"
          % (name, ok.sum(), rho.max(), worst))
