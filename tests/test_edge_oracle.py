"""The boundary bundles of oracle/edge_bundles.py really straddle their
boundaries in np_oracle, and (where the reference tree is staged) the
reference's own Spheroid.intercept / clip / refract / propagate make the same
decisions with the same bit patterns, signed zeros included.  CPU only."""
import warnings

import numpy as np
import pytest

import edge_bundles as eb
import np_oracle
import ref_shim

CASES = eb.cases()


def _bits(a):
    a = np.asarray(a, np.float64)
    return np.where(np.isnan(a), np.uint64(0x7ff8000000000000), a.view(np.uint64))


@pytest.mark.parametrize("c", CASES, ids=[c.name for c in CASES])
def test_bundle_straddles_its_boundary(c):
    Y, U, I, T = np_oracle.trace(c.table, c.y0, c.u0, clip=c.clip)
    for ik, il, at in c.edges:
        lost = np.isnan((U if at == "U" else Y)[0]).any(1)
        assert not lost[ik] and lost[il], (c.name, ik, il)
        # adjacent doubles in exactly one launch coordinate
        d = np.flatnonzero((c.y0[ik] != c.y0[il]) | (c.u0[ik] != c.u0[il]))
        la, lb = np.hstack([c.y0[ik], c.u0[ik]]), np.hstack([c.y0[il], c.u0[il]])
        walked = np.flatnonzero(la != lb)
        assert len(d) >= 1 and len(walked) >= 1
        k = walked[0]
        assert abs(int(eb.key(la[k])) - int(eb.key(lb[k]))) == 1, (c.name, la[k], lb[k])
        assert c.margin[ik] == c.margin[il] == 1
    assert len(c.margin) == len(c.y0)


def test_fused_rim_rays_exist():
    """rim_axial holds a ray whose clip decision a fused x*x + y*y would flip"""
    c = next(c for c in CASES if c.name == "rim_axial")
    near = np.isfinite(c.margin) & (c.margin <= eb.W + 1)
    assert eb.fused_flip_rim(1.3*1.3, c.y0[near, 0], c.y0[0, 1]).any()


def test_signed_zero_plane_intercept():
    """a ray starting on a plane (y.z = +0, u.z > 0) has T = -0 in the oracle"""
    c = next(c for c in CASES if c.name == "plane_zeros")
    Y, U, I, T = np_oracle.trace(c.table, c.y0, c.u0, clip=c.clip)
    start = (c.y0[:, 2] == 0) & ~np.signbit(c.y0[:, 2]) & (c.u0[:, 2] > 0)
    assert start.any() and np.signbit(T[0][start]).all()


@pytest.mark.skipif(not ref_shim.available(), reason="reference tree not present")
@pytest.mark.parametrize("c", CASES, ids=[c.name for c in CASES])
def test_reference_surface_decisions(c):
    """the reference's Spheroid methods on surface 0 of every case, bit for bit"""
    R = ref_shim.load()
    rec = c.table[0]
    e = c.elements[0][1]
    kw = dict(curvature=e.curvature, conic=e.conic, aspherics=e.aspherics,
              alternate_intersection=e.alternate_intersection)
    if np.isfinite(e.radius):
        kw["radius"] = e.radius
    with warnings.catch_warnings(), np.errstate(all="ignore"):
        warnings.simplefilter("ignore")
        s = R.Spheroid(**kw)
        s.get_n_mu = lambda n0, l: (float(rec["n"]), float(rec["mu"]))
        y = c.y0 - rec["offset"]
        u = c.u0
        # intercept / clip / refract one by one (the reference's own code)
        t = s.intercept(y.copy(), u)
        y1 = y + t[:, None]*u
        u1 = s.clip(y1, u) if c.clip else u
        mu = float(rec["mu"])
        u2 = s.refract(y1, u1, mu) if mu else u1
        ry, ru, rn, rt = s.propagate(y.copy(), u, float(rec["n0"]), 5.876e-7, clip=c.clip)
        Y, U, I, T = np_oracle.trace(c.table, c.y0, c.u0, clip=c.clip)
    newton = int(rec["n_asph"]) >= 0
    for got, want, what in ((ry, Y[0], "y"), (ru, U[0], "u"), (rt, T[0], "t"),
                            (y1, Y[0], "y (steps)"), (u2, U[0], "u (steps)")):
        if newton:      # fprime goes through np.dot (BLAS) in the reference
            assert np.array_equal(np.isnan(got), np.isnan(want)), (c.name, what)
            np.testing.assert_allclose(got, want, rtol=1e-13, atol=1e-13)
        else:
            assert np.array_equal(_bits(got), _bits(want)), (c.name, what)
