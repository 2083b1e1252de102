"""Host side of the tolerance analysis (rayopt_b200/tolerance.py): the
perturbed tables against pack_system of a reference System with the same
change made, the refusals, the delta generators, and the finite-ray rms of
the oracle against the reference's GeometricTrace.rms.  No GPU."""
import copy
import warnings

import numpy as np
import pytest

import ref_shim
import tolerance_oracle
from rayopt_b200.surface_table import SURFACE_DTYPE, pack_system
from rayopt_b200.tolerance import (monte_carlo_deltas, perturbed_tables, sensitivity_deltas)

needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="no reference tree staged")


@pytest.fixture(scope="module")
def R():
    warnings.simplefilter("ignore")
    np.seterr(all="ignore")
    return ref_shim.load()


def build(R, name):
    import yaml
    import systems_yaml
    s = R.System(**yaml.safe_load(systems_yaml.SYSTEMS[name]))
    s.update()
    s.paraxial.refocus()
    return s


def tables(s):
    return np.stack([pack_system(s, l, 1, None, n0=s.refractive_index(l, 0))[0]
                     for l in s.wavelengths])


class Shifted:
    """a material whose index is another's plus `d` at every wavelength"""

    def __init__(self, base, d):
        self.base, self.d = base, d
        self.mirror = getattr(base, "mirror", False)

    def refractive_index(self, l):
        return self.base.refractive_index(l) + self.d

    def __getattr__(self, k):
        return getattr(self.base, k)


def apply(s, j, kind, d):
    """the same change made to a reference System"""
    e = s[j]
    if kind == "curvature":
        e.curvature = e.curvature + d
    elif kind == "conic":
        e.conic = e.conic + d
    elif kind.startswith("asph"):
        i = int(kind[4:])
        a = list(e.aspherics) if e.aspherics is not None else []
        a += [0.]*(i + 1 - len(a))
        a[i] = a[i] + d
        e.aspherics = a
    elif kind == "distance":
        e.distance += d
    elif kind in ("tilt_x", "tilt_y"):
        a = np.zeros(3)
        a[int(kind == "tilt_y")] = d
        e.angles = a
    elif kind == "index":
        e.material = Shifted(e.material, d)


def bits_equal(a, b):
    return a.tobytes() == b.tobytes()


# (system, [(j, kind, delta)]); tilts and index on surfaces that allow them
CASES = {
    "cooke": [(1, "curvature", 1e-3), (2, "distance", -2e-2), (3, "conic", .3),
              (4, "asph2", 1e-7), (2, "tilt_x", 1e-3), (5, "tilt_y", -2e-3), (1, "index", 2e-3),
              (6, "index", -1e-3)],
    "cooke_asph": [(2, "asph1", 3e-8), (3, "curvature", -1e-3), (6, "distance", .1),
                   (1, "tilt_y", 5e-4)],
    "double_gauss": [(3, "curvature", 2e-4), (6, "distance", 1e-2), (7, "conic", -.1),
                     (4, "tilt_x", 7e-4), (1, "index", 1e-3), (8, "asph0", 1e-6)],
    "zoom": [(2, "curvature", 1e-3), (4, "distance", .05), (1, "tilt_x", 1e-3),
             (1, "index", 5e-4)],
}


@needs_ref
@pytest.mark.parametrize("name", list(CASES))
def test_records_match_reference_system(R, name):
    """each kind alone and all together: the records are bit for bit those of
    pack_system on the reference System with the change made (the tilt
    restates the reference's rotation arithmetic, so it is bit for bit too)"""
    s = build(R, name)
    nom = tables(s)
    cases = CASES[name]
    params = [(j, k) for j, k, _ in cases]
    d = np.array([[c[2] if i == p else 0. for i, c in enumerate(cases)]
                  for p in range(len(cases))] + [[c[2] for c in cases]] + [[0.]*len(cases)])
    try:
        got = perturbed_tables(nom, params, d)
    except ValueError as e:
        pytest.fail("%s: %s" % (name, e))
    assert got.shape == (len(d), len(s.wavelengths), nom.shape[1])
    for v, row in enumerate(d):
        ref = copy.deepcopy(s)
        for (j, kind), dv in zip(params, row):
            if dv:
                apply(ref, j, kind, dv)
        want = tables(ref)
        for w in range(len(s.wavelengths)):
            for r in range(nom.shape[1]):
                assert bits_equal(got[v, w, r], want[w, r]), (name, v, w, r, params, row,
                                                              got[v, w, r], want[w, r])
    assert bits_equal(got[-1], nom)                           # zero deltas: the nominal lens


def _table(S=4):
    t = np.zeros((2, S), SURFACE_DTYPE)
    t["rot"] = np.eye(3).reshape(9)
    t["radius2"] = np.inf
    t["n_asph"] = -1
    t["offset"][..., 2] = 1.
    n = np.array([1., 1.5, 1., 1.7])[:S]
    t["n0"] = np.r_[1., n[:-1]]
    t["n"] = n
    t["mu"] = t["n0"]/t["n"]
    t["muf"], t["sgn"], t["mu2m1"] = np.abs(t["mu"]), np.sign(t["mu"]), t["mu"]**2 - 1
    return t


@pytest.mark.parametrize("params,why", [
    ([(0, "curvature")], "surface 0"),
    ([(5, "curvature")], "past the last surface"),
    ([(1.5, "curvature")], "not an integer"),
    ([(1, "wobble")], "unknown kind"),
    ([(1, "asph10")], "unknown kind"),
    ([(2, "distance")], "decentred"),
    ([(3, "tilt_x")], "already rotated"),
    ([(4, "index")], "last surface"),
    ([(2, "index")], "next surface is a mirror"),
    ([(1, "index")], "mu = 1 and n = n0 after it"),
])
def test_refusals(params, why):
    t = _table()
    t["offset"][:, 1, 0] = .1
    t["flags"][:, 2] |= 1
    t["mu"][:, 2] = -1
    if why == "mu = 1 and n = n0 after it":
        t["mu"][:, 1], t["n"][:, 1] = 1., t["n0"][:, 1]
    with pytest.raises(ValueError):
        perturbed_tables(t, params, np.zeros((3, len(params))))


def test_refuses_bad_delta_shape():
    with pytest.raises(ValueError):
        perturbed_tables(_table(), [(1, "curvature")], np.zeros((3, 2)))


def test_asph_makes_newton_surface_only_when_moved():
    t = _table()
    got = perturbed_tables(t, [(1, "asph3")], [[0.], [1e-9]])
    assert (got["n_asph"][0, :, 0] == -1).all()
    assert (got["n_asph"][1, :, 0] == 4).all()
    assert got["asph"][1, 0, 0, 3] == 1e-9 and got["dasph"][1, 0, 0, 3] == 8e-9


def test_tilt_below_rayopts_tolerance_is_no_rotation():
    got = perturbed_tables(_table(), [(2, "tilt_x")], [[1e-9], [1e-3]])
    assert got["flags"][0, 0, 1] == 0 and got["flags"][1, 0, 1] == 1
    c, s = np.cos(1e-3), np.sin(1e-3)
    assert np.allclose(got["rot"][1, 0, 1].reshape(3, 3), [[1, 0, 0], [0, c, s], [0, -s, c]],
                       rtol=0, atol=1e-15) or np.allclose(
        got["rot"][1, 0, 1].reshape(3, 3), [[1, 0, 0], [0, c, -s], [0, s, c]], rtol=0, atol=1e-15)


def test_delta_generators():
    tol = np.array([1e-3, 2e-2, .5])
    d = sensitivity_deltas(tol)
    assert d.shape == (7, 3)
    assert (d[0] == 0).all()
    for p in range(3):
        assert d[1 + 2*p, p] == tol[p] and d[2 + 2*p, p] == -tol[p]
        assert np.count_nonzero(d[1 + 2*p]) == 1 and np.count_nonzero(d[2 + 2*p]) == 1
    m = monte_carlo_deltas(tol, 1000, seed=1)
    assert m.shape == (1000, 3)
    assert (np.abs(m) <= tol).all()
    assert np.array_equal(m, monte_carlo_deltas(tol, 1000, seed=1))
    assert not np.array_equal(m, monte_carlo_deltas(tol, 1000, seed=2))


@needs_ref
@pytest.mark.parametrize("name", ["cooke", "double_gauss"])
def test_oracle_rms_matches_reference(R, name):
    """the oracle's finite-ray rms of a perturbed lens is the reference's
    GeometricTrace.rms of the perturbed System fed the same launch rays,
    wherever no ray is lost"""
    s = build(R, name)
    nom = tables(s)
    params = [(1, "curvature"), (2, "distance")]
    d = np.array([[0., 0.], [1e-3, 0.], [0., -3e-2]])
    got = perturbed_tables(nom, params, d)
    l = s.wavelengths[0]
    z, p = s.pupil((0, .2), l=l)
    y0, u0 = s.aim((0, .2), .7*tolerance_oracle.disc(200, 3), z, p)
    rot0 = pack_system(s, l, 1, None)[2]
    checked = 0
    for v, row in enumerate(d):
        ref = copy.deepcopy(s)
        for (j, kind), dv in zip(params, row):
            if dv:
                apply(ref, j, kind, dv)
        g = R.GeometricTrace(ref)
        g.rays_given(y0, u0, l)
        g.propagate(clip=True)
        want = g.rms()
        c = np.r_[g.y[-1, 0, :2], 0., 0.]                      # about a ray in the spot
        m = tolerance_oracle.item_sums(got[v, 0], rot0, y0, u0, True, c)[0]
        rms = tolerance_oracle.rms_finite(m)
        assert abs(rms - tolerance_oracle.rms_finite_rows(g.y[-1])) <= 1e-12*rms
        if np.isfinite(want):
            assert m[4] == m[5]
            assert abs(rms - want) <= 1e-12*want, (name, v, rms, want)
            checked += 1
    assert checked
