"""Host side of the lens-parameter Jacobian (no GPU): the forward-mode oracle
(oracle/jac_oracle.py) against Richardson-extrapolated central differences
of np_oracle.trace through perturbed_tables, record_tangents against the
records perturbed_tables builds, and the optimiser's host logic.

Bound asserted for the oracle: |J - J_fd| <= 1e-7 x the column's scale (the
largest |J| of that parameter and axis over the rays).  Largest error seen
on these fixtures: 1.3e-9 of the scale (the differences' own rounding)."""
import copy
import warnings

import numpy as np
import pytest

import jac_oracle
import np_oracle
import ref_shim
from conftest import load_golden, load_systems
from rayopt_b200.rays import aim_infinite, disc
from rayopt_b200.surface_table import SURFACE_DTYPE, pack_system
from rayopt_b200.tolerance import KINDS, perturbed_tables, record_tangents

ORACLE_RTOL = 1e-7

# (fixture, [(j, kind)]): every kind, analytic and Newton surfaces, a mirror,
# rotated rows and a launch rotation
CASES = {
    "cooke": [(1, "curvature"), (2, "curvature"), (3, "conic"), (2, "distance"), (8, "distance"),
              (4, "asph0"), (3, "asph2"), (2, "tilt_x"), (6, "tilt_y"), (1, "index"),
              (6, "index"), (7, "curvature")],
    "cooke_asph": [(2, "asph1"), (3, "curvature"), (1, "curvature"), (6, "distance"),
                   (1, "tilt_y"), (2, "conic"), (3, "index")],
    "double_gauss": [(3, "curvature"), (6, "distance"), (7, "conic"), (4, "tilt_x"),
                     (1, "index"), (8, "asph0"), (12, "distance")],
    "mirror_folded": [(1, "curvature"), (1, "conic"), (2, "distance"), (1, "asph0")],
    "tilted_start3": [(2, "curvature"), (1, "curvature"), (1, "conic")],
    "tilted_clip0": [(1, "curvature"), (3, "curvature"), (1, "index"), (3, "distance")],
}


def fixture(name):
    """(table, rot0, y0, u0) with unclipped rays"""
    if name in ("mirror_folded", "tilted_start3", "tilted_clip0"):
        c = load_golden(name)
        return c["table"], c["rot0"], c["y0"], c["u0"]
    ent = load_systems()[name]
    aim = ent["aim"][0][2]
    y0, u0 = aim_infinite(aim["field"], disc(64, 3)*.9, aim["z"], aim["p"], ent["object_angle"])
    return ent["tables"][0], None, y0, u0


def step(table, j, kind):
    t = table[j - 1]
    rmax = min(np.sqrt(t["radius2"]), 20.) if np.isfinite(t["radius2"]) else 10.
    if kind.startswith("asph"):
        return 1e-4/rmax**(2*int(kind[4:]) + 2)
    if kind == "curvature":     # about c = 0 the analytic root is noisy at 1e-9 (SURVEY A.5)
        return 1e-4 if t["c"] else 1e-3
    return {"conic": 1e-3, "distance": 1e-4, "tilt_x": 1e-5,
            "tilt_y": 1e-5, "index": 1e-5}[kind]


def q_of(table, rot0, y0, u0, j, kind, d):
    t = perturbed_tables(table, [(j, kind)], [[d]])[0, 0]
    return np_oracle.trace(t, y0, u0, rot0=rot0)[0][-1, :, :2]


def richardson(table, rot0, y0, u0, j, kind):
    h = step(table, j, kind)
    D = [(q_of(table, rot0, y0, u0, j, kind, x) - q_of(table, rot0, y0, u0, j, kind, -x))/(2*x)
         for x in (h, h/2)]
    return ((4*D[1] - D[0])/3).T


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_against_differences(name):
    table, rot0, y0, u0 = fixture(name)
    params = [p for p in CASES[name]]
    moves = record_tangents(table, params)
    with np.errstate(all="ignore"):
        q, J = jac_oracle.trace(table, y0, u0, moves, rot0=rot0)
        q0 = np_oracle.trace(table, y0, u0, rot0=rot0)[0][-1, :, :2]
    assert np.array_equal(q, q0, equal_nan=True)
    worst = 0.
    for p, (j, kind) in enumerate(params):
        with np.errstate(all="ignore"):
            fd = richardson(table, rot0, y0, u0, j, kind)
        ok = np.isfinite(fd).all(0) & np.isfinite(J[p]).all(0)
        assert ok.mean() > .5, (name, j, kind)
        for a in range(2):
            # a column that is zero (a move that cannot reach the image, e.g.
            # an unrefracting plane tilted) is compared against the
            # differences' own rounding, 1e3 eps |q| / h
            noise = 1e3*2.**-52*np.abs(q[ok]).max()/step(table, j, kind)
            scale = max(np.abs(J[p, a, ok]).max(), noise/ORACLE_RTOL)
            err = np.abs(J[p, a, ok] - fd[a, ok]).max()/scale
            worst = max(worst, err)
            assert err <= ORACLE_RTOL, (name, j, kind, a, err)
    print("%s: largest error %.1e of the column scale" % (name, worst))


def test_oracle_launch_rotation():
    """a rot0 launch on an unrotated lens (the tilted fixtures cover rotated rows)"""
    table, _, y0, u0 = fixture("cooke")
    a = .01
    rot0 = np.array([[1, 0, 0], [0, np.cos(a), -np.sin(a)], [0, np.sin(a), np.cos(a)]])
    params = [(1, "curvature"), (4, "distance"), (3, "tilt_x")]
    with np.errstate(all="ignore"):
        _, J = jac_oracle.trace(table, y0, u0, record_tangents(table, params), rot0=rot0)
        for p, (j, kind) in enumerate(params):
            fd = richardson(table, rot0, y0, u0, j, kind)
            scale = np.abs(J[p]).max(1)
            assert (np.abs(J[p] - fd).max(1) <= ORACLE_RTOL*scale).all(), (j, kind)


def test_clipped_direction_is_nan():
    table, rot0, y0, u0 = fixture("cooke")
    tab = table.copy()
    tab["radius2"][2] = 1.
    with np.errstate(all="ignore"):
        q, J = jac_oracle.trace(tab, y0, u0, record_tangents(tab, [(1, "curvature")]), clip=True)
        Y = np_oracle.trace(tab, y0, u0, clip=True)[0][-1, :, :2]
    assert np.array_equal(q, Y, equal_nan=True)
    assert np.isnan(q).any() and np.array_equal(np.isnan(J[0]), np.isnan(q.T))


# ---- record_tangents -----------------------------------------------------
def all_kinds(table):
    S = len(table)
    mu, n, n0 = table["mu"], table["n"], table["n0"]
    idx = [j for j in range(1, S) if mu[j - 1] not in (1, -1) and mu[j] not in (1, -1)
           and not (mu[j - 1] == 1 and n[j - 1] == n0[j - 1])]
    ps = [(2, k) for k in KINDS if k not in ("index",)]
    return ps + [(idx[0], "index")] if idx else ps


@pytest.mark.parametrize("name", ["cooke", "cooke_asph", "double_gauss"])
def test_record_tangents_match_perturbed_tables(name):
    """linear fields: the exact difference of perturbed_tables' records per
    unit delta; kc2, mu, muf, mu2m1 and rot within 1e-9 relative"""
    tables = np.stack(load_systems()[name]["tables"])
    params = all_kinds(tables[0])
    tans = record_tangents(tables, params)
    assert len(tans) == len(params)
    lin = ("c", "k", "offset", "asph", "dasph", "n", "n0")
    for p, (j, kind) in enumerate(params):
        h = 2.**-20
        d = np.zeros((2, len(params)))
        d[0, p], d[1, p] = h, -h
        pt = perturbed_tables(tables, params, d)
        diff = {f: (pt[0][f] - pt[1][f])/(2*h) for f in SURFACE_DTYPE.names
                if f not in ("flags", "n_asph", "sgn", "radius2")}
        got = {f: np.zeros_like(v) for f, v in diff.items()}
        for row, rec in tans[p]:
            for f in got:
                got[f][:, row] += rec[f]
        for f in diff:
            if kind in ("tilt_x", "tilt_y") and f == "rot":
                # the difference of a rotated and an unrotated record is not
                # the derivative: compare _rot_rxyz's central difference
                from rayopt_b200.tolerance import _rot_rxyz
                a = np.zeros(3)
                a[int(kind == "tilt_y")] = 1e-6
                want = ((_rot_rxyz(a) - _rot_rxyz(-a))/2e-6).reshape(9)
                assert np.abs(got[f][:, j - 1] - want).max() <= 1e-9, kind
                continue
            if f in lin:
                assert np.array_equal(got[f], diff[f]), (name, kind, f)
            else:
                scale = max(np.abs(diff[f]).max(), 1e-300)
                assert np.abs(got[f] - diff[f]).max() <= 1e-9*scale, (name, kind, f)


def test_record_tangents_refusals_equal_perturbed_tables():
    ent = load_systems()["cooke"]
    table = ent["tables"][0]
    rot = table.copy()
    rot["flags"][1] |= 1
    for tab, params in [(table, [(0, "curvature")]), (table, [(9, "curvature")]),
                        (table, [(1, "wobble")]), (table, [(8, "index")]),
                        (table, [(7, "index")]), (rot, [(2, "tilt_x")]),
                        (load_golden("tilted_clip0")["table"], [(3, "index")])]:
        with pytest.raises(ValueError) as a:
            perturbed_tables(tab, params, np.zeros((1, 1)))
        with pytest.raises(ValueError) as b:
            record_tangents(tab, params)
        assert str(a.value) == str(b.value)


# ---- optimiser host logic --------------------------------------------------
def test_lm_step_matches_lstsq():
    from rayopt_b200.optimize import lm_step
    rng = np.random.default_rng(1)
    Jm = rng.normal(size=(300, 7))*np.logspace(0, 3, 7)
    r = rng.normal(size=300)
    JtJ, Jtr = Jm.T @ Jm, Jm.T @ r
    for lam in (1e-3, .1, 10.):
        aug = np.vstack([Jm, np.sqrt(lam)*np.diag(np.sqrt(np.diag(JtJ)))])
        want = np.linalg.lstsq(aug, -np.r_[r, np.zeros(7)], rcond=None)[0]
        got = lm_step(JtJ, Jtr, lam)
        assert np.allclose(got, want, rtol=1e-9, atol=0), lam


def test_lm_step_zero_column():
    """a parameter that does not move the spot gets a zero step, the others
    the step without it"""
    from rayopt_b200.optimize import lm_step
    rng = np.random.default_rng(3)
    Jm = rng.normal(size=(200, 4))
    Jm[:, 2] = 0
    r = rng.normal(size=200)
    JtJ, Jtr = Jm.T @ Jm, Jm.T @ r
    got = lm_step(JtJ, Jtr, .1)
    keep = [0, 1, 3]
    assert got[2] == 0
    assert np.allclose(got[keep], lm_step(JtJ[np.ix_(keep, keep)], Jtr[keep], .1), rtol=1e-12)
    assert np.all(lm_step(np.zeros((3, 3)), np.zeros(3), 1.) == 0)


def test_gauss_newton_formulas():
    """the host formulas from synthetic sums equal the definitions"""
    from rayopt_b200.optimize import gauss_newton
    rng = np.random.default_rng(2)
    n, P = 50, 3
    q = rng.normal(size=(n, 2))
    J = rng.normal(size=(P, 2, n))
    c = np.array([.1, -.2])
    d = q - c
    out = np.r_[n, d.sum(0), (d*d).sum(), J.sum(2).reshape(-1),
                np.einsum("kx,pxk->p", d, J),
                np.einsum("pxk,qxk->pq", J, J)[np.triu_indices(P)], 0.]
    rms2, JtJ, Jtr, grad = gauss_newton(out, P)
    qb = q.mean(0)
    r = ((q - qb)/np.sqrt(n)).T                              # (2, n)
    Jr = (J - J.mean(2, keepdims=True))/np.sqrt(n)           # (P, 2, n)
    assert np.isclose(rms2, (r*r).sum(), rtol=1e-12)
    assert np.allclose(JtJ, np.einsum("pxk,qxk->pq", Jr, Jr), rtol=1e-12, atol=1e-14)
    assert np.allclose(Jtr, np.einsum("pxk,xk->p", Jr, r), rtol=1e-12, atol=1e-14)
    assert np.allclose(grad, 2*Jtr)


def test_refused_kinds():
    from rayopt_b200.optimize import optimize_spot
    for kind in ("tilt_x", "tilt_y", "index"):
        with pytest.raises(ValueError):
            optimize_spot(None, [(1, kind)])


needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="no reference tree staged")


@needs_ref
def test_applier_matches_perturbed_tables():
    """after each step, pack_system of the updated System is
    perturbed_tables(previous table, params, step) bit for bit"""
    import yaml
    import systems_yaml
    from rayopt_b200.optimize import apply_deltas
    warnings.simplefilter("ignore")
    R = ref_shim.load()
    s = R.System(**yaml.safe_load(systems_yaml.SYSTEMS["cooke"]))
    s.update()
    params = [(1, "curvature"), (3, "conic"), (4, "asph1"), (2, "distance"), (7, "distance")]
    rng = np.random.default_rng(4)
    for _ in range(3):
        prev = np.stack([pack_system(s, l, 1, None, n0=s.refractive_index(l, 0))[0]
                         for l in s.wavelengths])
        stp = rng.normal(size=len(params))*[1e-3, .1, 1e-7, 1e-2, 1e-2]
        s = apply_deltas(copy.deepcopy(s), params, stp)
        got = np.stack([pack_system(s, l, 1, None, n0=s.refractive_index(l, 0))[0]
                        for l in s.wavelengths])
        want = perturbed_tables(prev, params, stp[None])[0]
        assert got.tobytes() == want.tobytes()
