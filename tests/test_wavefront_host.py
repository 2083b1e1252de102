"""Host side of the wavefront derivatives (no GPU): the one-component
Gauss-Newton formulas of optimize.gauss_newton_wavefront against the
residuals written out, the rtx_wavefront_sums row layout, the host chain
the device derivatives are checked against, and the refusals that come
before any device work."""
import copy
import warnings

import numpy as np
import pytest

import epi_oracle
import np_oracle
import ref_shim
import test_jacobian_host as jac_host
import wavefront_chain
import wavefront_oracle
from conftest import load_systems
from rayopt_b200 import optimize as opt
from rayopt_b200.engine import wavefront_sums_unpack
from rayopt_b200.rays import aim_infinite, disc
from rayopt_b200.tolerance import record_tangents

ORACLE_RTOL = 1e-9   # largest error seen: 1.1e-10 of the column scale (double_gauss)


def sums_row(A, dA, a0):
    """rtx_wavefront_sums' row of host A (N,), dA (P, N), written out"""
    P = dA.shape[0]
    d = A - a0
    ok = np.isfinite(d) & np.isfinite(dA).all(0)
    bad = np.isfinite(d) & ~np.isfinite(dA).all(0)
    d, J = d[ok], dA[:, ok]
    iu = np.triu_indices(P)
    return np.r_[ok.sum(), d.sum(), (d*d).sum(), J.sum(1), J @ d, (J @ J.T)[iu], bad.sum()]


def test_unpack_layout():
    rng = np.random.default_rng(1)
    P = 5
    A, dA = rng.normal(size=100), rng.normal(size=(P, 100))
    row = sums_row(A, dA, .3)
    assert len(row) == 4 + 2*P + P*(P + 1)//2
    s = wavefront_sums_unpack(row, P)
    assert np.allclose(s["K"], dA @ dA.T) and np.allclose(s["H"], dA @ (A - .3))
    assert s["n"] == 100 and s["bad"] == 0


@pytest.mark.parametrize("P", [0, 1, 4])
def test_gauss_newton_formulas(P):
    """rms^2, JtJ and Jtr from the sums equal those of the residuals
    r_k = (W_k - Wbar)/sqrt(n), W = -(A - a_ref)/wl, and their Jacobian"""
    rng = np.random.default_rng(P)
    N, wl = 3000, 5.5e-4
    A = 100 + rng.normal(0, 1e-3, N)
    dA = rng.normal(0, 1e-2, (P, N))
    A[7] = np.nan
    if P:
        dA[0, 9] = np.inf
    rms2, JtJ, Jtr, grad = opt.gauss_newton_wavefront(sums_row(A, dA, A[0]), P, wl)
    ok = np.isfinite(A) & np.isfinite(dA).all(0)
    W = -(A[ok] - A[0])/wl
    n = ok.sum()
    r = (W - W.mean())/np.sqrt(n)
    J = -(dA[:, ok] - dA[:, ok].mean(1)[:, None]).T/(wl*np.sqrt(n))
    assert np.isclose(rms2, r @ r, rtol=1e-9)
    assert np.allclose(JtJ, J.T @ J, rtol=1e-9, atol=0)
    assert np.allclose(Jtr, J.T @ r, rtol=1e-9, atol=1e-12*np.abs(J.T @ r).max(initial=0))
    assert np.allclose(grad, 2*Jtr)


def test_chain_is_the_device_epilogue():
    """the host chain in FP64 is epi_oracle.opd_epilogue of np_oracle's march
    (the restatement of rtx_trace_opd) to rounding, and in long double
    agrees with it to 1e-12 of the path"""
    ent = load_systems()["cooke"]
    aim = ent["aim"][0][2]
    y0, u0 = aim_infinite(aim["field"], disc(32, 1)*.8, aim["z"], aim["p"], ent["object_angle"])
    table = ent["tables"][0][:-1]
    spec = dict(y0_ref=y0[0], u0_ref=u0[0], n0=1., n_after=1., M=rot(.02, .01),
                d=np.array([.1, -.2, -3.]), radius=-80., infinite=1)
    Y, U, _, T = np_oracle.trace(table, y0, u0)
    want = epi_oracle.opd_epilogue(y0, Y[-1], U[-1], T.cumsum(0)[-1], spec)[0]
    for dt, tol in ((np.float64, 1e-14), (np.longdouble, 1e-12)):
        A = np.asarray(wavefront_chain.path(table, y0, u0, spec, dtype=dt), np.float64)
        assert np.abs(A - want).max() <= tol*np.abs(want).max(), dt


def rot(a, b):
    """a frame change: rotations by a about x and b about y"""
    ca, sa, cb, sb = np.cos(a), np.sin(a), np.cos(b), np.sin(b)
    return np.array([[1, 0, 0], [0, ca, -sa], [0, sa, ca]]) @ np.array(
        [[cb, 0, sb], [0, 1, 0], [-sb, 0, cb]])


# (fixture, [(j, kind)] on the OPD march table = the fixture's table minus
# its last row): every kind, analytic and Newton surfaces, a mirror,
# rotated rows; the specs add a frame change, a finite object and a moving
# sphere centre and index
ORACLE_CASES = {
    "cooke": [(1, "curvature"), (2, "curvature"), (3, "conic"), (2, "distance"),
              (4, "asph0"), (3, "asph2"), (2, "tilt_x"), (6, "tilt_y"), (1, "index"),
              (3, "index"), (7, "distance")],
    "cooke_asph": [(2, "asph1"), (3, "curvature"), (1, "curvature"), (6, "distance"),
                   (1, "tilt_y"), (2, "conic"), (3, "index")],
    "double_gauss": [(3, "curvature"), (6, "distance"), (7, "conic"), (4, "tilt_x"),
                     (1, "index"), (8, "asph0"), (11, "distance")],
    "mirror_folded": [(1, "curvature"), (1, "conic"), (1, "asph0")],
    "tilted_start3": [(1, "curvature"), (1, "conic")],
    "tilted_clip0": [(1, "curvature"), (3, "curvature"), (1, "index"), (3, "distance")],
}


def opd_fixture(name, infinite=1, M=None):
    table, rot0, y0, u0 = jac_host.fixture(name)
    with np.errstate(all="ignore"):
        Y = np_oracle.trace(table, y0[:1], u0[:1], rot0=rot0)[0][-1, 0]
    spec = dict(y0_ref=y0[0], u0_ref=u0[0], n0=1., n_after=float(table["n"][-2]),
                M=np.eye(3) if M is None else M, d=-np.asarray(table["offset"][-1], float) - Y,
                radius=-60., infinite=infinite)
    return table[:-1], rot0, y0, u0, spec


def check_oracle(table, rot0, y0, u0, spec, params, dopd, rtol=ORACLE_RTOL):
    moves = record_tangents(table, params)
    with np.errstate(all="ignore"):
        A, dA = wavefront_oracle.trace_opd(table, y0, u0, moves, spec, dopd, rot0=rot0)
    assert np.array_equal(np.isnan(A), np.isnan(wavefront_chain.path(table, y0, u0, spec,
                                                                      rot0=rot0,
                                                                      dtype=np.float64)))
    cols = []
    for p, (j, kind) in enumerate(params):
        fd = wavefront_chain.march_column(table, y0, u0, spec, j, kind,
                                          jac_host.step(table, j, kind), rot0=rot0,
                                          dopd=dopd[p])
        ok = np.isfinite(fd) & np.isfinite(dA[p])
        assert ok.mean() > .5, (j, kind)
        cols.append((j, kind, ok, fd))
    top = max(np.abs(dA[p, ok]).max() for p, (_, _, ok, _) in enumerate(cols))
    worst = 0.
    for p, (j, kind, ok, fd) in enumerate(cols):
        # a column far below the others is held to 1e-3 of the largest
        scale = max(np.abs(dA[p, ok]).max(), 1e-3*top)
        err = np.abs(dA[p, ok] - fd[ok]).max()/scale
        worst = max(worst, err)
        assert err <= rtol, (j, kind, err)
    return worst


@pytest.mark.parametrize("name", list(ORACLE_CASES))
def test_oracle_against_differences(name):
    table, rot0, y0, u0, spec = opd_fixture(name)
    params = [p for p in ORACLE_CASES[name] if p[0] <= len(table)]
    dopd = np.zeros((len(params), 4))
    dopd[0] = [.02, -.01, .03, .1]
    print("%s: %.1e" % (name, check_oracle(table, rot0, y0, u0, spec, params, dopd)))


def test_oracle_frame_change_finite_object_rot0():
    """a frame change M, an object at a finite distance (no input plane) and
    a launch rotation"""
    table, _, y0, u0, spec = opd_fixture("cooke", infinite=0, M=rot(.03, -.02))
    a = .01
    rot0 = np.array([[1, 0, 0], [0, np.cos(a), -np.sin(a)], [0, np.sin(a), np.cos(a)]])
    params = [(1, "curvature"), (4, "distance"), (3, "tilt_x"), (3, "index")]
    dopd = np.random.default_rng(2).normal(0, .05, (4, 4))
    check_oracle(table, rot0, y0, u0, spec, params, dopd)


def cooke():
    import yaml
    import systems_yaml
    warnings.simplefilter("ignore")
    R = ref_shim.load()
    s = R.System(**yaml.safe_load(systems_yaml.SYSTEMS["cooke"]))
    s.update()
    return s


@pytest.mark.skipif(not ref_shim.available(), reason="no reference tree")
def test_refusals_before_device_work():
    """shape parameters of the image surface and tilts of the last two
    surfaces are refused before anything is aimed (engine=None would need
    a device)"""
    s = cooke()
    L = len(s)
    for params in ([(L - 1, "curvature")], [(L - 1, "conic")], [(L - 1, "asph0")],
                   [(L - 2, "tilt_x")], [(L - 1, "tilt_y")], [(L - 1, "index")],
                   [(1, "curvature"), (0, "distance")]):
        with pytest.raises(ValueError):
            opt.wavefront_jacobian(copy.deepcopy(s), params, engine=object())
    with pytest.raises(ValueError):
        opt.optimize_wavefront(copy.deepcopy(s), [(1, "tilt_x")], engine=object())
    with pytest.raises(ValueError):
        opt.optimize_wavefront(copy.deepcopy(s), [(L - 1, "curvature")], engine=object())
