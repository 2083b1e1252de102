"""spot_jacobian and optimize_spot (rayopt_b200/optimize.py) on the device,
on the reference's own Cooke triplet.  Needs a GPU and the staged reference."""
import copy
import warnings

import numpy as np
import pytest

import jac_oracle
import ref_shim
from rayopt_b200 import optimize as opt
from rayopt_b200.engine import Engine
from rayopt_b200.surface_table import pack_system
from rayopt_b200.tolerance import monte_carlo_deltas, record_tangents

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not ref_shim.available(), reason="no reference tree staged")]

HEIGHTS = (0., .7, 1.)


@pytest.fixture(scope="module")
def eng():
    e = Engine(0)
    yield e
    e.close()


def cooke():
    import yaml
    import systems_yaml
    warnings.simplefilter("ignore")
    np.seterr(all="ignore")
    R = ref_shim.load()
    s = R.System(**yaml.safe_load(systems_yaml.SYSTEMS["cooke"]))
    s.update()
    s.paraxial.refocus()
    return s


def cooke_params(s):
    t = pack_system(s, s.wavelengths[0], 1, None)[0]
    cs = [j for j in range(1, len(t) + 1) if t["c"][j - 1] != 0][:6]
    return [(j, "curvature") for j in cs] + [(len(t), "distance")]


def tables_of(s):
    return np.stack([pack_system(s, l, 1, None, n0=s.refractive_index(l, 0))[0]
                     for l in s.wavelengths])


def test_gradient_matches_differences(eng):
    """grad rms^2 against Richardson central differences of the fixed-bundle
    rms^2 (rtx_trace_reduce_many on perturbed_tables, clip off), 1e-6 of the
    bundle's largest gradient"""
    s = cooke()
    params = cooke_params(s)
    wl = [s.wavelengths[0]]
    res = opt.spot_jacobian(copy.deepcopy(s), params, HEIGHTS, wl, nrays=400, engine=eng)
    B = opt._Bundles(copy.deepcopy(s), HEIGHTS, wl, 400, "hexapolar", eng, False)
    try:
        P = len(params)
        fd = np.zeros((len(HEIGHTS), P))
        for p, (j, kind) in enumerate(params):
            h = 1e-5 if kind == "curvature" else 1e-3
            D = []
            for x in (h, h/2):
                d = np.zeros((2, P))
                d[0, p], d[1, p] = x, -x
                rms2 = []
                for b in range(len(HEIGHTS)):
                    w = np.zeros(len(HEIGHTS))
                    w[b] = 1
                    rms2.append(opt._merits(eng, B, params, d, w, False, False))
                rms2 = np.array(rms2)
                D.append((rms2[:, 0] - rms2[:, 1])/(2*x))
            fd[:, p] = (4*D[1] - D[0])/3
        # the host Gram of the oracle's J of the same rays
        moves = record_tangents(B.nominal, params)
        for b, (y, u) in enumerate(B.rays):
            mv = [[(r, rec[0]) for r, rec in m] for m in moves]
            q, J = jac_oracle.trace(B.nominal[0], y.download(), u.download(), mv, rot0=B.rot0)
            ok = np.isfinite(q).all(1) & np.isfinite(J).all((0, 1))
            n = ok.sum()
            Jc = (J[:, :, ok] - J[:, :, ok].mean(2, keepdims=True))/np.sqrt(n)
            gram = np.einsum("pxk,qxk->pq", Jc, Jc)
            got = res["JtJ"][b, 0]
            assert np.abs(got - gram).max() <= 1e-10*np.abs(gram).max(), b
    finally:
        B.close()
    g = res["grad"][:, 0]
    assert np.all(np.abs(g - fd) <= 1e-6*np.abs(fd).max(1, keepdims=True)), np.abs(g - fd).max()


def test_optimize_cooke(eng):
    s = cooke()
    params = cooke_params(s)
    before = tables_of(s).tobytes()
    wl = list(s.wavelengths)
    nominal = opt.optimize_spot(s, params, HEIGHTS, wl, iterations=0, nrays=400,
                                engine=eng)["merit"][0]
    # a Monte-Carlo-perturbed Cooke (curvatures only), optimised back
    d = monte_carlo_deltas([2e-3]*6 + [0.], 1, seed=3)[0]
    bad = opt.apply_deltas(copy.deepcopy(s), params, d)
    res = opt.optimize_spot(bad, params, HEIGHTS, wl, iterations=20, nrays=400, engine=eng)
    # the first step is the numpy LM step from the oracle's normal equations
    B = opt._Bundles(copy.deepcopy(bad), HEIGHTS, wl, 400, "hexapolar", eng, False)
    try:
        moves = record_tangents(B.nominal, params)
        JtJ, Jtr = 0, 0
        for b, (y, u) in enumerate(B.rays):
            w = b % len(wl)
            mv = [[(r, rec[w]) for r, rec in m] for m in moves]
            q, J = jac_oracle.trace(B.nominal[w], y.download(), u.download(), mv, rot0=B.rot0)
            ok = np.isfinite(q).all(1) & np.isfinite(J).all((0, 1))
            n = ok.sum()
            Jc = (J[:, :, ok] - J[:, :, ok].mean(2, keepdims=True))/np.sqrt(n)
            r = ((q[ok] - q[ok].mean(0))/np.sqrt(n)).T
            JtJ = JtJ + np.einsum("pxk,qxk->pq", Jc, Jc)
            Jtr = Jtr + np.einsum("pxk,xk->p", Jc, r)
    finally:
        B.close()
    assert res["lam"][0] > 0, "the first step was not accepted"
    want = opt.lm_step(JtJ, Jtr, res["lam"][0])
    assert np.abs(res["step"][0] - want).max() <= 1e-8*np.abs(want).max()
    acc = res["lam"] > 0
    assert np.all(res["trial"][acc] < res["merit"][:-1][acc])
    ratio = res["merit"][-1]/nominal
    print("perturbed %.4g -> %.4g, nominal %.4g, ratio %.3f after %d accepted steps"
          % (res["merit"][0], res["merit"][-1], nominal, ratio, acc.sum()))
    assert ratio <= 1.05
    assert tables_of(s).tobytes() == before
    assert tables_of(bad).tobytes() != tables_of(res["system"]).tobytes()
