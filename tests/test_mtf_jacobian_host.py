"""Host side of the MTF derivatives (no GPU): the long-double OTF-derivative
oracle (tests/otf_jac_oracle.py) against mpmath and the OTF's identities,
the derivative chain d|S|/dp = Re(conj(S) dS)/|S| with the centre held
fixed against Richardson differences of the MTF of re-centred variants, and
the optimiser's host logic and refusals."""
import numpy as np
import pytest

import jac_oracle
import np_oracle
import otf_jac_oracle as oj
from conftest import load_systems
from rayopt_b200 import optimize as opt
from rayopt_b200.engine import otf_jacobian_sums_unpack
from rayopt_b200.rays import aim_infinite, disc
from rayopt_b200.tolerance import perturbed_tables, record_tangents

CHAIN_RTOL = 1e-7


def random_case(seed, N=40, P=3):
    rng = np.random.default_rng(seed)
    q = rng.normal(0, .05, (N, 2))
    J = rng.normal(0, 1, (P, 2, N))
    q[1, 0] = np.nan
    q[2, 1] = np.inf
    q[3] = -np.inf
    J[0, 1, 4] = np.nan          # finite q, non-finite derivatives: bad
    J[P - 1, 0, 5] = -np.inf
    J[1, 0, 2] = np.inf          # and with a non-finite q: not bad
    return q, J


def test_oracle_against_mpmath():
    mp = pytest.importorskip("mpmath")
    mp.mp.dps = 40
    q, J = random_case(1)
    c = np.array([.003, -.01])
    nu = np.array([0., 3.5, 17., -40.25])
    r = oj.sums(q, J, nu, c)
    d, inn, bad = oj.enter(q, J, c)
    assert r["n"] == inn.sum() == 35 and r["bad"] == bad.sum() == 2
    P, F = J.shape[0], len(nu)
    for a in range(2):
        for j in range(F):
            S = mp.mpc(0)
            dS = [mp.mpc(0)]*P
            for k in np.flatnonzero(inn):
                e = mp.exp(-2j*mp.pi*mp.mpf(nu[j])*mp.mpf(d[k, a]))
                S += e
                for p in range(P):
                    dS[p] += -2j*mp.pi*mp.mpf(nu[j])*mp.mpf(J[p, a, k])*e
            tol = oj.oracle_error(r["n"], r["phi"])
            assert abs(float(S.real) - float(r["Sre"][a, j])) <= tol*r["n"]
            assert abs(float(S.imag) - float(r["Sim"][a, j])) <= tol*r["n"]
            for p in range(P):
                u = max(r["absJ"][p, a, j], 1e-300)
                assert abs(float(dS[p].real) - float(r["dre"][p, a, j])) <= tol*u
                assert abs(float(dS[p].imag) - float(r["dim"][p, a, j])) <= tol*u


def test_oracle_identities():
    q, J = random_case(2, N=200, P=2)
    nu = np.array([0., 5., 12.])
    r = oj.sums(q, J, nu)
    n = r["n"]
    assert np.all(r["Sre"][:, 0] == n) and np.all(r["Sim"][:, 0] == 0)
    assert np.all(r["dre"][:, :, 0] == 0) and np.all(r["dim"][:, :, 0] == 0)
    # the shift theorem: S about c = exp(2 pi i nu c) S about 0 (c exact in d)
    c = np.array([.25, -.125])
    rc = oj.sums(q, J, nu, c)
    S0 = r["Sre"].astype(complex) + 1j*r["Sim"].astype(complex)
    Sc = rc["Sre"].astype(complex) + 1j*rc["Sim"].astype(complex)
    ph = np.exp(2j*np.pi*nu[None, :]*c[:, None])
    assert np.allclose(Sc, ph*S0, rtol=0, atol=1e-12*n)
    # and |S| and the MTF gradient do not change with the centre
    dS0 = r["dre"].astype(complex) + 1j*r["dim"].astype(complex)
    dSc = rc["dre"].astype(complex) + 1j*rc["dim"].astype(complex)
    m0, g0 = oj.mtf_grad(S0, dS0, n)
    mc, gc = oj.mtf_grad(Sc, dSc, n)
    assert np.allclose(m0, mc, rtol=0, atol=1e-13)
    assert np.allclose(g0[..., 1:], gc[..., 1:], rtol=0, atol=1e-11*np.abs(g0[..., 1:]).max())


# ---- the derivative chain on the golden lenses ------------------------------
LENSES = {
    "cooke": [(1, "curvature"), (3, "conic"), (4, "distance"), (6, "asph0"), (7, "distance")],
    "double_gauss": [(3, "curvature"), (6, "distance"), (7, "conic"), (12, "distance")],
}
FREQS = np.array([10., 25., 40.])


def _bundles(ent, field):
    """per wavelength: (table, y0, u0, chief y0, chief u0) at field index `field`"""
    out = []
    for li, table in enumerate(ent["tables"]):
        aim = ent["aim"][li][field]
        y0, u0 = aim_infinite(aim["field"], disc(48, 5)*.9, aim["z"], aim["p"], ent["object_angle"])
        cy, cu = aim_infinite(aim["field"], np.zeros((1, 2)), aim["z"], aim["p"],
                              ent["object_angle"])
        out.append((table, y0, u0, cy, cu))
    return out


def _otf_of(tables, bundles, c=None):
    """per wavelength (S complex (2, F), n) of the np_oracle trace of `tables`
    (W, S), about the wavelength-0 chief ray of those tables (or `c`)"""
    if c is None:
        _, _, _, cy, cu = bundles[0]
        c = np_oracle.trace(tables[0], cy, cu)[0][-1, 0, :2]
    res = []
    for w, (_, y0, u0, _, _) in enumerate(bundles):
        q = np_oracle.trace(tables[w], y0, u0)[0][-1, :, :2]
        r = oj.sums(q, None, FREQS, c)
        res.append((r["Sre"].astype(float) + 1j*r["Sim"].astype(float), r["n"]))
    return res


def _mtfs(res):
    mtf = np.array([abs(S)/n for S, n in res])
    poly = abs(sum(S/n for S, n in res)/len(res))
    return mtf, poly


@pytest.mark.parametrize("name", list(LENSES))
def test_chain_against_recentred_differences(name):
    """the exact chain (centre held fixed) equals differences of the MTF of
    variants each centred on its own chief ray: no centre term is missing"""
    ent = load_systems()[name]
    params = LENSES[name]
    bundles = _bundles(ent, 3)
    tables = np.stack(ent["tables"])
    moves = record_tangents(tables, params)
    _, _, _, cy, cu = bundles[0]
    c0 = np_oracle.trace(tables[0], cy, cu)[0][-1, 0, :2]
    otf, dotf, Js = [], [], []
    for w, (table, y0, u0, _, _) in enumerate(bundles):
        mv = [[(row, rec[w]) for row, rec in m] for m in moves]
        with np.errstate(all="ignore"):
            q, J = jac_oracle.trace(table, y0, u0, mv)
        r = oj.sums(q, J, FREQS, c0)
        assert r["bad"] == 0 and r["n"] == len(y0)
        Js.append(J)
        S = r["Sre"].astype(float) + 1j*r["Sim"].astype(float)
        dS = r["dre"].astype(float) + 1j*r["dim"].astype(float)
        otf.append(S/r["n"])
        dotf.append(dS/r["n"])
    Js = np.array(Js)
    mtf, grad = oj.mtf_grad(np.array(otf), np.array(dotf), 1.)       # (W, 2, F), (W, P, 2, F)
    poly = np.mean(otf, 0)
    pmtf, pgrad = oj.mtf_grad(poly, np.mean(dotf, 0), 1.)
    m0, p0 = _mtfs(_otf_of(tables, bundles))
    assert np.allclose(m0, mtf, rtol=0, atol=1e-12) and np.allclose(p0, pmtf, rtol=0, atol=1e-12)
    worst = 0.
    for p, (j, kind) in enumerate(params):
        # a step that moves the phase of the highest frequency by 0.01 rad
        h = .01/(2*np.pi*FREQS.max()*np.abs(Js[:, p]).max())

        def at(x):
            t = perturbed_tables(tables, [(j, kind)], [[x]])[0]
            return _mtfs(_otf_of(t, bundles))
        D = []
        for x in (h, h/2):
            (mp_, pp_), (mm_, pm_) = at(x), at(-x)
            D.append(((mp_ - mm_)/(2*x), (pp_ - pm_)/(2*x)))
        fd = (4*D[1][0] - D[0][0])/3, (4*D[1][1] - D[0][1])/3
        for got, want in ((grad[:, p], fd[0]), (pgrad[p], fd[1])):
            scale = np.abs(got).max()
            assert scale > 0, (j, kind)
            err = np.abs(got - want).max()/scale
            worst = max(worst, err)
            assert err <= CHAIN_RTOL, (name, j, kind, err)
    print("%s: largest error %.1e of the column scale" % (name, worst))


def test_centre_changes_only_the_phase():
    """a variant's S about its own chief ray and about the nominal one
    differ, their moduli do not: the premise of the chain test"""
    ent = load_systems()["cooke"]
    bundles = _bundles(ent, 5)
    tables = np.stack(ent["tables"])
    t = perturbed_tables(tables, [(4, "distance")], [[1e-3]])[0]
    free = _otf_of(t, bundles)
    _, _, _, cy, cu = bundles[0]
    fixed = _otf_of(t, bundles, np_oracle.trace(tables[0], cy, cu)[0][-1, 0, :2])
    for (Sa, _), (Sb, _) in zip(free, fixed):
        assert np.allclose(abs(Sa), abs(Sb), rtol=1e-12)
        assert not np.allclose(Sa, Sb, rtol=1e-6)


# ---- host logic -------------------------------------------------------------
def test_unpack_layout():
    P, F = 2, 3
    out = np.arange(2 + 4*F + 4*P*F, dtype=float)
    u = otf_jacobian_sums_unpack(out, P, F)
    assert u["n"] == 0 and u["bad"] == out[-1]
    a, j = 1, 2
    assert u["S"][a, j] == out[1 + 2*(a*F + j)] + 1j*out[2 + 2*(a*F + j)]
    p = 1
    e = 1 + 4*F + 2*((2*p + a)*F + j)
    assert u["dS"][p, a, j] == out[e] + 1j*out[e + 1]


def test_normal_equations_against_lstsq():
    rng = np.random.default_rng(3)
    H, F, P = 2, 4, 3
    g = rng.normal(size=(H, 2, F, P))
    M = rng.uniform(0, 1, (H, 2, F))
    t = rng.uniform(.5, 1, (H, 2, F))
    w = rng.uniform(.1, 2, (H, 2, F))
    g[0, 1, 2, 1] = np.nan                 # left out
    JtJ, Jtr = opt.mtf_normal(M, g, t, w)
    ok = np.isfinite(g).all(-1)
    A = np.sqrt(w[ok])[:, None]*g[ok]
    b = np.sqrt(w[ok])*(t - M)[ok]
    want = np.linalg.lstsq(A, b, rcond=None)[0]
    assert np.allclose(opt.lm_step(JtJ, Jtr, 0.), want, rtol=1e-10, atol=1e-12)
    assert np.allclose(Jtr, -(A.T @ b), rtol=1e-12)


def test_mtf_result_gradient_and_nan():
    """_mtf_result's MTF gradient against the complex chain, NaN where |S| = 0"""
    rng = np.random.default_rng(4)
    H, W, P, F = 2, 3, 2, 3
    rows = rng.normal(size=(H*W, 2 + 4*F + 4*P*F))
    rows[:, 0] = 100.
    rows[0, 1 + 2*(0*F + 1):3 + 2*(0*F + 1)] = 0.       # S[x, 1] = 0 for bundle 0
    sw = np.array([1., 2., 3.])
    res = opt._mtf_result(rows, H, W, P, F, sw)
    u = otf_jacobian_sums_unpack(rows[1], P, F)
    S, dS = u["S"]/100, u["dS"]/100
    g = (np.conj(S)[None]*dS).real/abs(S)[None]
    assert np.allclose(res["grad"][0, 1], np.moveaxis(g, 0, -1))
    assert np.isnan(res["grad"][0, 0, 0, 1]).all() and np.isfinite(res["grad"][0, 0, 1]).all()
    us = [otf_jacobian_sums_unpack(r, P, F) for r in rows[W:2*W]]
    poly = sum(s*x["S"]/100 for s, x in zip(sw, us))/sw.sum()
    dpoly = sum(s*x["dS"]/100 for s, x in zip(sw, us))/sw.sum()
    assert np.allclose(res["poly"][1], poly) and np.allclose(res["poly_mtf"][1], abs(poly))
    assert np.allclose(res["poly_grad"][1],
                       np.moveaxis((np.conj(poly)[None]*dpoly).real/abs(poly)[None], 0, -1))


class _NoEngine:
    def __getattr__(self, name):
        raise AssertionError("device work before the refusal: %s" % name)


@pytest.mark.parametrize("kw, msg", [
    (dict(freqs=[]), "frequencies"),
    (dict(freqs=[1., np.nan]), "frequencies"),
    (dict(freqs=np.arange(257.)), "frequencies"),
    (dict(targets=np.ones(5)), "targets"),
    (dict(weights=np.ones((4, 2, 3))), "weights"),
    (dict(params=[(1, "tilt_x")]), "cannot optimise"),
    (dict(params=[(1, "bogus")]), "cannot optimise"),
    (dict(spectral_weights=[1., 2.]), "spectral_weights"),
])
def test_refusals_before_device_work(kw, msg):
    system = _StubSystem()
    args = dict(params=[(1, "curvature")], freqs=[10., 20., 30.])
    args.update(kw)
    with pytest.raises(ValueError, match=msg):
        opt.optimize_mtf(system, engine=_NoEngine(), **args)


@pytest.mark.parametrize("kw, msg", [
    (dict(freqs=[np.inf]), "frequencies"),
    (dict(spectral_weights=[1.]), "spectral_weights"),
    (dict(chunk=0), "chunk"),
])
def test_jacobian_refusals_before_device_work(kw, msg):
    args = dict(params=[(1, "curvature")], freqs=[10.])
    args.update(kw)
    with pytest.raises(ValueError, match=msg):
        opt.mtf_jacobian(_StubSystem(), engine=_NoEngine(), **args)


class _StubSystem:
    """what the refusals read of a System: its wavelengths"""
    wavelengths = [5.8756e-07, 6.5627e-07, 4.8613e-07]
