"""rtx_otf_jacobian_sums, mtf_jacobian and optimize_mtf on the device: the
kernel against the long-double oracle (tests/otf_jac_oracle.py) within the
bound of include/rtx.h, against rtx_otf_rows on traced lenses, determinism,
guard bands and refusals, and the optimiser end to end on the reference's
Cooke triplet."""
import copy
import warnings

import numpy as np
import pytest

import otf_jac_oracle as oj
import ref_shim
from conftest import load_systems
from rayopt_b200 import optimize as opt
from rayopt_b200._lib import ptr
from rayopt_b200.engine import Engine, otf_bound, otf_spec
from rayopt_b200.mtf import geometric_mtf
from rayopt_b200.tolerance import monte_carlo_deltas, record_tangents
from test_gpu_jacobian import CASES, case_params, get_case, same_bits

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    e = Engine(0)
    yield e
    e.close()


def synthetic(N, P, F, seed, ld=None, qstride=2):
    rng = np.random.default_rng(seed)
    q = rng.normal(0, .03, (max(N, 1), qstride)) + [.5, -.2, 0.][:qstride]
    ld = ld or max(32, -(-N//32)*32)
    J = rng.normal(0, 2., (max(P, 1), 2, ld))
    if N > 4:
        k = rng.choice(N, min(N//7 + 1, 40), replace=False)
        q[k[0::4], 0] = np.nan
        q[k[1::4], 1] = np.inf
        J[rng.integers(0, max(P, 1), len(k[2::4])), rng.integers(0, 2, len(k[2::4])), k[2::4]] = np.nan
        J[0, 1, k[3::4]] = -np.inf
    nu = np.r_[0., rng.uniform(-60, 120, F - 1)] if F > 1 else np.array([33.3])
    return q, J, nu, np.array([.5002, -.2001])


def device_sums(eng, q, J, nu, c, N, P):
    dq = eng.to_device(q)
    dJ = eng.to_device(J[:P]) if P else None
    try:
        return eng.otf_jacobian_sums(dq, dJ, nu, c, N=N)
    finally:
        dq.free()
        if dJ is not None:
            dJ.free()


def check(got, r, N, chunks=1):
    assert got["n"] == r["n"] and got["bad"] == r["bad"]
    bS, bdS = oj.device_bound(N, r["phi"], chunks)
    e = oj.oracle_error(r["n"], r["phi"])
    tol = (bS + e)*r["n"]
    assert np.all(np.abs(got["S"].real - r["Sre"].astype(float)) <= tol)
    assert np.all(np.abs(got["S"].imag - r["Sim"].astype(float)) <= tol)
    tol = (bdS + e)*r["absJ"]
    assert np.all(np.abs(got["dS"].real - r["dre"].astype(float)) <= tol)
    assert np.all(np.abs(got["dS"].imag - r["dim"].astype(float)) <= tol)


CASES_K = ([(N, 5, 7, 2) for N in (0, 1, 31, 32, 33, 4095, 4096, 4097, 16383, 16384, 16385)]
           + [(N, 0, 7, 3) for N in (0, 1, 33, 16385)]
           + [(70001, 64, 7, 2), (70001, 1, 64, 3)]
           + [(3000, P, 64, 2) for P in (0, 1, 5, 17, 64)]
           + [(3000, 17, F, s) for F in (1, 7, 64, 256) for s in (2, 3)]
           + [(16385, 5, 256, 2)])


@pytest.mark.parametrize("N, P, F, qstride", CASES_K)
def test_kernel_matches_oracle(eng, N, P, F, qstride):
    q, J, nu, c = synthetic(N, P, F, seed=N + 7*P + F, qstride=qstride)
    got = device_sums(eng, q, J, nu, c, N, P)
    r = oj.sums(q[:N], J[:P, :, :N] if P else None, nu, c)
    check(got, r, N)
    assert got["S"].shape == (2, F) and got["dS"].shape == (P, 2, F)
    if P and N:
        # S does not depend on P where no ray is bad
        keep = np.isfinite(J[:P, :, :N]).all((0, 1))
        q2 = np.where(keep[:, None], q[:N], np.nan)
        a = device_sums(eng, q2, J, nu, c, N, P)
        b = device_sums(eng, q2, J, nu, c, N, 0)
        assert a["bad"] == 0 and same_bits(a["S"].view(float), b["S"].view(float))


# ---- on traced lenses, against rtx_otf_rows -----------------------------------
@pytest.mark.parametrize("exact", [True, False], ids=["exact", "fast"])
@pytest.mark.parametrize("name", list(CASES))
def test_traced_lenses_against_otf_rows(eng, name, exact):
    systems = load_systems()
    table, rot0, y0, u0, params = get_case(systems, name)
    params = case_params(table, params)
    moves = record_tangents(table, params)
    N = len(y0)
    dy, du = eng.to_device(y0), eng.to_device(u0)
    ld = max(64, -(-N//64)*64)
    Y, I = eng.empty((1, ld, 3)), eng.empty((1, ld, 3))
    try:
        q, J = eng.trace_jacobian(table, dy, du, moves, clip=True, rot0=rot0, exact=exact)
        eng.trace_device(table, dy, du, Y, None, I, None, N=N, ld=ld, clip=True, keep_last=True,
                         rot0=rot0, exact=exact)
        qh = q.download()
        fin = np.isfinite(qh).all(1)
        c = qh[fin].mean(0) if fin.any() else np.zeros(2)
        spread = np.abs(qh[fin] - c).max() if fin.any() else 1.
        dnu = 3/max(spread, 1e-9)/16
        F = 16
        nu = np.arange(F)*dnu
        a = eng.otf_jacobian_sums(q, J, nu, c)
        b = eng.otf_jacobian_sums(Y.rows(0), None, nu, c, N=N)
        S, count = eng.otf_rows(Y.rows(0), I.rows(0), otf_spec((0.,), dnu, F, c), N=N)
        Jh = J.download()[:, :, :N]
        q.free(), J.free()
    finally:
        for x in (dy, du, Y, I):
            x.free()
    assert a["n"] + a["bad"] == count[0] == b["n"]
    r = oj.sums(qh, Jh, nu, c)
    check(a, r, N)
    if a["bad"] == 0:
        assert same_bits(a["S"].view(float), b["S"].view(float))
        phi = r["phi"]
        tol = oj.device_bound(N, phi)[0]*a["n"] + otf_bound(otf_spec((0.,), dnu, F, c), N, count,
                                                              phi)[0]
        assert np.all(np.abs((a["S"] - S[0]).view(float)) <= tol)


# ---- determinism, guard bands, refusals ---------------------------------------
def test_deterministic_across_calls_contexts_and_chunks(eng):
    N, P, F = 70001, 9, 20
    q, J, nu, c = synthetic(N, P, F, seed=3)
    a = device_sums(eng, q, J, nu, c, N, P)
    b = device_sums(eng, q, J, nu, c, N, P)
    e2 = Engine(0)
    try:
        d = device_sums(e2, q, J, nu, c, N, P)
    finally:
        e2.close()
    assert a["out"].tobytes() == b["out"].tobytes() == d["out"].tobytes()
    r = oj.sums(q[:N], J[:, :, :N], nu, c)
    cut = 30011
    parts = [device_sums(eng, q[r0:r1], np.ascontiguousarray(J[:, :, r0:r1]), nu, c, r1 - r0, P)
             for r0, r1 in ((0, cut), (cut, N))]
    summed = dict(n=parts[0]["n"] + parts[1]["n"], bad=parts[0]["bad"] + parts[1]["bad"],
                  S=parts[0]["S"] + parts[1]["S"], dS=parts[0]["dS"] + parts[1]["dS"])
    check(summed, r, N, chunks=2)


def test_guard_bands_untouched(eng):
    N, P, F = 5000, 3, 9
    q, J, nu, c = synthetic(N, P, F, seed=5, ld=5056)
    dq = eng.to_device(np.r_[q[:N], np.full((64, 2), 7.)])
    dJ = eng.to_device(np.r_[J.reshape(-1), np.full(256, 7.)])
    W = 2 + 4*F + 4*P*F
    out = np.full(W + 64, 7.)
    assert eng.lib.rtx_otf_jacobian_sums(eng.ctx, N, P, dq.ptr, 2, dJ.ptr, 5056, ptr(c), F,
                                         ptr(nu), ptr(out[32:])) == 0
    assert (out[:32] == 7.).all() and (out[32 + W:] == 7.).all()
    assert (dq.download()[N:] == 7.).all() and (dJ.download()[-256:] == 7.).all()
    for x in (dq, dJ):
        x.free()


def test_refusals_launch_and_allocate_nothing(eng):
    q, J = eng.empty((100, 2)), eng.empty((2, 2, 128))
    nu, c, out = np.array([1., 2.]), np.zeros(2), np.zeros(2 + 4*256 + 4*65*256)
    L = eng.lib

    def call(**kw):
        a = dict(ctx=eng.ctx, N=100, P=2, q=q.ptr, qs=2, J=J.ptr, ld=128, c=ptr(c), F=2,
                 nu=ptr(nu), out=ptr(out))
        a.update(kw)
        return L.rtx_otf_jacobian_sums(*a.values())
    before = eng.launch_count()
    for kw in [dict(ctx=None), dict(out=None), dict(q=None), dict(J=None), dict(N=-1),
               dict(P=-1), dict(P=65), dict(qs=1), dict(qs=4), dict(ld=99), dict(F=0),
               dict(F=257), dict(nu=None), dict(nu=ptr(np.array([1., np.nan]))),
               dict(nu=ptr(np.array([np.inf, 1.]))), dict(c=ptr(np.array([0., np.inf])))]:
        assert call(**kw) == -1, kw
    assert eng.launch_count() == before
    # what is allowed: J NULL with P = 0, q NULL with N = 0, ld < N with P = 0
    assert call(P=0, J=None, ld=0) == 0 and call(N=0, q=None, J=None) == 0
    with pytest.raises(ValueError):
        eng.otf_jacobian_sums(q, J, [])
    with pytest.raises(ValueError):
        eng.otf_jacobian_sums(q, J, [np.nan])
    q.free(), J.free()


# ---- end to end on the reference's Cooke triplet ------------------------------
needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="no reference tree staged")
HEIGHTS = (0., .7, 1.)


def cooke():
    from test_gpu_optimize import cooke as c
    return c()


def params_of(s):
    from test_gpu_optimize import cooke_params
    return cooke_params(s)


def freqs_of(s, F=4):
    from rayopt_b200.mtf import default_dnu
    return np.arange(1, F + 1)*default_dnu(s, 8)


@needs_ref
def test_mtf_equals_geometric_mtf(eng):
    s = cooke()
    dnu = freqs_of(s)[0]
    res = opt.mtf_jacobian(copy.deepcopy(s), params_of(s), np.arange(8)*dnu, HEIGHTS,
                           nrays=2000, engine=eng)
    g = geometric_mtf(copy.deepcopy(s), HEIGHTS, nrays=2000, defocus=(0.,), dnu=dnu, nfreq=8,
                      engine=eng)
    assert (res["bad"] == 0).all() and np.array_equal(res["n"], g["count"][:, :, 0])
    assert np.allclose(res["mtf"], g["mtf"][:, :, 0], rtol=0, atol=1e-11)
    assert np.allclose(res["poly_mtf"], np.abs(g["poly"][:, 0]), rtol=0, atol=1e-11)


@needs_ref
def test_gradient_matches_trial_scorer(eng):
    """poly_grad against Richardson differences of the trial scorer's
    polychromatic MTF on the same bundles, 1e-6 of the largest gradient;
    clip off, so that no ray is lost between the variants"""
    s = cooke()
    params = params_of(s)
    nu = freqs_of(s)
    res = opt.mtf_jacobian(copy.deepcopy(s), params, nu, HEIGHTS, nrays=600, clip=False,
                           engine=eng)
    B = opt._Bundles(copy.deepcopy(s), HEIGHTS, s.wavelengths, 600, "hexapolar", eng, False)
    sw = np.ones(len(s.wavelengths))
    try:
        M0 = opt._trial_mtf(eng, B, params, np.zeros((1, len(params))), nu, sw, False, False)[0]
        assert np.allclose(M0, res["poly_mtf"], rtol=0, atol=1e-12)
        for p in range(len(params)):
            g = res["poly_grad"][..., p]
            scale = np.nanmax(np.abs(g))
            h = 1e-3/max(scale, 1.)
            d = np.zeros((4, len(params)))
            d[:, p] = [h, -h, h/2, -h/2]
            M = opt._trial_mtf(eng, B, params, d, nu, sw, False, False)
            fd = (4*(M[2] - M[3])/h - (M[0] - M[1])/(2*h))/3
            ok = np.isfinite(g)
            assert ok.any() and np.abs(g[ok] - fd[ok]).max() <= 1e-6*scale, p
    finally:
        B.close()


def oracle_normal(eng, s, params, nu, targets):
    """mtf_normal of the oracle's poly MTF and gradient (jac_oracle and
    otf_jac_oracle on the downloaded launch rays of the same bundles)"""
    import jac_oracle
    B = opt._Bundles(copy.deepcopy(s), HEIGHTS, s.wavelengths, 600, "hexapolar", eng, False)
    W, P, F = B.W, len(params), len(nu)
    try:
        moves = record_tangents(B.nominal, params)
        rows = []
        for b, (y, u) in enumerate(B.rays):
            w = b % W
            mv = [[(r, rec[w]) for r, rec in m] for m in moves]
            with np.errstate(all="ignore"):
                q, J = jac_oracle.trace(B.nominal[w], y.download(), u.download(), mv, clip=True,
                                        rot0=B.rot0)
            r = oj.sums(q, J, nu, B.centers[b - w, :2])
            row = np.zeros(2 + 4*F + 4*P*F)
            row[0], row[-1] = r["n"], r["bad"]
            row[1:1 + 4*F] = np.stack([r["Sre"], r["Sim"]], -1).astype(float).reshape(-1)
            row[1 + 4*F:-1] = np.stack([r["dre"], r["dim"]], -1).astype(float).reshape(-1)
            rows.append(row)
    finally:
        B.close()
    res = opt._mtf_result(np.array(rows), len(HEIGHTS), W, P, F, np.ones(W))
    return opt.mtf_normal(res["poly_mtf"], res["poly_grad"], targets, 1.), res["poly_mtf"]


@needs_ref
def test_optimize_mtf(eng):
    warnings.simplefilter("ignore")
    s = cooke()
    params = params_of(s)
    nu = freqs_of(s)
    # a Monte-Carlo-perturbed Cooke (curvatures only)
    d = monte_carlo_deltas([2e-3]*(len(params) - 1) + [0.], 1, seed=3)[0]
    bad = opt.apply_deltas(copy.deepcopy(s), params, d)
    keep = copy.deepcopy(bad)
    res = opt.optimize_mtf(bad, params, nu, 1., HEIGHTS, iterations=3, damping=1., nrays=600,
                           engine=eng)
    # the caller's System is unchanged
    for a, b in zip(keep, bad):
        assert a.distance == b.distance and a.curvature == b.curvature
    # every accepted trial lowers the merit it was scored against
    acc = res["lam"] > 0
    assert acc[0]
    assert np.all(res["trial"][acc] < res["merit"][:-1][acc])
    # the first step is lm_step on the oracle's normal equations
    (JtJ, Jtr), M0 = oracle_normal(eng, bad, params, nu, 1.)
    want = opt.lm_step(JtJ, Jtr, res["lam"][0])
    assert np.allclose(res["step"][0], want, rtol=0, atol=1e-8*np.abs(want).max())
    assert np.isclose(res["merit"][0], ((1 - M0)**2).sum(), rtol=1e-10)
    # the optimised lens has a higher polychromatic MTF at the chosen frequencies
    before = opt.mtf_jacobian(copy.deepcopy(bad), params, nu, HEIGHTS, nrays=600, engine=eng)
    after = opt.mtf_jacobian(res["system"], params, nu, HEIGHTS, nrays=600, engine=eng)
    assert after["poly_mtf"].mean() > before["poly_mtf"].mean()
    assert res["merit"][-1] < res["merit"][0]
