"""rtx_trace_opd_jacobian, rtx_wavefront_sums, wavefront_jacobian and
optimize_wavefront on the device.  Needs a GPU.

A is compared with rtx_trace_opd's bit for bit.  dA is compared ray by ray
with the forward-mode oracle (tests/wavefront_oracle.py, itself held to
long-double Richardson differences in tests/test_wavefront_host.py) within
1e-10 of the column's scale, with test_gpu_jacobian.py's comparison and
exclusions.  The sums are compared with math.fsum of the device's own A and
dA within the bound include/rtx.h states."""
import copy
import math
import warnings

import numpy as np
import pytest

import np_oracle
import ref_shim
import wavefront_oracle
from conftest import load_golden, load_systems
from test_gpu_jacobian import CASES as JCASES
from test_gpu_jacobian import FAST_ULPS, case_params, check_against_oracle, edge_cases, get_case, \
    plates
from rayopt_b200.rays import aim_infinite, disc
from rayopt_b200.tolerance import record_tangents

pytestmark = pytest.mark.gpu

EPS = 2.0**-52


@pytest.fixture(scope="module")
def eng():
    from rayopt_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def same_bits(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and a[~na].tobytes() == b[~nb].tobytes()


def opd_case(name, n=64, seed=3, scale=.9, radius=None):
    """(full table, rot0, y0, u0, spec): the OPD march table is full[:-1];
    the sphere is centred on ray 0's image point"""
    if name in ("mirror_folded", "tilted_start3", "tilted_clip0"):
        c = load_golden(name)
        table, rot0, y0, u0 = c["table"], c["rot0"], c["y0"][:n], c["u0"][:n]
    else:
        ent = load_systems()[name]
        aim = ent["aim"][0][2]
        y0, u0 = aim_infinite(aim["field"], disc(n, seed)*scale, aim["z"], aim["p"],
                              ent["object_angle"])
        table, rot0 = ent["tables"][0], None
    with np.errstate(all="ignore"):
        Y = np_oracle.trace(table, y0[:1], u0[:1], rot0=rot0)[0][-1, 0]
    spec = dict(y0_ref=y0[0], u0_ref=u0[0], n0=1., n_after=float(table["n"][-2]), M=np.eye(3),
                d=-np.asarray(table["offset"][-1], float) - Y,
                radius=radius or 50.*np.sign(table["offset"][-1][2] or 1.), infinite=1)
    return table, rot0, np.ascontiguousarray(y0), np.ascontiguousarray(u0), spec


def device_opd_jac(eng, table, rot0, y0, u0, spec, moves, dopd, clip, exact):
    dy, du = eng.to_device(y0), eng.to_device(u0)
    try:
        A, dA = eng.trace_opd_jacobian(table, dy, du, spec, moves, dopd, clip=clip, rot0=rot0,
                                       exact=exact)
        N = len(y0)
        out = A.download(), dA.download()[:, :N], eng.wavefront_sums(A, dA)["bad"]
        A.free(), dA.free()
        return out
    finally:
        dy.free(), du.free()


def device_opd(eng, table, rot0, y0, u0, spec, clip, exact):
    dy, du = eng.to_device(y0), eng.to_device(u0)
    A, P = eng.empty((len(y0),)), eng.empty((len(y0), 3))
    try:
        eng.trace_opd(table, dy, du, spec, A, P, clip=clip, rot0=rot0, exact=exact)
        return A.download()
    finally:
        for a in (dy, du, A, P):
            a.free()


# ---- the primal is rtx_trace_opd's A -------------------------------------
@pytest.mark.parametrize("exact", [True, False], ids=["exact", "fast"])
@pytest.mark.parametrize("clip", [True, False], ids=["clip", "noclip"])
@pytest.mark.parametrize("N", [0, 1, 33, 513, 70001])
def test_A_is_trace_opd(eng, exact, clip, N):
    full, rot0, y0, u0, spec = opd_case("double_gauss", max(N, 1), seed=N, scale=1.05)
    table = full[:-1]
    cs = [j for j in range(1, len(table) + 1) if table["c"][j - 1] != 0]
    want = device_opd(eng, table, rot0, y0, u0, spec, clip, exact) if N else None
    for P in (1, 4, 5, 17, 64):
        params = [(cs[p % len(cs)], ("curvature", "conic", "distance")[p % 3]) for p in range(P)]
        moves = record_tangents(table, params)
        dopd = np.random.default_rng(P).normal(0, 1e-3, (P, 4))
        if not N:
            dy = eng.to_device(np.zeros((1, 3)))
            A, dA = eng.trace_opd_jacobian(table, dy, dy, spec, moves, dopd, N=0)
            for a in (A, dA, dy):
                a.free()
            continue
        A, dA, _ = device_opd_jac(eng, table, rot0, y0[:N], u0[:N], spec, moves, dopd, clip, exact)
        assert same_bits(A, want), P
        assert np.isnan(dA).any(0)[np.isnan(A)].all()


# ---- dA against the forward-mode oracle ------------------------------------
def check(A, dA, Ao, dAo, bad, **kw):
    """test_gpu_jacobian's ray-by-ray comparison (the NaN rule, the bad
    count, near-singular rays, JAC_RTOL = 1e-10 of the column scale) on the
    one-component path, given as two equal components"""
    two = lambda x, ax: np.stack([x, x], ax)  # noqa: E731
    return check_against_oracle(two(A, 1), two(dA, 1), two(Ao, 1), two(dAo, 1), bad, **kw)


def opd_spec_of(table, rot0, y0, u0, M=None, infinite=1):
    """an rtx_opd record for the march `table`: a sphere of radius -60
    centred near ray 0's intercept with the last row"""
    with np.errstate(all="ignore"):
        Y = np_oracle.trace(table, y0[:1], u0[:1], rot0=rot0)[0][-1, 0]
    Y = np.where(np.isfinite(Y), Y, 0.)
    return dict(y0_ref=y0[0], u0_ref=u0[0], n0=1., n_after=float(table["n"][-1]),
                M=np.eye(3) if M is None else M, d=np.array([0., 0., 5.]) - Y, radius=-60.,
                infinite=infinite)


@pytest.mark.parametrize("clip", [False, True], ids=["noclip", "clip"])
@pytest.mark.parametrize("exact", [True, False], ids=["exact", "fast"])
@pytest.mark.parametrize("name", list(JCASES))
def test_dA_matches_oracle(eng, name, exact, clip):
    """every lens of test_gpu_jacobian (the epilogue test systems with
    plates256, the Newton, mirror and tilted fixtures), its table the OPD
    march; a frame change, a moving sphere centre and index"""
    table, rot0, y0, u0, params = get_case(load_systems(), name)
    params = [p for p in case_params(table, params)
              if not (p[0] == len(table) and p[1].startswith("tilt"))]
    M = np.array([[1, 0, 0], [0, np.cos(.02), -np.sin(.02)], [0, np.sin(.02), np.cos(.02)]])
    spec = opd_spec_of(table, rot0, y0, u0, M)
    moves = record_tangents(table, params)
    dopd = np.random.default_rng(len(params)).normal(0, .05, (len(params), 4))
    A, dA, bad = device_opd_jac(eng, table, rot0, y0, u0, spec, moves, dopd, clip, exact)
    assert same_bits(A, device_opd(eng, table, rot0, y0, u0, spec, clip, exact))
    with np.errstate(all="ignore"):
        Ao, dAo = wavefront_oracle.trace_opd(table, y0, u0, moves, spec, dopd, clip=clip,
                                             rot0=rot0)
    print("%s: %.1e" % (name, check(A, dA, Ao, dAo, bad)))


def test_dA_finite_object(eng):
    table, rot0, y0, u0, _ = get_case(load_systems(), "cooke")
    spec = opd_spec_of(table, rot0, y0, u0, infinite=0)
    params = [(1, "curvature"), (3, "index"), (5, "distance")]
    moves = record_tangents(table, params)
    dopd = np.full((3, 4), .01)
    A, dA, bad = device_opd_jac(eng, table, rot0, y0, u0, spec, moves, dopd, True, False)
    with np.errstate(all="ignore"):
        Ao, dAo = wavefront_oracle.trace_opd(table, y0, u0, moves, spec, dopd, clip=True)
    check(A, dA, Ao, dAo, bad)


@pytest.mark.parametrize("exact", [True, False], ids=["exact", "fast"])
def test_dA_edge_bundles(eng, exact):
    """oracle/edge_bundles.py's decision-boundary bundles, with
    test_gpu_jacobian.test_J_edge_bundles' exclusions: rays whose kept/lost
    decision flips in fast mode, and rays within 1e10 ulps of a singular
    boundary, which are held to the NaN rule and the bad count only"""
    for name, c in edge_cases().items():
        params = [(1, "curvature"), (2, "distance"), (1, "asph0")]
        if c.table["c"][0] != 0:
            params.append((1, "conic"))
        moves = record_tangents(c.table, params)
        spec = opd_spec_of(c.table, None, c.y0, c.u0)
        dopd = np.zeros((len(params), 4))
        A, dA, bad = device_opd_jac(eng, c.table, None, c.y0, c.u0, spec, moves, dopd, c.clip,
                                    exact)
        with np.errstate(all="ignore"):
            Ao, dAo = wavefront_oracle.trace_opd(c.table, c.y0, c.u0, moves, spec, dopd,
                                                 clip=c.clip)
        flip = np.isfinite(A) != np.isfinite(Ao)
        if exact:
            assert not flip.any(), name
        else:
            assert (c.margin[flip] <= FAST_ULPS).all(), name
        singular = name.startswith(("tangent", "critical", "hemisphere", "paraboloid",
                                    "newton"))
        near = c.margin <= 1e10 if singular else np.zeros(len(A), bool)
        try:
            check(A, dA, Ao, dAo, bad, edge=True, exclude=flip, novalue=near)
        except AssertionError as e:
            raise AssertionError("%s: %s" % (name, e))


def test_plates256_n_after(eng):
    """a 92 KB table (past 48 KB of shared memory) and d(n_after) through dopd"""
    t, rot0, y0, u0 = plates()
    spec = opd_spec_of(t, None, y0, u0)
    params = [(1, "curvature"), (100, "distance"), (50, "index"), (7, "asph0")]
    moves = record_tangents(t, params)
    dopd = np.zeros((4, 4))
    dopd[2, 3] = .7
    A, dA, bad = device_opd_jac(eng, t, None, y0, u0, spec, moves, dopd, False, True)
    with np.errstate(all="ignore"):
        Ao, dAo = wavefront_oracle.trace_opd(t, y0, u0, moves, spec, dopd)
    check(A, dA, Ao, dAo, bad)


# ---- the sums ------------------------------------------------------------
@pytest.mark.parametrize("P", [0, 1, 6])
def test_sums_against_fsum(eng, P):
    full, rot0, y0, u0, spec = opd_case("cooke", 40000, seed=5, scale=1.1)
    table = full[:-1]
    params = [(1, "curvature"), (3, "conic"), (2, "distance"), (4, "asph0"), (1, "index"),
              (5, "curvature")][:max(P, 1)]
    moves = record_tangents(table, params)
    dy, du = eng.to_device(y0), eng.to_device(u0)
    try:
        A, dA = eng.trace_opd_jacobian(table, dy, du, spec, moves, np.zeros((len(moves), 4)),
                                       clip=True)
        a0 = float(A.download()[0])
        Ah, dAh = A.download(), dA.download()[:P, :len(y0)]
        dAp = None if P == 0 else dA
        s = eng.wavefront_sums(A, dAp, a0)
        s2 = eng.wavefront_sums(A, dAp, a0)
        assert s["out"].tobytes() == s2["out"].tobytes()
        # a second context, and the rays in two chunks added in order
        from rayopt_b200.engine import Engine
        e2 = Engine(0)
        try:
            A2, dA2 = e2.to_device(Ah), None if P == 0 else e2.to_device(dAh)
            assert e2.wavefront_sums(A2, dA2, a0)["out"].tobytes() == s["out"].tobytes()
            A2.free()
            if dA2 is not None:
                dA2.free()
        finally:
            e2.close()
        A.free(), dA.free()
    finally:
        dy.free(), du.free()
    d = Ah - a0
    ok = np.isfinite(d) & np.isfinite(dAh).all(0)
    d, J = d[ok], dAh[:, ok]
    N = len(y0)
    bound = (2*16384 + -(-N//16384))*EPS
    terms = [(np.ones_like(d),), (d,), (d*d,)] + [(J[a],) for a in range(P)] \
        + [(d*J[a],) for a in range(P)] \
        + [(J[a]*J[b],) for a in range(P) for b in range(a, P)]
    for e, (t,) in enumerate(terms):
        exact = math.fsum(t)
        assert abs(s["out"][e] - exact) <= bound*math.fsum(np.abs(t)) + 1e-300, e
    assert s["n"] == ok.sum()


# ---- guard bands and refusals --------------------------------------------
def test_guard_band_and_refusals(eng):
    from rayopt_b200 import _lib
    full, rot0, y0, u0, spec = opd_case("cooke", 100)
    table = full[:-1]
    moves = record_tangents(table, [(1, "curvature"), (2, "distance")])
    dy, du = eng.to_device(y0), eng.to_device(u0)
    try:
        # columns N .. ld-1 of dA and A past N are not written
        N, ld = 70, 96
        from rayopt_b200.engine import _moves, _opd_record
        P, first, rows, recs = _moves(dy, moves, len(table))
        A, dA = eng.to_device(np.full(100, 7.)), eng.to_device(np.full((2, ld), 7.))
        dopd = np.zeros((2, 4))
        rec = _opd_record(spec)
        call = lambda rec, dop: eng.lib.rtx_trace_opd_jacobian(  # noqa: E731
            eng.ctx, table.ctypes.data, len(table), None, 0, N, dy.ptr, du.ptr, 0,
            None if rec is None else rec.ctypes.data, 2, first.ctypes.data, rows.ctypes.data,
            recs.ctypes.data, None if dop is None else dop.ctypes.data, A.ptr, dA.ptr, ld, 0)
        assert call(rec, dopd) == 0
        eng.sync()
        a, d = A.download(), dA.download()
        assert np.isfinite(a[:N]).all() and np.isfinite(d[:, :N]).all()
        assert (a[N:] == 7.).all() and (d[:, N:] == 7.).all()
        lc = eng.lib.rtx_launch_count(eng.ctx)
        assert call(rec, None) != 0 and call(None, dopd) != 0      # NULL dopd with P > 0, NULL opd
        A.free(), dA.free()
        S = len(table)
        bad = [dict(spec, radius=0.), dict(spec, radius=np.inf), dict(spec, radius=np.nan)]
        for sp in bad:
            with pytest.raises(_lib.RtxError):
                eng.trace_opd_jacobian(table, dy, du, sp, moves, np.zeros((2, 4)))
        with pytest.raises(_lib.RtxError):
            eng.trace_opd_jacobian(table, dy, du, spec, moves, np.full((2, 4), np.nan))
        tilt = record_tangents(table, [(S, "tilt_x")])
        with pytest.raises(_lib.RtxError):
            eng.trace_opd_jacobian(table, dy, du, spec, tilt, np.zeros((1, 4)))
        assert eng.lib.rtx_launch_count(eng.ctx) == lc
        out = np.zeros(8)
        for args in ((eng.ctx, -1, 1, dy.ptr, dy.ptr, 100, 0., out.ctypes.data),
                     (eng.ctx, 10, 65, dy.ptr, dy.ptr, 100, 0., out.ctypes.data),
                     (eng.ctx, 10, 1, dy.ptr, None, 100, 0., out.ctypes.data),
                     (eng.ctx, 10, 1, dy.ptr, dy.ptr, 5, 0., out.ctypes.data)):
            assert eng.lib.rtx_wavefront_sums(*args) != 0
        assert eng.lib.rtx_wavefront_sums(eng.ctx, 10, 0, dy.ptr, None, 10, 0.,
                                          out.ctypes.data) == 0
        assert eng.lib.rtx_launch_count(eng.ctx) == lc + 2
    finally:
        dy.free(), du.free()


# ---- the optimiser on the reference's Cooke --------------------------------
needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="no reference tree staged")
HEIGHTS = (0., .7, 1.)


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
    from rayopt_b200.surface_table import pack_system
    t = pack_system(s, s.wavelengths[0], 1, None)[0]
    cs = [j for j in range(1, len(t)) if t["c"][j - 1] != 0][:5]
    return [(j, "curvature") for j in cs] + [(len(t), "distance")]


@needs_ref
def test_gradient_matches_trial_scorer(eng):
    from rayopt_b200 import optimize as opt
    s = cooke()
    params = cooke_params(s)
    wl = [s.wavelengths[0]]
    res = opt.wavefront_jacobian(copy.deepcopy(s), params, HEIGHTS, wl, nrays=400, engine=eng)
    B = opt._Bundles(copy.deepcopy(s), HEIGHTS, wl, 400, "hexapolar", eng, False)
    st = None
    try:
        st = opt._Wavefront(eng, s, B, HEIGHTS, None, None, False, False)
        P = len(params)
        for b in range(len(HEIGHTS)):
            w = np.zeros(len(HEIGHTS))
            w[b] = 1
            merit = lambda d: opt._wavefront_merits(eng, B, st, params, d, w, False, False)  # noqa
            m0 = merit(np.zeros((1, P)))[0]
            assert np.isclose(np.sqrt(m0), res["rms"][b, 0], rtol=1e-9)
            g = res["grad"][b, 0]
            for p in range(P):
                h = 1e-5 if params[p][1] == "curvature" else 1e-3
                e = np.zeros((4, P))
                e[:, p] = [h, -h, h/2, -h/2]
                m = merit(e)
                fd = (4*(m[2] - m[3])/h - (m[0] - m[1])/(2*h))/3
                assert abs(fd - g[p]) <= 1e-6*np.abs(g).max() + 1e-9*abs(m0), (b, p, fd, g[p])
    finally:
        if st is not None:
            st.close()
        B.close()


@needs_ref
def test_optimize_wavefront(eng):
    from rayopt_b200 import optimize as opt
    s = cooke()
    params = cooke_params(s)
    wl = [s.wavelengths[0]]
    rng = np.random.default_rng(4)
    opt.apply_deltas(s, params[:-1], rng.uniform(-2e-4, 2e-4, len(params) - 1))
    keep = copy.deepcopy(s)
    r = opt.optimize_wavefront(s, params, HEIGHTS, wl, iterations=4, nrays=300, engine=eng)
    # the caller's System is untouched
    assert [e.curvature for e in s] == [e.curvature for e in keep]
    assert [e.distance for e in s] == [e.distance for e in keep]
    # every accepted trial lowers the fixed-bundle merit, and the lens ends lower
    for k in range(len(r["lam"])):
        if r["lam"][k]:
            assert r["trial"][k] < r["merit"][k]
    assert r["merit"][-1] < r["merit"][0]
    # the first step is lm_step of wavefront_jacobian's normal equations
    j = opt.wavefront_jacobian(copy.deepcopy(keep), params, HEIGHTS, wl, nrays=300, engine=eng)
    assert r["lam"][0], "the first step of a perturbed Cooke was not accepted"
    step = opt.lm_step(j["JtJ"].sum((0, 1)), j["Jtr"].sum((0, 1)), r["lam"][0])
    assert np.allclose(step, r["step"][0], rtol=1e-8, atol=1e-8*np.abs(step).max())


@needs_ref
@pytest.mark.parametrize("height", [0., .7])
def test_rms_is_opd_rays(eng, height):
    """wavefront_jacobian's rms is the rms about its mean of
    ResidentMixin.opd_rays' t (opd() before regridding, the reference's
    own conventions for the sphere, the index after the last surface and
    the table), on the same rays"""
    from rayopt_b200 import ResidentTrace
    from rayopt_b200 import optimize as opt
    s = cooke()
    wl = s.wavelengths[0]
    res = opt.wavefront_jacobian(copy.deepcopy(s), [(1, "curvature")], (height,), [wl],
                                 nrays=1000, clip=True, engine=eng)
    g = ResidentTrace(copy.deepcopy(s), engine=eng)
    try:
        g.rays_point((0, height), wl, nrays=1000, distribution="hexapolar", clip=True)
        _, _, t = g.opd_rays()
    finally:
        g.free()
    t = t[np.isfinite(t)]
    assert res["n"][0, 0] == t.size
    want = np.sqrt(np.mean((t - t.mean())**2))
    assert abs(res["rms"][0, 0] - want) <= 1e-12*want, (res["rms"][0, 0], want)


@needs_ref
def test_focus_only_is_stationary(eng):
    from rayopt_b200 import optimize as opt
    s = cooke()
    L = len(s)
    params = [(L - 1, "distance")]
    r = opt.optimize_wavefront(s, params, (0.,), [s.wavelengths[0]], iterations=6, nrays=300,
                               engine=eng)
    sf = r["system"]
    B = opt._Bundles(copy.deepcopy(sf), (0.,), [s.wavelengths[0]], 300, "hexapolar", eng, False)
    st = None
    try:
        st = opt._Wavefront(eng, sf, B, (0.,), None, None, False, False)
        h = 1e-3
        m = opt._wavefront_merits(eng, B, st, params, np.array([[0.], [h], [-h]]), np.ones(1),
                                  False, False)
        assert m[1] >= m[0] and m[2] >= m[0], m
    finally:
        if st is not None:
            st.close()
        B.close()
