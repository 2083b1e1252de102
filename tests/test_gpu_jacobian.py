"""rtx_trace_jacobian and rtx_jacobian_sums on the device.  Needs a GPU.

q is compared with rtx_trace's stored last row bit for bit.  J is compared
ray by ray with the forward-mode oracle (oracle/jac_oracle.py, itself held
to Richardson differences in tests/test_jacobian_host.py) within
JAC_RTOL x the column's scale (the largest |J| of the parameter and axis,
at least 1e-3 of the largest of any column).
The sums are compared with math.fsum of the device's own q and J within the
bound include/rtx.h states."""
import math

import numpy as np
import pytest

import jac_oracle
from conftest import load_golden, load_systems
from rayopt_b200.rays import aim_infinite, disc
from rayopt_b200.tolerance import record_tangents

pytestmark = pytest.mark.gpu

EPS = 2.0**-52
JAC_RTOL = 1e-10
FAST_ULPS = 16   # tests/test_gpu_domain_edges.py: fast mode decides as the reference past this


@pytest.fixture(scope="module")
def eng():
    from rayopt_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def systems():
    return load_systems()


def system_case(systems, name, n, seed=0, li=0, field=2, scale=1.):
    ent = systems[name]
    aim = ent["aim"][li][field]
    y0, u0 = aim_infinite(aim["field"], disc(n, seed)*scale, aim["z"], aim["p"],
                          ent["object_angle"])
    return ent["tables"][li], None, y0, u0


def golden_case(name):
    c = load_golden(name)
    return c["table"], c["rot0"], c["y0"], c["u0"]


def same_bits(a, b):
    """bit for bit, NaN for NaN (a NaN's payload is not part of the result)"""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and a[~na].tobytes() == b[~nb].tobytes()


def curved(table):
    return [j for j in range(1, len(table) + 1) if table["c"][j - 1] != 0]


def device_jac(eng, table, rot0, y0, u0, moves, clip, exact):
    """q, J and the sums' bad-tangent count of one launch"""
    dy, du = eng.to_device(y0), eng.to_device(u0)
    try:
        q, J = eng.trace_jacobian(table, dy, du, moves, clip=clip, rot0=rot0, exact=exact)
        N = len(y0)
        out = q.download(), J.download()[:, :, :N], eng.jacobian_sums(q, J)["bad"]
        q.free(), J.free()
        return out
    finally:
        dy.free(), du.free()


def plates(S=256):
    """a stack of plane-parallel plates: a 92 KB FP64 table, past the 48 KB
    of shared memory a kernel gets without opting in"""
    from rayopt_b200.surface_table import SURFACE_DTYPE
    t = np.zeros(S, SURFACE_DTYPE)
    t["rot"] = np.eye(3).reshape(9)
    t["offset"][:, 2] = .01
    t["radius2"] = np.inf
    t["n_asph"] = -1
    n = np.where(np.arange(S) % 2 == 0, 1.5, 1.0)
    t["n0"], t["n"] = np.r_[1.0, n[:-1]], n
    t["mu"] = t["n0"]/t["n"]
    t["muf"], t["sgn"], t["mu2m1"] = np.abs(t["mu"]), np.sign(t["mu"]), t["mu"]**2 - 1
    rng = np.random.default_rng(11)
    u = rng.normal(0, .1, (3000, 2))
    return t, None, np.c_[rng.normal(0, 1, (3000, 2)), np.zeros(3000)], \
        np.c_[u, np.sqrt(1 - np.square(u).sum(1))]


# ---- the primal is the trace's last row ---------------------------------
@pytest.mark.parametrize("exact", [True, False], ids=["exact", "fast"])
@pytest.mark.parametrize("N", [0, 1, 31, 32, 33, 511, 512, 513, 70001])
def test_q_is_trace_last_row(eng, systems, exact, N):
    table, rot0, y0, u0 = system_case(systems, "double_gauss", max(N, 1), seed=N)
    y0, u0 = y0[:N], u0[:N]
    cs = curved(table)
    for P in (1, 4, 5, 17, 64):
        params = [(cs[p % len(cs)], ("curvature", "conic", "distance")[p % 3]) for p in range(P)]
        moves = record_tangents(table, params)
        dy, du = eng.to_device(np.zeros((max(N, 1), 3))), eng.to_device(np.zeros((max(N, 1), 3)))
        if N:
            dy.upload(y0), du.upload(u0)
        q, J = eng.trace_jacobian(table, dy, du, moves, clip=True, exact=exact, N=N)
        got = q.download()
        if N:
            Y = eng.trace(table, y0, u0, clip=True, keep_last=True, exact=exact, want=("y",))[0]
            assert same_bits(got, Y[0, :, :2]), P
            Jh = J.download()[:, :, :N]
            nanq = np.isnan(got).any(1)
            assert np.isnan(Jh).any((0, 1))[nanq].all()
        for a in (q, J, dy, du):
            a.free()


# ---- J against the oracle ----------------------------------------------
# every epilogue test system (tests/test_gpu_epilogues.py) and the fixtures
# with Newton surfaces, mirrors and rotated rows
CASES = {
    "cooke": ("sys", [(1, "curvature"), (3, "conic"), (2, "distance"), (4, "asph0"),
                      (3, "asph2"), (2, "tilt_x"), (6, "tilt_y"), (1, "index"), (6, "index")]),
    "cooke_asph": ("sys", [(2, "asph1"), (3, "curvature"), (1, "curvature"), (6, "distance"),
                           (1, "tilt_y"), (2, "conic"), (3, "index")]),
    "double_gauss": ("sys", [(3, "curvature"), (6, "distance"), (7, "conic"), (4, "tilt_x"),
                             (1, "index"), (8, "asph0"), (12, "distance")]),
    "zoom": ("sys", [(2, "curvature"), (4, "distance"), (1, "tilt_x"), (1, "index")]),
    "mirror": ("sys", [(1, "curvature"), (1, "conic"), (1, "asph0"), (1, "distance"),
                       (1, "tilt_y")]),
    "s1": ("sys", [(1, "curvature"), (1, "conic"), (1, "distance"), (1, "asph1"),
                   (1, "tilt_x")]),
    "plates256": ("plates", [(1, "curvature"), (100, "distance"), (50, "index"), (7, "asph0"),
                             (3, "tilt_x"), (256, "distance")]),
    "mirror_folded": ("gold", [(1, "curvature"), (1, "conic"), (2, "distance"), (1, "asph0")]),
    "tilted_start3": ("gold", [(2, "curvature"), (1, "curvature"), (1, "conic")]),
    "tilted_clip0": ("gold", [(1, "curvature"), (3, "curvature"), (1, "index"), (3, "distance")]),
    "newton_edge_clip1": ("gold", None),
    "cooke_asph_f07_clip": ("gold", None),
}


def case_params(table, params):
    if params is not None:
        return params
    cs = curved(table) or [1]
    return [(j, "curvature") for j in cs[:4]] + [(len(table), "distance")]


def check_against_oracle(q, J, qo, Jo, bad, edge=False, exclude=None, novalue=None):
    """J against the oracle ray by ray; returns the largest error over the
    compared rays in units of the column's scale.

    A ray with a NaN q has NaN tangents.  A ray with a finite q and a
    non-finite tangent ("bad", the grazing rays rtx_jacobian_sums counts)
    must be bad in the oracle too, except where the other side's tangent is
    finite but near-singular (more than 1e6 x the typical ray's): there
    the two differ only by whether the FMA-contracted or the numpy
    denominator rounded to exactly 0.  Such near-singular rays are not
    compared either.  On a lens (not an edge bundle) fewer than 1 % of the
    finite rays may be bad and at least 90 % must be compared; on an edge
    bundle, whose walked rays sit ulps from a tangent or critical ray, at
    least a quarter of the rays not in `novalue`.  `exclude`: rays left out
    after the bad count is checked; `novalue`: rays whose values are not
    compared and whose bad flag may differ from the oracle's (rays near a
    singular boundary)."""
    assert bad == (np.isfinite(q).all(1) & ~np.isfinite(J).all((0, 1))).sum()
    if exclude is not None:
        q, J, qo, Jo = q[~exclude], J[:, :, ~exclude], qo[~exclude], Jo[:, :, ~exclude]
        novalue = None if novalue is None else novalue[~exclude]
    fq = np.isfinite(q).all(1)
    assert np.array_equal(fq, np.isfinite(qo).all(1))
    nj = ~np.isfinite(J).all((0, 1))
    noj = ~np.isfinite(Jo).all((0, 1))
    assert nj[~fq].all(), "a NaN q with a finite tangent"
    dbad, obad = fq & nj, fq & noj
    both = fq & ~nj & ~noj
    # a ray's tangents are near-singular when they exceed 1e6 x the typical
    # ray's largest |J| (the median over the rays of the largest |J| of any
    # column; at least 1e-3 of the largest, for bundles whose typical ray
    # does not move, such as axial rays)
    rmax = np.abs(Jo[:, :, both]).max((0, 1)) if both.any() else np.zeros(1)
    typ = max(np.median(rmax), 1e-3*rmax.max())

    def huge(X):
        return (np.abs(X) > 1e6*max(typ, 1e-300)).any((0, 1))
    # within ulps of a singular boundary the disagreement may also hide in a
    # column that is 0 in exact arithmetic (the singular tangents cancel):
    # there only the count against the sums is checked
    free = np.zeros(len(q), bool) if novalue is None else novalue
    assert not (dbad & ~obad & ~free
                & ~huge(np.nan_to_num(Jo, nan=0., posinf=0., neginf=0.))).any()
    assert not (obad & ~dbad & ~free
                & ~huge(np.nan_to_num(J, nan=0., posinf=0., neginf=0.))).any()
    ok = both & ~huge(J) & ~huge(Jo)
    n = fq.sum()
    if novalue is not None:
        ok &= ~novalue
        n = (fq & ~novalue).sum()
    if edge:
        assert ok.sum() >= n/4, (ok.sum(), n)
    else:
        assert dbad.sum() <= .01*n and ok.sum() >= .9*n, (dbad.sum(), ok.sum(), n)
    worst = 0.
    gok = np.abs(Jo[:, :, ok]).max(initial=0.)
    for p in range(J.shape[0]):
        for a in range(2):
            if not ok.any():
                continue
            # a column far below the others is held to 1e-3 of the largest
            # (on an edge bundle to the largest: its small tables' columns are
            # of one size, and a column that is 0 in exact arithmetic, such as
            # a sphere with mu = 1 grazed by the ray, is the FP64 rounding of
            # tangents larger than any q-derivative)
            scale = max(np.abs(Jo[p, a, ok]).max(), (1. if edge else 1e-3)*gok, 1e-300)
            err = np.abs(J[p, a, ok] - Jo[p, a, ok]).max()/scale
            worst = max(worst, err)
    assert worst <= JAC_RTOL, worst
    return worst


def get_case(systems, name):
    src, params = CASES[name]
    if src == "sys":
        ent = systems["cooke" if name == "s1" else name]
        aim = ent["aim"][0][2]
        y0, u0 = aim_infinite(aim["field"], disc(3000, 7), aim["z"], aim["p"],
                              ent["object_angle"])
        table = ent["tables"][0][:1] if name == "s1" else ent["tables"][0]
        return table, None, y0, u0, params
    if src == "plates":
        return plates() + (params,)
    return golden_case(name) + (params,)


@pytest.mark.parametrize("clip", [False, True], ids=["noclip", "clip"])
@pytest.mark.parametrize("exact", [True, False], ids=["exact", "fast"])
@pytest.mark.parametrize("name", list(CASES))
def test_J_matches_oracle(eng, systems, name, exact, clip):
    table, rot0, y0, u0, params = get_case(systems, name)
    params = case_params(table, params)
    moves = record_tangents(table, params)
    q, J, bad = device_jac(eng, table, rot0, y0, u0, moves, clip, exact)
    with np.errstate(all="ignore"):
        qo, Jo = jac_oracle.trace(table, y0, u0, moves, clip=clip, rot0=rot0)
    T = eng.trace(table, y0, u0, clip=clip, keep_last=True, rot0=rot0, exact=exact,
                  want=("y",))[0]
    assert same_bits(q, T[0, :, :2])
    print("%s: %.1e" % (name, check_against_oracle(q, J, qo, Jo, bad)))


def edge_cases():
    import edge_bundles
    return {c.name: c for c in edge_bundles.cases()}


@pytest.mark.parametrize("exact", [True, False], ids=["exact", "fast"])
def test_J_edge_bundles(eng, exact):
    """the decision-boundary bundles of oracle/edge_bundles.py: tangent,
    critical-angle, rim, mirror, mu = 1, paraboloid and Newton rays, where the
    tangents of grazing rays are non-finite and counted as bad"""
    for name, c in edge_cases().items():
        params = [(1, "curvature"), (2, "distance"), (1, "asph0")]
        if c.table["c"][0] != 0:
            params.append((1, "conic"))
        moves = record_tangents(c.table, params)
        q, J, bad = device_jac(eng, c.table, None, c.y0, c.u0, moves, c.clip, exact)
        with np.errstate(all="ignore"):
            qo, Jo = jac_oracle.trace(c.table, c.y0, c.u0, moves, clip=c.clip)
        T = eng.trace(c.table, c.y0, c.u0, clip=c.clip, keep_last=True, exact=exact,
                      want=("y",))[0]
        assert same_bits(q, T[0, :, :2]), name
        # fast mode's intercepts may differ from the reference's by an ulp, so
        # a walked ray next to a boundary may be kept where the oracle loses
        # it (tests/test_gpu_domain_edges.py states the rule); exact mode
        # decides every ray as the oracle does
        flip = np.isfinite(q).all(1) != np.isfinite(qo).all(1)
        if exact:
            assert not flip.any(), name
        else:
            assert (c.margin[flip] <= FAST_ULPS).all(), name
        # Where the boundary is a singularity of the step (a tangent intercept,
        # the critical angle, a Newton root at a flat slope), a ray near it
        # carries intermediate tangents of order 1/sqrt(distance); its
        # q-derivative keeps their FP64 rounding (eps times that size), which
        # the FMA-contracted and the numpy tangents round differently, even
        # where the exact q-derivative is 0 (a sphere with mu = 1).  The rays
        # walked within ulps and those 1e-9 away (edge_bundles.FAR) may also
        # round the denominator to exactly 0 on one side only; they are held
        # to the NaN rule and the sums' count; the rays 1e-3 away are compared.
        singular = name.startswith(("tangent", "critical", "hemisphere", "paraboloid",
                                    "newton"))
        near = c.margin <= 1e10 if singular else np.zeros(len(q), bool)
        try:
            check_against_oracle(q, J, qo, Jo, bad, edge=True, exclude=flip, novalue=near)
        except AssertionError as e:
            raise AssertionError("%s: %s" % (name, e))


def test_rot0_launch(eng, systems):
    table, _, y0, u0 = system_case(systems, "cooke", 2000, seed=3)
    a = .01
    rot0 = np.array([[1, 0, 0], [0, np.cos(a), -np.sin(a)], [0, np.sin(a), np.cos(a)]])
    moves = record_tangents(table, [(1, "curvature"), (4, "distance"), (3, "tilt_x")])
    q, J, bad = device_jac(eng, table, rot0, y0, u0, moves, True, False)
    with np.errstate(all="ignore"):
        qo, Jo = jac_oracle.trace(table, y0, u0, moves, clip=True, rot0=rot0)
    check_against_oracle(q, J, qo, Jo, bad)


def test_pickup_is_the_sum_of_its_moves(eng, systems):
    """a two-move parameter (shift a group: distance j and -distance j+1)"""
    table, rot0, y0, u0 = system_case(systems, "cooke", 4000, seed=9)
    (mj,), (mk,) = record_tangents(table, [(3, "distance"), (4, "distance")])
    neg = record_tangents(table, [(4, "distance")])[0][0][1]
    neg["offset"] *= -1
    q, J, _ = device_jac(eng, table, rot0, y0, u0, [[mj], [mk], [mj, (mk[0], neg[()])]], True,
                         False)
    ok = np.isfinite(J).all((0, 1))
    assert ok.sum() >= .9*np.isfinite(q).all(1).sum()
    scale = np.abs(J[:2][..., ok]).max()
    assert np.abs(J[2][:, ok] - (J[0][:, ok] - J[1][:, ok])).max() <= JAC_RTOL*scale


# ---- the sums -----------------------------------------------------------
def fsum_row(q, J, c):
    """the exact sums of the device's own q, J (math.fsum per output) and
    sum|term| per output, in include/rtx.h's layout"""
    P = J.shape[0]
    d = q - c
    fin = np.isfinite(d).all(1) & np.isfinite(J).all((0, 1))
    bad = np.isfinite(d).all(1) & ~np.isfinite(J).all((0, 1))
    d, Jf = d[fin], J[:, :, fin]
    rows, mags = [], []

    def add(*prods):
        terms = np.concatenate([a*b for a, b in prods])
        rows.append(math.fsum(terms))
        mags.append(np.abs(terms).sum())
    one = np.ones(len(d))
    add((one, one))
    add((one, d[:, 0]))
    add((one, d[:, 1]))
    add((d[:, 0], d[:, 0]), (d[:, 1], d[:, 1]))
    for p in range(P):
        for a in range(2):
            add((one, Jf[p, a]))
    for p in range(P):
        add((d[:, 0], Jf[p, 0]), (d[:, 1], Jf[p, 1]))
    for a in range(P):
        for b in range(a, P):
            add((Jf[a, 0], Jf[b, 0]), (Jf[a, 1], Jf[b, 1]))
    rows.append(float(bad.sum()))
    mags.append(0.)
    return np.array(rows), np.array(mags)


def bound(N, mags, chunks=1):
    D = 2*16384 + -(-N//16384) + chunks - 1
    return D*EPS*mags


@pytest.mark.parametrize("N", [1, 513, 16384, 16385, 70001])
def test_sums_match_fsum(eng, systems, N):
    table, rot0, y0, u0 = system_case(systems, "double_gauss", N, seed=N)
    cs = curved(table)
    params = [(j, "curvature") for j in cs[:5]] + [(len(table), "distance")]
    moves = record_tangents(table, params)
    dy, du = eng.to_device(y0), eng.to_device(u0)
    q, J = eng.trace_jacobian(table, dy, du, moves, clip=True)
    c = np.array([.01, -.02])
    s = eng.jacobian_sums(q, J, c)
    want, mags = fsum_row(q.download(), J.download()[:, :, :N], c)
    assert np.all(np.abs(s["out"] - want) <= bound(N, mags)), np.abs(s["out"] - want).max()
    assert s["out"][0] == want[0] and s["out"][-1] == want[-1]
    # bit-identical across calls and contexts
    assert eng.jacobian_sums(q, J, c)["out"].tobytes() == s["out"].tobytes()
    from rayopt_b200.engine import Engine
    e2 = Engine(0)
    try:
        q2, J2 = e2.to_device(q.download()), e2.to_device(J.download())
        assert e2.jacobian_sums(q2, J2, c)["out"].tobytes() == s["out"].tobytes()
    finally:
        e2.close()
    # chunked (the first half, then the rest) within the bound of unchunked
    if N > 1:
        h = N//2
        a = eng.jacobian_sums(*eng.trace_jacobian(table, dy.rows(0, h), du.rows(0, h), moves,
                                                  clip=True), c)["out"]
        b = eng.jacobian_sums(*eng.trace_jacobian(table, dy.rows(h, N), du.rows(h, N), moves,
                                                  clip=True), c)["out"]
        assert np.all(np.abs(a + b - want) <= bound(N, mags, 2))
    for x in (q, J, dy, du):
        x.free()


def test_guard_bands_untouched(eng, systems):
    N, P = 1000, 3
    table, rot0, y0, u0 = system_case(systems, "cooke", N, seed=2)
    moves = record_tangents(table, [(1, "curvature"), (2, "curvature"), (3, "distance")])
    ld = 1100
    dy, du = eng.to_device(y0), eng.to_device(u0)
    qb = eng.to_device(np.full((N + 64, 2), 7.))
    Jb = eng.to_device(np.full((P*2*ld + 256,), 7.))
    from rayopt_b200._lib import ptr
    first = np.array([0, 1, 2, 3], np.int32)
    rows = np.array([r for mv in moves for r, _ in mv], np.int32)
    recs = np.array([x for mv in moves for _, x in mv])
    assert eng.lib.rtx_trace_jacobian(eng.ctx, ptr(table), len(table), None, 0, N, dy.ptr,
                                      du.ptr, 1, P, ptr(first), ptr(rows), ptr(recs), qb.ptr,
                                      Jb.ptr, ld, 0) == 0
    qh, Jh = qb.download(), Jb.download()
    assert (qh[N:] == 7.).all()
    Jr = Jh[:P*2*ld].reshape(P, 2, ld)
    assert (Jr[:, :, N:] == 7.).all() and (Jh[P*2*ld:] == 7.).all()
    for x in (dy, du, qb, Jb):
        x.free()


def test_refusals_launch_and_allocate_nothing(eng, systems):
    from rayopt_b200._lib import ptr
    table, rot0, y0, u0 = system_case(systems, "cooke", 100)
    S = len(table)
    dy, du = eng.to_device(y0), eng.to_device(u0)
    q, J = eng.empty((100, 2)), eng.empty((2, 2, 128))
    moves = record_tangents(table, [(1, "curvature"), (2, "curvature")])
    rows = np.array([0, 1], np.int32)
    recs = np.array([moves[0][0][1], moves[1][0][1]])
    good = np.array([0, 1, 2], np.int32)
    L = eng.lib

    def call(**kw):
        a = dict(ctx=eng.ctx, surf=ptr(table), S=S, rot0=None, dtype=0, N=100, y0=dy.ptr,
                 u0=du.ptr, clip=1, P=2, first=ptr(good), rows=ptr(rows), recs=ptr(recs),
                 q=q.ptr, J=J.ptr, ld=128, flags=0)
        a.update(kw)
        return L.rtx_trace_jacobian(*a.values())
    before = eng.launch_count()
    # an index-like move on a row that does not refract (mu = 1)
    mu_rows = np.array([0, int(np.flatnonzero(table["mu"] == 1)[0])], np.int32)
    mu_recs = recs.copy()
    mu_recs[1]["mu"] = 1.
    bad_t = table.copy()
    bad_t["n_asph"][0] = 11
    for kw, code in [(dict(ctx=None), -1), (dict(q=None), -1), (dict(J=None), -1),
                     (dict(y0=None), -1), (dict(first=None), -1), (dict(rows=None), -1),
                     (dict(recs=None), -1), (dict(P=0), -1), (dict(P=65), -1),
                     (dict(first=ptr(np.array([1, 1, 2], np.int32))), -1),
                     (dict(first=ptr(np.array([0, 1, 1], np.int32))), -1),
                     (dict(first=ptr(np.array([0, 2, 1], np.int32))), -1),
                     (dict(rows=ptr(np.array([0, S], np.int32))), -1),
                     (dict(rows=ptr(np.array([-1, 0], np.int32))), -1),
                     (dict(recs=ptr(mu_recs), rows=ptr(mu_rows)), -1),
                     (dict(ld=99), -1), (dict(dtype=1), -1), (dict(N=-1), -1),
                     (dict(S=0), -1), (dict(surf=ptr(bad_t)), -2)]:
        assert call(**kw) == code, kw
    for args, code in [((None, 100, 2, q.ptr, J.ptr, 128, None, ptr(np.zeros(20))), -1),
                       ((eng.ctx, 100, 2, q.ptr, J.ptr, 128, None, None), -1),
                       ((eng.ctx, 100, 0, q.ptr, J.ptr, 128, None, ptr(np.zeros(20))), -1),
                       ((eng.ctx, 100, 65, q.ptr, J.ptr, 128, None, ptr(np.zeros(9999))), -1),
                       ((eng.ctx, 100, 2, None, J.ptr, 128, None, ptr(np.zeros(20))), -1),
                       ((eng.ctx, 200, 2, q.ptr, J.ptr, 128, None, ptr(np.zeros(20))), -1),
                       ((eng.ctx, -1, 2, q.ptr, J.ptr, 128, None, ptr(np.zeros(20))), -1)]:
        assert L.rtx_jacobian_sums(*args) == code, args
    assert eng.launch_count() == before
    with pytest.raises(ValueError):      # (W,) records per move: not one table's
        eng.trace_jacobian(table, dy, du, record_tangents(np.stack([table, table]),
                                                          [(1, "curvature")]))
    with pytest.raises(ValueError):
        eng.trace_jacobian(table, dy, du, [[]])
    with pytest.raises(ValueError):
        eng.trace_jacobian(table, dy, du, [[(S, moves[0][0][1])]])
    for x in (dy, du, q, J):
        x.free()
