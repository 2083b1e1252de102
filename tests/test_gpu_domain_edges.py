"""The trace at its decision boundaries, against the numpy oracle.

Rays sit on (and one to three ulps either side of) the boundaries where the
reference decides between a number and NaN: the aperture rim (r2 <= radius2),
a tangent intercept (discriminant 0), the critical angle (a*a - b = 0), the
conic's domain (w = 0, the hemisphere rim), the paraboloid's axis ray (e = 0),
Newton's F == 0 / F' == 0 / fifth-iteration exits, planes with signed-zero
and parallel rays, and launch rays with NaN, infinite or signed-zero
components in warps of ordinary rays (oracle/edge_bundles.py builds them;
tests/test_edge_oracle.py checks on the CPU that they straddle).

  exact  every stored entry of Y, U, I, T equals the oracle's bit pattern
         (any NaN matches any NaN; signs of zero and infinities must match)
         in the default, rpt = 1, rpt = 2 and per-thread-store kernels; the
         vignetting mask is the oracle's finite U[-1].x, the path sum the
         oracle's left-to-right sum of T, and rtx_trace_reduce's #finite,
         #total and #good the oracle's counts.
  fast   the NaN mask may differ only on rays within FAST_ULPS ulps (of the
         walked launch coordinate) of the oracle's boundary, and not at all
         at the aperture rim where the intercept is the oracle's own; values
         within 1e-10 on every ray farther than NEAR_ULPS from a boundary
         (closer in, the reference's own problem is ill-conditioned: the
         grazing exit just inside the critical angle turns an ulp of a*a - b
         into 1e-8 of the direction; the largest difference is printed).
  fp32   the NaN mask may differ only on rays within NEAR_ULPS such ulps
         (2^36: 128 single-precision ulps) of the boundary; flips inside are
         counted.  Newton's convergence boundary is exempt: the FP32 kernels
         stop at 4 ulp of the iterate, not at the reference's 1e-7.

Launch rays with a NaN or infinite component are outside the bit-identity
promise (include/rtx.h): for them the engine's entry is the oracle's, or NaN
where the oracle's is NaN or infinite, and the mask and counts agree.
Every case prints its boundary rays and flips per mode (`pytest -s`).
Needs a GPU: `pytest -m gpu`.
"""
import numpy as np
import pytest

import edge_bundles as eb
import np_oracle
from conftest import load_golden
from epi_oracle import reduce_terms

pytestmark = pytest.mark.gpu

FAST_ULPS = 16
NEAR_ULPS = 2.**36
CASES = {c.name: c for c in eb.cases()}
EXACT_CFGS = [("default", {}), ("rpt1", dict(rpt=1)), ("rpt2", dict(rpt=2)),
              ("direct", dict(direct=True))]


@pytest.fixture(scope="module")
def eng():
    from rayopt_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def _run(eng, tab, y0, u0, clip, dtype=np.float64, exact=False, **kw):
    """one rtx_trace on the device with mask and path sum; host copies back"""
    y0 = np.ascontiguousarray(y0, dtype)
    u0 = np.ascontiguousarray(u0, dtype)
    N, S = len(y0), len(tab)
    ld = (N + 127)//128*128
    dy, du = eng.to_device(y0), eng.to_device(u0)
    out = [eng.empty((S, ld, 3), dtype) for _ in range(3)] + [eng.empty((S, ld), dtype)]
    mask = eng.empty(((N + 31)//32,), np.uint32)
    ps = eng.empty((N,), dtype)
    eng.trace_device(tab, dy, du, *out, N=N, ld=ld, clip=clip, exact=exact, mask=mask,
                     path_sum=ps, **kw)
    eng.sync()
    cfg = eng.last_launch_config()
    Y, U, I, T = (a.download()[:, :N] for a in out)
    bits = np.unpackbits(mask.download().view(np.uint8), bitorder="little")[:N].astype(bool)
    m = eng.trace_reduce(tab, dy, du, clip=clip, exact=exact)
    got = dict(Y=Y, U=U, I=I, T=T, mask=bits, ps=ps.download(), m=m, cfg=cfg)
    for a in out + [dy, du, mask, ps]:
        a.free()
    return got


def _oracle(tab, y0, u0, clip):
    Y, U, I, T = np_oracle.trace(tab, y0, u0, clip=clip)
    ps = np.zeros(len(y0))
    for t in T:
        ps = ps + t
    terms = reduce_terms(Y[-1], I[-1])
    return dict(Y=Y, U=U, I=I, T=T, mask=np.isfinite(U[-1][:, 0]), ps=ps,
                counts=terms[:, [4, 5, 8]].sum(0))


def _same_bits(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return (a.view(np.uint64) == b.view(np.uint64)) | (np.isnan(a) & np.isnan(b))


def _check_exact(got, want, fin, label):
    """bit patterns where the launch ray is finite; elsewhere the oracle's
    bits or NaN for the oracle's NaN / inf; mask, path sum and counts exact"""
    for k in ("Y", "U", "I", "T", "ps"):
        a, b = got[k], want[k]
        ok = _same_bits(a, b)
        lax = ok | (np.isnan(a) & np.isinf(b))
        rays = {3: fin[None, :, None], 2: fin[None, :], 1: fin}[a.ndim]
        bad = ~np.where(rays, ok, lax)
        if bad.any():
            idx = np.argwhere(bad)[0]
            raise AssertionError("%s %s: %d entries differ, first at %s: engine %r (%016x), "
                                 "oracle %r (%016x)" % (
                                     label, k, bad.sum(), tuple(idx), a[tuple(idx)],
                                     np.float64(a[tuple(idx)]).view(np.uint64),
                                     b[tuple(idx)], np.float64(b[tuple(idx)]).view(np.uint64)))
    assert np.array_equal(got["mask"], want["mask"]), (label, "mask",
                                                       np.flatnonzero(got["mask"] != want["mask"]))
    assert np.array_equal(got["m"][[4, 5, 8]], want["counts"]), (label, "counts",
                                                                 got["m"][[4, 5, 8]],
                                                                 want["counts"])


def _flips(got, want):
    """rays whose NaN status differs at any surface, in any stored array"""
    f = np.zeros(got["T"].shape[1], bool)
    for k in ("Y", "U", "I"):
        f |= (np.isnan(got[k]) != np.isnan(want[k])).any(axis=(0, 2))
    f |= (np.isnan(got["T"]) != np.isnan(want["T"])).any(0)
    return f


@pytest.mark.parametrize("name", list(CASES))
def test_boundary_case(eng, name):
    c = CASES[name]
    want = _oracle(c.table, c.y0, c.u0, c.clip)
    fin = np.ones(len(c.y0), bool)
    near = np.isfinite(c.margin) & (c.margin <= eb.W + 1)
    print("\n%s: %d rays, %d at the boundary (edge pairs %d)" % (
        name, len(c.y0), near.sum(), len(c.edges)))
    for label, kw in EXACT_CFGS:
        got = _run(eng, c.table, c.y0, c.u0, c.clip, exact=True, **kw)
        if "rpt" in kw:
            assert got["cfg"][0] == kw["rpt"], (label, got["cfg"])
        if kw.get("direct"):
            assert got["cfg"][1] == 0, (label, got["cfg"])
        _check_exact(got, want, fin, "%s exact %s" % (name, label))
    for label, kw in EXACT_CFGS[:3:2]:
        got = _run(eng, c.table, c.y0, c.u0, c.clip, **kw)
        flips = _flips(got, want)
        print("  fast %-7s flips %d, at margins %s" % (label, flips.sum(), c.margin[flips]))
        assert not (flips & ~(c.margin <= FAST_ULPS)).any(), (name, label, c.margin[flips])
        if name.startswith("rim"):      # the clip decision on the oracle's own intercept
            own = (_same_bits(got["Y"][0], want["Y"][0])).all(1)
            assert not (flips & own).any(), (name, label, "clip flip on an exact intercept")
        both = np.isfinite(want["Y"]) & np.isfinite(got["Y"])
        err = np.where(both, np.abs(got["Y"] - want["Y"])/np.maximum(np.abs(want["Y"]), 1.), 0)
        far = ~(c.margin <= NEAR_ULPS)
        print("  fast %-7s max rel err %.1e away from boundaries, %.1e near them" % (
            label, err[:, far].max(initial=0), err[:, ~far].max(initial=0)))
        assert (err[:, far] <= 1e-10).all(), (name, label)
    y32, u32 = c.y0.astype(np.float32), c.u0.astype(np.float32)
    want32 = _oracle(c.table, y32.astype(np.float64), u32.astype(np.float64), c.clip)
    got = _run(eng, c.table, y32, u32, c.clip, dtype=np.float32)
    flips = _flips({k: got[k].astype(np.float64) for k in "YUIT"}, want32)
    print("  fp32 flips %d (of %d rays within the fp32 margin)" % (
        flips.sum(), (c.margin <= NEAR_ULPS).sum()))
    if not name.startswith("newton_fifth"):
        assert not (flips & ~(c.margin <= NEAR_ULPS)).any(), (name, "fp32", c.margin[flips])


@pytest.mark.parametrize("golden", ["double_gauss_l0_clip", "cooke_asph_f07_clip"])
def test_axis_and_nonfinite_rays_through_a_system(eng, golden):
    """on-axis rays with every sign of zero, and launch rays with one NaN,
    +-inf or +-0 component mixed into warps of the golden's rays"""
    g = load_golden(golden)
    y0, u0 = g["y0"][:200].copy(), g["u0"][:200].copy()
    z = y0[0, 2]
    axis_y, axis_u = [], []
    for sx in (0., -0.):
        for sy in (0., -0.):
            axis_y.append([sx, sy, z])
            axis_u.append([sy, sx, 1.])
    y0 = np.vstack([axis_y, y0])
    u0 = np.vstack([axis_u, u0])
    y0, u0, fin = eb.mixed_bundle(y0, u0)
    want = _oracle(g["table"], y0, u0, g["clip"])
    print("\n%s: %d rays, %d with a non-finite launch component" % (golden, len(y0),
                                                                    (~fin).sum()))
    for label, kw in EXACT_CFGS:
        got = _run(eng, g["table"], y0, u0, g["clip"], exact=True, **kw)
        _check_exact(got, want, fin, "%s exact %s" % (golden, label))
    lax = sum(int((~_same_bits(got[k], want[k])).sum()) for k in "YUIT")
    print("  exact: %d entries NaN where the oracle has an infinity" % lax)
    got = _run(eng, g["table"], y0, u0, g["clip"])
    flips = _flips(got, want)
    print("  fast flips %d" % flips.sum())
    assert not flips[fin].any()
    assert np.array_equal(got["mask"], want["mask"])


def _ulps(got, exact):
    """|got - exact| in ulps of the double nearest to `exact` (Fractions)"""
    out = []
    for g, e in zip(got, exact):
        r = float(e)
        out.append(float(abs(g - e)/np.spacing(abs(r))))
    return np.array(out)


def test_fast_primitives_within_their_bounds(eng):
    """div2_rn_noslow is __ddiv_rn bit for bit (signed zeros, operands near
    2^+-1000, quotients at the normal and overflow limits, zero and infinite
    divisors); rcp_fast and sqrt_rsqrt_fast hold their stated bounds over the
    normal range, against exact Fractions"""
    from fractions import Fraction
    rng = np.random.default_rng(11)
    n = 1 << 14
    a = rng.standard_normal(n)*2.0**rng.integers(-1000, 1001, n)
    b = rng.standard_normal(n)*2.0**rng.integers(-1000, 1001, n)
    c = rng.standard_normal(n)*10.0**rng.integers(-8, 9, n)
    # quotients near the normal / overflow limits, zeros and infinities
    a[:64] = np.ldexp(1 + rng.random(64), -1000)
    b[:64] = np.ldexp(1 + rng.random(64), 21)
    a[64:128] = np.ldexp(1 + rng.random(64), 1000)
    b[64:128] = np.ldexp(1 + rng.random(64), -23)
    sp = [0., -0., 1., -1., 3., -3., np.inf, -np.inf, np.nan]
    k = 128
    for x in sp:
        for y in sp:
            a[k], b[k], c[k] = x, y, -x
            k += 1
    out = eng.selftest_math2(a, b, c)
    with np.errstate(all="ignore"):
        q = a/b
        normal = np.isfinite(q) & ((np.abs(q) >= np.finfo(float).tiny) | (q == 0))
        normal &= np.isfinite(c/b) & ((np.abs(c/b) >= np.finfo(float).tiny) | (c/b == 0))
    normal &= np.abs(b) < 2.**1022                  # the reciprocal stays normal
    ieee = np.isnan(a) | np.isnan(b) | np.isnan(c) | (b == 0)
    for i, j in ((0, 2), (1, 3)):
        same = _same_bits(out[i], out[j])
        for cls, sel in (("specials", slice(128, k)), ("near the normal limit", slice(0, 64)),
                         ("near overflow", slice(64, 128)), ("2^+-1000", slice(k, n))):
            print("div2 %d %s: %d of %d differ" % (i, cls, (~same[sel]).sum(),
                                                     same[sel].size))
        assert same[normal | ieee].all(), ("div2", i, np.flatnonzero(~same & (normal | ieee))[:5])
    assert _same_bits(out[2][normal], q[normal]).all()
    # rcp_fast: < 1 ulp (no final rounding step), +-inf for +-0
    ok = np.isfinite(b) & (b != 0) & (np.abs(b) < 2.**1022)
    idx = np.flatnonzero(ok)[:4000]
    e = _ulps([Fraction(float(x)) for x in out[4][idx]], [1/Fraction(float(x)) for x in b[idx]])
    print("\nrcp_fast: max %.3f ulp" % e.max())
    assert e.max() < 1.0
    assert np.array_equal(out[4][b == 0], np.copysign(np.inf, b[b == 0]))
    # sqrt_rsqrt_fast: sqrt correctly rounded (the same sequence as
    # sqrt_rn_noslow), 1/sqrt within 2^-52 relative; sqrt(+-0) = +-0
    pos = np.flatnonzero(np.isfinite(a) & (a > 0) & (a >= np.finfo(float).tiny))[:4000]
    assert _same_bits(out[5][pos], np.sqrt(a[pos])).all()
    rs = out[6][pos]
    rel = [abs(Fraction(float(r))**2*Fraction(float(x)) - 1)/2 for r, x in zip(rs, a[pos])]
    print("1/sqrt: max rel %.3e" % max(float(r) for r in rel))
    assert max(rel) < Fraction(1, 2**52)
    zero = a == 0
    assert _same_bits(out[5][zero], a[zero]).all()
