"""Parity of the CUDA engine (through the C ABI) with the oracle and the
golden vectors of the live reference.  Needs a GPU: `pytest -m gpu`."""
import numpy as np
import pytest

import np_oracle
from conftest import golden_names, load_golden, assert_parity
from rayopt_b200.rays import aim_infinite, disc

pytestmark = pytest.mark.gpu

FP64_RTOL = 1e-10     # north_star: <= 1e-10 rel for FP64
FP32_RTOL = 1e-5      # north_star: <= 1e-5 rel for FP32


@pytest.fixture(scope="module")
def eng():
    from rayopt_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def _cmp(got, c, rtol, tag):
    worst = 0.
    for a, b, w in zip(got, (c["Y"], c["U"], c["I"], c["T"]), "yuit"):
        worst = max(worst, assert_parity(a, b, rtol, "%s %s %s" % (c["name"], tag, w)))
    return worst


def _same_bits(a, b):
    """bit patterns equal; any NaN matches any NaN"""
    return (a.view(np.uint64) == b.view(np.uint64)) | (np.isnan(a) & np.isnan(b))


def test_fp64_primitives(eng):
    """the kernels' branch-free FP64 division and sqrt are the IEEE results
    bit for bit (signs of zero included) wherever operands and quotient are
    normal or zero -- operands from 1e-8..1e8, near 2^+-1000, quotients near
    the smallest normal and near overflow -- and for NaN operands and x/0.
    Infinite operands are outside that domain (include/rtx.h)."""
    rng = np.random.default_rng(3)
    n = 1 << 20
    a = rng.standard_normal(n)*10.0**rng.integers(-8, 9, n)
    b = rng.standard_normal(n)*10.0**rng.integers(-8, 9, n)
    m = n//8                                   # operands near 2^+-1000
    a[:m] = rng.standard_normal(m)*2.0**rng.integers(-1000, 1001, m)
    b[:m] = rng.standard_normal(m)*2.0**rng.integers(-1000, 1001, m)
    a[m:2*m] = np.ldexp(1 + rng.random(m), -1000)            # quotient ~ 2^-1021
    b[m:2*m] = np.ldexp(1 + rng.random(m), 21)*rng.choice([-1, 1], m)
    a[2*m:3*m] = np.ldexp(1 + rng.random(m), 1000)           # quotient ~ 2^1023
    b[2*m:3*m] = np.ldexp(1 + rng.random(m), -23)*rng.choice([-1, 1], m)
    sp = [0., -0., np.nan, 1., -1., 4., 7., 2., np.inf, -np.inf]
    pa, pb = np.meshgrid(sp, sp[:8] + [0., -0.])
    a[3*m:3*m + pa.size], b[3*m:3*m + pa.size] = pa.ravel(), pb.ravel()
    out = eng.selftest_math(a, b)
    with np.errstate(all="ignore"):
        q = a/b
    tiny = np.finfo(np.float64).tiny
    normal = lambda x: (np.abs(x) >= tiny) & np.isfinite(x)  # noqa: E731
    ops = (normal(a) | (a == 0)) & normal(b) & np.isfinite(a) & (np.abs(b) < 2.**1022)
    dom = (ops & (normal(q) | (q == 0))) | np.isnan(a) | np.isnan(b) | ((b == 0) & np.isfinite(a))
    for cls, sel in (("2^+-1000", slice(0, m)), ("near the smallest normal", slice(m, 2*m)),
                     ("near overflow", slice(2*m, 3*m)), ("specials", slice(3*m, 3*m + pa.size))):
        print("division %s: %d of %d in the domain differ" % (
            cls, (~_same_bits(out[0], out[1]) & dom)[sel].sum(), dom[sel].sum()))
    assert _same_bits(out[0], out[1])[dom].all(), "division"
    assert _same_bits(out[1], q)[dom].all(), "__ddiv_rn vs numpy"
    sq = np.isnan(a) | (a == 0) | (a < 0) | normal(a)
    assert _same_bits(out[2], out[3])[sq & np.isfinite(a)].all(), "sqrt"
    with np.errstate(all="ignore"):
        assert _same_bits(out[3], np.sqrt(a))[sq & np.isfinite(a)].all()
    pos = normal(a) & (a > 0)
    np.testing.assert_allclose(out[4][pos], out[5][pos], rtol=4e-16)


@pytest.mark.parametrize("rpt", [1, 2])
@pytest.mark.parametrize("name", golden_names())
def test_exact_mode_vs_reference_golden(eng, name, rpt):
    """RTX_EXACT: bit-identical to the reference on unrotated analytic
    systems; a few ulp where the reference itself goes through BLAS dot
    products (rotations, Newton fprime)."""
    c = load_golden(name)
    got = eng.trace(c["table"], c["y0"], c["u0"], clip=c["clip"], rot0=c["rot0"], exact=True,
                    rpt=rpt)
    newton = bool((c["table"]["n_asph"] >= 0).any())
    if not c["rotated"] and not newton:
        for a, b, w in zip(got, (c["Y"], c["U"], c["I"], c["T"]), "yuit"):
            assert np.array_equal(a, b, equal_nan=True), "%s %s not bit-exact" % (name, w)
    else:
        _cmp(got, c, 1e-12, "exact")


@pytest.mark.parametrize("rpt", [1, 2])
@pytest.mark.parametrize("name", golden_names())
def test_fast_mode_vs_reference_golden(eng, name, rpt):
    c = load_golden(name)
    got = eng.trace(c["table"], c["y0"], c["u0"], clip=c["clip"], rot0=c["rot0"], rpt=rpt)
    _cmp(got, c, FP64_RTOL, "fast")


def _fp32_err(a, b):
    """SURVEY 8(d) comparator on the entries finite in both: max of
    |a-b| / max(|b|, scale), scale = max finite |b| of the surface's array for
    lengths (floor 1: direction cosines); returns (error, #NaN-mask flips)"""
    a = np.asarray(a, np.float64)
    flips = int((np.isnan(a) != np.isnan(b)).sum())
    fin = ~np.isnan(a) & ~np.isnan(b)
    absb = np.where(np.isnan(b), 0, np.abs(b))
    scale = np.maximum(absb.reshape(len(b), -1).max(1), 1.0).reshape((-1,) + (1,)*(b.ndim - 1))
    with np.errstate(invalid="ignore"):
        e = np.where(fin, np.abs(a - b)/np.maximum(np.abs(np.where(fin, b, 1)), scale), 0)
    return float(e.max()), flips


# goldens built to sit ON a numerical edge (Newton at the limit of convergence;
# total internal reflection / aperture edges of steep conics): in single
# precision the NaN mask legitimately depends on the last bit
FP32_EDGE = ("newton_edge", "conics")


@pytest.mark.parametrize("name", golden_names())
def test_fp32_vs_reference_golden(eng, name):
    """FP32 kernels against the FP64 reference with the per-surface comparator
    of SURVEY 8(d) at north_star's 1e-5.  Where single precision itself cannot
    hold 1e-5 -- the on-axis image spot after 20 refractions (zoom_f0: the
    direction error ~1.3e-6 times the 19 mm to the image), Newton at the edge
    of convergence -- the bound is what a float32 numpy evaluation of the
    REFERENCE'S OWN formulas (oracle/np_oracle.py, dtype=float32, with the
    engine's FP32 Newton stopping rule) achieves on the same rays, times 1.5.
    newton_edge_clip0 holds a ray that a steep asphere makes ill-conditioned:
    its FP64 trace moves by up to 2.6e-5 at surface 2 when its inputs move by
    6e-8 (float32 rounding), so the float32 budget, not 2e-5, bounds it."""
    c = load_golden(name)
    got = eng.trace(c["table"], c["y0"], c["u0"], clip=c["clip"], rot0=c["rot0"],
                    dtype=np.float32)
    f32 = np_oracle.trace(c["table"], c["y0"], c["u0"], clip=c["clip"], rot0=c["rot0"],
                          dtype=np.float32)
    edge = name.startswith(FP32_EDGE)
    for a, o, b, w in zip(got, f32, (c["Y"], c["U"], c["I"], c["T"]), "yuit"):
        err, flips = _fp32_err(a, b)
        err_np, flips_np = _fp32_err(o, b)
        if edge:
            # mask-aware: the engine may flip no more rays than the reference's
            # formulas in float32 do, and stays within 2e-5 where both are finite
            assert flips <= max(flips_np, 3*len(c["table"])), (name, w, flips, flips_np)
            assert err <= max(2e-5, 1.5*err_np), (name, w, err, err_np)
        else:
            assert flips == 0, "%s fp32 %s: NaN mask differs at %d entries" % (name, w, flips)
            assert err <= max(FP32_RTOL, 1.5*err_np), "%s fp32 %s: %.2e (numpy float32 %.2e)" % (
                name, w, err, err_np)


@pytest.mark.parametrize("sysname", ["double_gauss", "cooke", "cooke_asph", "zoom"])
def test_fp32_large_bundles(eng, systems, sysname):
    """2e5-ray aimed bundles, FP32, per-surface comparator at 1e-5; rays within
    FP32 resolution of an aperture edge may flip (< 0.1 % of the entries)"""
    ent = systems[sysname]
    aim = ent["aim"][0][3]
    y0, u0 = aim_infinite(aim["field"], disc(200000, 9), aim["z"], aim["p"], ent["object_angle"])
    want = np_oracle.trace(ent["tables"][0], y0, u0, clip=True)
    got = eng.trace(ent["tables"][0], y0, u0, clip=True, dtype=np.float32)
    for a, b, w in zip(got, want, "yuit"):
        err, flips = _fp32_err(a, b)
        assert flips <= 1e-3*b.size, (sysname, w, flips)
        assert err <= FP32_RTOL, "%s fp32 %s: %.2e" % (sysname, w, err)


def test_store_paths_identical_large(eng, systems):
    """per-CTA bulk stores (default), per-warp bulk stores (rpt 1, 2) and
    per-thread stores give bit-identical arrays on a 70k-ray ragged bundle"""
    ent = systems["zoom"]
    table, aim = ent["tables"][1], ent["aim"][1][2]
    y0, u0 = aim_infinite(aim["field"], disc(70001, 9), aim["z"], aim["p"], ent["object_angle"])
    ref = eng.trace(table, y0, u0, clip=True, direct=True)
    for rpt in (0, 1, 2):
        got = eng.trace(table, y0, u0, clip=True, rpt=rpt)
        for x, y in zip(got, ref):
            assert np.array_equal(x, y, equal_nan=True), rpt
    last = eng.trace(table, y0, u0, clip=True, keep_last=True)
    for x, y in zip(last, ref):
        assert np.array_equal(x[0], y[-1], equal_nan=True)


@pytest.mark.parametrize("name", ["double_gauss_l0_clip", "cooke_asph_f07_clip",
                                  "tilted_clip1", "singlet_c1"])
def test_store_paths_identical(eng, name):
    """TMA bulk-store path == per-thread store path, bit for bit"""
    c = load_golden(name)
    for exact in (False, True):
        b = eng.trace(c["table"], c["y0"], c["u0"], clip=c["clip"], rot0=c["rot0"], exact=exact,
                      direct=True)
        for rpt in (1, 2):
            a = eng.trace(c["table"], c["y0"], c["u0"], clip=c["clip"], rot0=c["rot0"],
                          exact=exact, rpt=rpt)
            for x, y in zip(a, b):
                assert np.array_equal(x, y, equal_nan=True)


def test_keep_last_and_null_outputs(eng):
    c = load_golden("zoom_f1_clip")
    full = eng.trace(c["table"], c["y0"], c["u0"], clip=True)
    last = eng.trace(c["table"], c["y0"], c["u0"], clip=True, keep_last=True)
    for a, b in zip(full, last):
        assert b.shape[0] == 1
        assert np.array_equal(a[-1], b[0], equal_nan=True)
    y, u, i, t = eng.trace(c["table"], c["y0"], c["u0"], clip=True, want=("y",))
    assert u is None and i is None and t is None
    assert np.array_equal(y, full[0], equal_nan=True)


def test_device_arrays_any_pitch(eng):
    """rtx_trace on device buffers: ld = N (odd, direct stores) and ld
    padded to 64 (bulk stores) give the same rows"""
    c = load_golden("double_gauss_f1_noclip")
    N, S = c["y0"].shape[0] - 3, len(c["table"])     # odd N
    y0 = eng.to_device(c["y0"][:N])
    u0 = eng.to_device(c["u0"][:N])
    for ld in (N, 320):
        Y, U, I = (eng.empty((S, ld, 3)) for _ in range(3))
        T = eng.empty((S, ld))
        eng.trace_device(c["table"], y0, u0, Y, U, I, T, N=N, ld=ld, clip=False)
        eng.sync()
        assert_parity(Y.download()[:, :N], c["Y"][:, :N], FP64_RTOL, "Y ld=%d" % ld)
        assert_parity(U.download()[:, :N], c["U"][:, :N], FP64_RTOL, "U ld=%d" % ld)
        assert_parity(I.download()[:, :N], c["I"][:, :N], FP64_RTOL, "I ld=%d" % ld)
        assert_parity(T.download()[:, :N], c["T"][:, :N], FP64_RTOL, "T ld=%d" % ld)
        for a in (Y, U, I, T):
            a.free()


@pytest.mark.parametrize("sysname,n,clip", [("double_gauss", 300000, True),
                                            ("zoom", 200000, True),
                                            ("cooke_asph", 100000, True),
                                            ("cooke", 100000, False)])
def test_large_bundle_vs_oracle(eng, systems, sysname, n, clip):
    """sizes the oracle finishes in seconds: multi-chunk grid, ragged tail"""
    ent = systems[sysname]
    n += 37                                       # ragged: not a multiple of 32
    for li in range(min(2, len(ent["tables"]))):
        table = ent["tables"][li]
        aim = ent["aim"][li][3]                   # field (0, .7)
        y0, u0 = aim_infinite(aim["field"], disc(n, 5 + li), aim["z"], aim["p"],
                              ent["object_angle"])
        want = np_oracle.trace(table, y0, u0, clip=clip)
        newton = bool((table["n_asph"] >= 0).any())
        # default configuration: per-CTA TMA bulk stores (N > 32768), ragged tail
        got = eng.trace(table, y0, u0, clip=clip, exact=True)
        for a, b, w in zip(got, want, "yuit"):
            if newton:
                assert_parity(a, b, 1e-12, "%s exact %s" % (sysname, w))
            else:
                assert np.array_equal(a, b, equal_nan=True), (sysname, w)
        got = eng.trace(table, y0, u0, clip=clip, rpt=(0, 1, 2)[(li + len(sysname)) % 3])
        for a, b, w in zip(got, want, "yuit"):
            assert_parity(a, b, FP64_RTOL, "%s fast %s" % (sysname, w))


def test_known_answer_rms_through_dropin(eng):
    """rayopt/test/test_raytrace.py:192-195 through the CUDA path"""
    c = load_golden("cooke_radau13")
    Y, U, I, T = eng.trace(c["table"], c["y0"], c["u0"], exact=True)
    rms = np_oracle.rms(Y[-1], c["w"])
    assert abs(rms - 0.052)/0.052 < 1e-2
    assert rms == c["meta"]["rms"]
    q = load_golden("cooke_square500")                 # test_raytrace.py:196-199
    Yq = eng.trace(q["table"], q["y0"], q["u0"])[0]
    assert abs(np_oracle.rms(Yq[-1], q["w"]) - rms)/rms < 5e-2


def test_moments_and_device_rms(eng):
    c = load_golden("double_gauss_l1_clip")
    N = c["y0"].shape[0]
    Y = eng.to_device(c["Y"][-1])
    w = eng.to_device(np.full(N, 1.0/N))
    m = eng.moments(Y, w)
    y = c["Y"][-1, :, :2]
    good = np.isfinite(y).all(1)
    assert m[4] == good.sum() and m[5] == N
    np.testing.assert_allclose(m[0], good.sum()/N, rtol=1e-13)
    np.testing.assert_allclose(m[1:3], (y[good]/N).sum(0), rtol=1e-12, atol=1e-15)
    np.testing.assert_allclose(m[3], (np.square(y[good]).sum(1)/N).sum(), rtol=1e-12)
    np.testing.assert_allclose(m[6:8], y[good].sum(0), rtol=1e-12, atol=1e-13)
    # reference semantics: not NaN-masked
    assert np.isnan(eng.rms(Y, w))
    # the reference's known answer, on the device (test_raytrace.py:192-195)
    k = load_golden("cooke_radau13")
    Yk, wk = eng.to_device(k["Y"][-1]), eng.to_device(k["w"])
    rms = eng.rms(Yk, wk)
    assert abs(rms - k["meta"]["rms"]) < 1e-13 and abs(rms - 0.052)/0.052 < 1e-2
    assert abs(eng.rms(Yk, wk, ref_point=k["Y"][-1, 0, :2]) -
               np_oracle.rms(k["Y"][-1], k["w"], ref=0)) < 1e-13


def test_empty_and_bad_arguments(eng):
    c = load_golden("singlet_c1")
    out = eng.trace(c["table"], np.zeros((0, 3)), np.zeros((0, 3)))
    assert out[0].shape == (3, 0, 3)
    from rayopt_b200._lib import RtxError
    bad = c["table"].copy()
    bad["n_asph"][0] = 99
    with pytest.raises(RtxError):
        eng.trace(bad, c["y0"], c["u0"])
    with pytest.raises(RtxError):
        eng.trace(c["table"], c["y0"], c["u0"], dtype=np.float32, exact=True)


def test_round_trip_properties_full_size(eng, systems):
    """size-independent properties at a BASELINE-scale bundle (1e7 rays, 12
    surfaces, FP64): directions stay unit length, intercepts lie on their
    surfaces (sag residual), optical path is additive, NaN is absorbing."""
    ent = systems["double_gauss"]
    table = ent["tables"][0]
    aim = ent["aim"][0][3]
    n = 10_000_000
    y0, u0 = aim_infinite(aim["field"], disc(n, 0), aim["z"], aim["p"], ent["object_angle"])
    S = len(table)
    d_y0, d_u0 = eng.to_device(y0), eng.to_device(u0)
    ld = ((n + 63)//64)*64
    Y, U = eng.empty((S, ld, 3)), eng.empty((S, ld, 3))
    eng.trace_device(table, d_y0, d_u0, Y, U, None, None, N=n, ld=ld, clip=True)
    eng.sync()
    rng = np.random.default_rng(0)
    for j in (0, 4, 5, S - 1):
        y = Y.rows(j).download()[0, :n]
        u = U.rows(j).download()[0, :n]
        ok = np.isfinite(u[:, 0])
        # unit directions (refract keeps |u| = 1 to ~2e-16, SURVEY 8a13)
        assert np.abs(np.square(u[ok]).sum(1) - 1).max() < 1e-13
        # intercepts on the surface
        res = np_oracle.surface_sag(table[j], y[np.isfinite(y[:, 0])][::97])
        assert np.abs(res).max() < 1e-11
        if j == S - 1:
            assert 0.90 < ok.mean() < 0.97        # ~6 % vignetted (SURVEY 8d)
    # a sample against the oracle
    idx = rng.choice(n, 5000, replace=False)
    want = np_oracle.trace(table, y0[idx], u0[idx], clip=True)
    got_y = np.stack([Y.rows(j).download()[0][idx] for j in range(S)])
    assert_parity(got_y, want[0], FP64_RTOL, "1e7 sample y")
    for a in (Y, U, d_y0, d_u0):
        a.free()


def test_sharded_trace_single_rank(eng):
    """rayopt_b200.sharding on the CUDA engine (world of one); the two-rank
    gloo variant of the same class runs on CPU in tests/test_sharding_gloo.py"""
    from rayopt_b200.sharding import ShardedTrace
    c = load_golden("double_gauss_f1_noclip")
    st = ShardedTrace(engine=eng)
    spot = st.spot(c["table"], c["y0"], c["u0"], clip=False)
    assert_parity(spot[None], c["Y"][-1:], FP64_RTOL, "sharded spot")
    assert abs(st.rms(c["table"], c["y0"], c["u0"]) - np_oracle.rms(c["Y"][-1])) < 1e-12


def test_element_level_entry_points(eng):
    """rayopt_b200.elements.{propagate,intercept,refract} on the CUDA engine
    against the oracle's single-surface functions (elements.py:306-315 etc.)"""
    from rayopt_b200 import elements as el
    c = load_golden("conics_clip1")
    rec = c["table"][1]

    class E:
        curvature, conic = float(rec["c"]), float(rec["k"])
        aspherics, alternate_intersection = None, False
        radius = float(np.sqrt(rec["radius2"]))

        def get_n_mu(self, n0, l):
            return float(rec["n"]), n0/float(rec["n"])
    rng = np.random.default_rng(2)
    y0 = np.c_[rng.uniform(-3, 3, (500, 2)), -np.ones(500)]
    u0 = rng.normal(0, .1, (500, 2))
    u0 = np.c_[u0, np.sqrt(1 - np.square(u0).sum(1))]
    n0 = float(rec["n0"])
    one = np.zeros(1, c["table"].dtype)
    from rayopt_b200.surface_table import pack_element

    class Bare(E):
        offset, rotated = (0., 0., 0.), False
    pack_element(one[0], Bare(), n0, None)
    wy, wu, wt = np_oracle.propagate_surface(one[0], y0, u0, True)
    y, u, n, t = el.propagate(E(), y0, u0, n0, None, clip=True, engine=eng, exact=True)
    assert n == float(rec["n"])
    for a, b in ((y, wy), (u, wu), (t, wt)):
        assert np.array_equal(a, b, equal_nan=True)
    s = el.intercept(E(), y0, u0, engine=eng, exact=True)
    assert np.array_equal(s, np_oracle.intercept(one[0], y0, u0), equal_nan=True)
    on = np.isfinite(wy[:, 0])
    r = el.refract(E(), wy[on], u0[on], float(one["mu"][0]), engine=eng)
    assert_parity(r[None], np_oracle.refract(one[0], wy[on], u0[on])[None], FP64_RTOL, "refract")


@pytest.mark.parametrize("with_i", [False, True])
@pytest.mark.parametrize("n,off", [(70016, 192), (70001, 192), (3000, 64), (1000, 5)])
def test_trace_gather_epilogue(eng, systems, n, off, with_i):
    """rtx_trace_gather: the last surface's intercepts (and, optionally, its
    incidence directions -- analysis.py:274-280 reads both) are stored by the
    trace kernel itself into several gather buffers at a ray offset (here two
    local buffers stand in for peer GPUs; the NVLink runs are bench.py's C4 leg
    and tests/gpu_scripts/multi_gpu_check.py).  Whatever N and the offset --
    whole 64-ray groups (bulk stores) or ragged (per-ray fallback) -- EXACTLY
    rays off .. off+N-1 are written: a shard never spills into its neighbour."""
    ent = systems["double_gauss"]
    table, aim = ent["tables"][0], ent["aim"][0][3]
    y0, u0 = aim_infinite(aim["field"], disc(n, 4), aim["z"], aim["p"], ent["object_angle"])
    ref_y, _, ref_i, _ = eng.trace(table, y0, u0, clip=True, keep_last=True)
    npad = (off + n + 63)//64*64 + 64
    bufs = [eng.empty((npad, 3)) for _ in range(2)]
    bufs_i = [eng.empty((npad, 3)) for _ in range(2)] if with_i else None
    for b in bufs + (bufs_i or []):
        eng.lib.rtx_memset(eng.ctx, b.ptr, 0xff, b.nbytes)
    d_y0, d_u0 = eng.to_device(y0), eng.to_device(u0)
    eng.trace_gather(table, d_y0, d_u0, [b.ptr for b in bufs], off, clip=True,
                     dst_i_ptrs=[b.ptr for b in bufs_i] if with_i else None)
    eng.sync()
    for group, ref in ((bufs, ref_y[0]), (bufs_i or [], ref_i[0])):
        for b in group:
            h = b.download()
            assert np.array_equal(h[off:off + n], ref, equal_nan=True)
            assert np.isnan(h[:off]).all()            # nothing written in front of the shard
            assert np.isnan(h[off + n:]).all()        # ... nor behind it
            b.free()
    # (x,y)-only gather (RTX_GATHER_XY): (N,2) buffers, same rays, same guarantees
    bxy = [eng.empty((npad, 2)) for _ in range(2)]
    for b in bxy:
        eng.lib.rtx_memset(eng.ctx, b.ptr, 0xff, b.nbytes)
    eng.trace_gather(table, d_y0, d_u0, [b.ptr for b in bxy], off, clip=True, xy=True)
    eng.sync()
    for b in bxy:
        h = b.download()
        assert np.array_equal(h[off:off + n], ref_y[0][:, :2], equal_nan=True)
        assert np.isnan(h[:off]).all() and np.isnan(h[off + n:]).all()
        b.free()
    d_y0.free()
    d_u0.free()


def test_memory_helpers_and_numa(eng):
    """rtx_memcpy_d2d, page-locked arrays that outlive their owner, and
    rtx_numa_bind (bind + restore; a platform that reports no node is fine)"""
    import gc
    import os
    a = np.arange(30, dtype=np.float64).reshape(10, 3)
    d1, d2 = eng.to_device(a), eng.empty((10, 3))
    d2.copy_from(d1)
    assert np.array_equal(d2.download(), a)
    assert np.array_equal(eng.download_rays(d2, np.arange(1, 10, 3)), a[1:10:3])
    assert np.array_equal(eng.download_rays(d2, [7, 2, 2]), a[[7, 2, 2]])
    p = eng.pinned_empty((4, 1000, 3))
    p[:] = 3.
    row = p[2]
    del p
    gc.collect()
    assert row.sum() == 9000.                 # the view keeps the allocation alive
    before = os.sched_getaffinity(0)
    node = eng.numa_bind(True)
    assert node >= -1 and len(os.sched_getaffinity(0)) >= 1
    q = eng.pinned_empty((1000, 3))           # allocated under the binding
    q[:] = 1.
    eng.numa_bind(False)
    assert os.sched_getaffinity(0) == before
    assert q.sum() == 3000.


def test_device_refocus_shift(eng):
    """Engine.refocus_shift == the shift GeometricTrace.refocus computes
    (geometric_trace.py:82-99) on host arrays"""
    c = load_golden("double_gauss_l0_clip")
    at = -2
    y, i, w = c["Y"][at], c["I"][at], c["w"]
    u = i[:, :2]/i[:, 2:]
    good = np.all(np.isfinite(u), axis=1)
    yg, ug, wg = y[good, :2], u[good], w[good]
    yg = yg - yg.mean(0)
    ug = ug - ug.mean(0)
    want = -np.dot((wg[:, None]*yg).ravel(), ug.ravel())/np.dot((wg[:, None]*ug).ravel(), ug.ravel())
    got = eng.refocus_shift(eng.to_device(y), eng.to_device(i), eng.to_device(w))
    assert abs(got - want) <= 1e-11*abs(want)


def test_limits_and_degenerate_sizes(eng):
    """N = 1, S = 1, the maximum table (S = 256) and the argument errors"""
    from rayopt_b200._lib import RtxError
    c = load_golden("cooke_single_ray")
    got = eng.trace(c["table"], c["y0"], c["u0"], exact=True)
    for a, b in zip(got, (c["Y"], c["U"], c["I"], c["T"])):
        assert np.array_equal(a, b, equal_nan=True)
    one = eng.trace(c["table"][:1], c["y0"], c["u0"], exact=True)
    assert np.array_equal(one[0][0], c["Y"][0])
    # 256 surfaces: a stack of thin plane-parallel plates (alternating n)
    big = np.zeros(256, c["table"].dtype)
    big["rot"] = np.eye(3).reshape(9)
    big["offset"][:, 2] = .01
    big["radius2"] = np.inf
    big["n_asph"] = -1
    nn = np.where(np.arange(256) % 2 == 0, 1.5, 1.0)
    n0 = np.r_[1.0, nn[:-1]]
    big["n0"], big["n"] = n0, nn
    big["mu"] = n0/nn
    big["muf"], big["sgn"], big["mu2m1"] = np.abs(big["mu"]), np.sign(big["mu"]), big["mu"]**2 - 1
    rng = np.random.default_rng(0)
    y0 = np.c_[rng.normal(0, 1, (5000, 2)), np.zeros(5000)]
    u0 = rng.normal(0, .1, (5000, 2))
    u0 = np.c_[u0, np.sqrt(1 - np.square(u0).sum(1))]
    want = np_oracle.trace(big, y0, u0)
    got = eng.trace(big, y0, u0, exact=True)
    for a, b in zip(got, want):
        assert np.array_equal(a, b, equal_nan=True)
    with pytest.raises(RtxError):
        eng.trace(np.concatenate([big, big[:1]]), y0, u0)          # 257 surfaces
    with pytest.raises(ValueError):
        eng.trace(big, y0[:, :2], u0[:, :2])                       # not (N, 3)


@pytest.mark.parametrize("n", [1000, 70001])
def test_vignetting_mask_ballot(eng, systems, n):
    """rtx_set_mask_output: the warp-ballot mask equals isfinite(u[-1]) of the
    reference trace, also when nothing else is stored"""
    ent = systems["double_gauss"]
    table, aim = ent["tables"][2], ent["aim"][2][3]          # field 0.7: ~5 % vignetted
    y0, u0 = aim_infinite(aim["field"], disc(n, 3), aim["z"], aim["p"], ent["object_angle"])
    want = np.isfinite(np_oracle.trace(table, y0, u0, clip=True)[1][-1, :, 0])
    assert 0 < want.mean() < 1
    d_y0, d_u0 = eng.to_device(y0), eng.to_device(u0)
    mask = eng.empty(((n + 31)//32,), np.uint32)
    for keep in ("last", "none"):
        eng.lib.rtx_memset(eng.ctx, mask.ptr, 0, mask.nbytes)
        Y = eng.empty((1, (n + 63)//64*64, 3)) if keep == "last" else None
        eng.trace_device(table, d_y0, d_u0, Y, None, None, None, N=n, clip=True, keep_last=True,
                         mask=mask)
        eng.sync()
        bits = np.unpackbits(mask.download().view(np.uint8), bitorder="little")[:n].astype(bool)
        assert np.array_equal(bits, want)
    check_off = eng.empty((2, 64, 3))
    eng.trace_device(table[:2], eng.to_device(y0[:10]), eng.to_device(u0[:10]), check_off, None,
                     None, None, N=10, clip=True)            # mask switched off again
    eng.sync()


def test_resident_trace_lazy_rows(eng, systems):
    """ResidentTrace: results stay in HBM, rows come to the host on demand,
    sub-range propagate starts from the resident row, rms never moves rays"""
    from rayopt_b200 import PackedSystem, ResidentTrace
    ent = systems["double_gauss"]
    ps = PackedSystem(ent["wavelengths"], ent["tables"], [n[0] for n in ent["n"]])
    c = load_golden("double_gauss_l0_clip")
    g = ResidentTrace(ps, engine=eng, exact=True)
    g.rays_given(c["y0"], c["u0"], l=ent["wavelengths"][0], w=c["w"])
    g.propagate(clip=True)
    assert g.y.fetched_bytes == 0                     # nothing copied yet
    assert np.array_equal(g.y[-1], c["Y"][-1], equal_nan=True)
    assert np.array_equal(g.y[-1, :, :2], c["Y"][-1, :, :2], equal_nan=True)
    assert np.array_equal(g.i[-1], c["I"][-1], equal_nan=True)
    assert g.y.fetched_bytes == g._ld*24 and g.u.fetched_bytes == 0
    assert np.array_equal(g.y[0], c["y0"]) and np.array_equal(g.u[0], c["u0"])
    assert np.array_equal(np.asarray(g.t)[1:], c["T"], equal_nan=True)
    assert np.array_equal(g.u[3:5], c["U"][2:4], equal_nan=True)
    assert np.array_equal(g.n[1:], c["n"])
    # sub-range re-trace from a resident row (geometric_trace.py:72-80)
    c2 = load_golden("double_gauss_sub_4_9")
    g2 = ResidentTrace(ps, engine=eng, exact=True)
    g2.rays_given(c2["y0"], c2["u0"], l=ent["wavelengths"][0])   # any rays: rows are overwritten
    g2.y.set_row(3, np.pad(c2["y0"], ((0, g2._ld - len(c2["y0"])), (0, 0))))
    g2.u.set_row(3, np.pad(c2["u0"], ((0, g2._ld - len(c2["u0"])), (0, 0))))
    g2.n[3] = c2["table"]["n0"][0]
    g2.propagate(start=4, stop=9, clip=True)
    assert np.array_equal(g2.y[4:9], c2["Y"], equal_nan=True)
    assert np.array_equal(g2.t[4:9], c2["T"], equal_nan=True)
    # device rms == reference rms on the surviving rays
    k = load_golden("cooke_radau13")
    pk = PackedSystem([587.56e-9], [k["table"]], [k["table"]["n0"][0]])
    gk = ResidentTrace(pk, engine=eng, exact=True)
    gk.rays_given(k["y0"], k["u0"], l=587.56e-9, w=k["w"])
    gk.propagate()
    assert abs(gk.rms() - k["meta"]["rms"]) < 1e-13 and gk.y.fetched_bytes == 0
    # launch rays generated in HBM: same trace as from host rays
    aim = ent["aim"][0][3]
    gd = ResidentTrace(ps, engine=eng, exact=True)
    gd.rays_infinite(aim["field"], aim["z"], aim["p"], ent["object_angle"],
                     l=ent["wavelengths"][0], nrays=3000)
    gd.propagate(clip=True)
    gh = ResidentTrace(ps, engine=eng, exact=True)
    gh.rays_given(gd.y[0], gd.u[0], l=ent["wavelengths"][0])
    gh.propagate(clip=True)
    assert np.array_equal(gd.y[-1], gh.y[-1], equal_nan=True)
    assert np.array_equal(gd.i[0], gd.u[0])
    for t in (g, g2, gk, gd, gh):
        t.free()


def test_device_ray_generation(eng, systems):
    """rtx_aim_infinite: launch rays generated in HBM equal the host
    restatement of InfiniteConjugate.aim (rayopt_b200/rays.py, itself
    bit-identical to the reference): bit for bit for given pupil coordinates,
    to the last ulps of sin/cos for the on-the-fly hexapolar grid; traced, they
    agree with the oracle to 1e-10."""
    from rayopt_b200.rays import hexapolar
    ent = systems["double_gauss"]
    table, aim = ent["tables"][0], ent["aim"][0][3]
    yp = disc(5001, 3)
    hy, hu = aim_infinite(aim["field"], yp, aim["z"], aim["p"], ent["object_angle"])
    dy, du = eng.aim_infinite_device(aim["field"], aim["z"], aim["p"], ent["object_angle"],
                                     yp=eng.to_device(yp))
    eng.sync()
    assert np.array_equal(dy.download(), hy) and np.array_equal(du.download(), hu)
    rings, xy = hexapolar(30000)
    hy, hu = aim_infinite(aim["field"], xy, aim["z"], aim["p"], ent["object_angle"])
    dy, du = eng.aim_infinite_device(aim["field"], aim["z"], aim["p"], ent["object_angle"],
                                     nrays=30000)
    eng.sync()
    assert dy.shape == hy.shape == (1 + 3*rings*(rings + 1), 3)
    np.testing.assert_allclose(dy.download(), hy, rtol=0, atol=2e-14)
    assert np.array_equal(du.download(), hu)
    n = hy.shape[0]
    ld = (n + 63)//64*64
    Y = eng.empty((len(table), ld, 3))
    eng.trace_device(table, dy, du, Y, None, None, None, N=n, ld=ld, clip=True)
    eng.sync()
    want = np_oracle.trace(table, hy, hu, clip=True)[0]
    assert_parity(Y.download()[:, :n], want, FP64_RTOL, "device-generated bundle")


def test_path_sum_output(eng):
    """rtx_set_path_sum_output: per-ray sum of the optical path over the
    first surfaces, as GeometricTrace.opd accumulates it (geometric_trace.py:102)"""
    c = load_golden("zoom_f1_clip")
    n, S = c["y0"].shape[0], len(c["table"])
    d_y0, d_u0 = eng.to_device(c["y0"]), eng.to_device(c["u0"])
    acc = eng.empty((n,))
    for upto in (-1, S - 3, 0):
        eng.trace_device(c["table"], d_y0, d_u0, None, None, None, None, N=n, clip=True,
                         exact=True, path_sum=acc, path_sum_upto=upto)
        eng.sync()
        k = S if upto < 0 else upto + 1
        want = np.zeros(n)
        for j in range(k):                 # same left-to-right order as the kernel
            want = want + c["T"][j]
        assert np.array_equal(acc.download(), want, equal_nan=True), upto


def test_pitch_of_32_ray_groups(eng, systems):
    """ld a multiple of 32 but not of 64, N > 32768: one-ray-per-thread bulk
    stores; same rows as the default configuration"""
    ent = systems["zoom"]
    table, aim = ent["tables"][0], ent["aim"][0][1]
    n = 40000
    y0, u0 = aim_infinite(aim["field"], disc(n, 6), aim["z"], aim["p"], ent["object_angle"])
    d_y0, d_u0 = eng.to_device(y0), eng.to_device(u0)
    S = len(table)
    out = {}
    for ld in (40032, 40064):
        Y, T = eng.empty((S, ld, 3)), eng.empty((S, ld))
        eng.trace_device(table, d_y0, d_u0, Y, None, None, T, N=n, ld=ld, clip=True, exact=True)
        eng.sync()
        out[ld] = (Y.download()[:, :n], T.download()[:, :n])
        Y.free(), T.free()
    for a, b in zip(out[40032], out[40064]):
        assert np.array_equal(a, b, equal_nan=True)
    want = np_oracle.trace(table, y0, u0, clip=True)
    assert np.array_equal(out[40032][0], want[0], equal_nan=True)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_batched_bundles_one_launch(eng, systems, dtype):
    """rtx_trace_batch: three wavelength bundles of different (ragged) sizes in
    ONE launch give exactly the arrays of three separate launches"""
    ent = systems["double_gauss"]
    ns = [70001, 40000, 99999]
    S = ent["S"]
    ld = (max(ns) + 63)//64*64
    rays, single, outs = [], [], []
    for li, n in enumerate(ns):
        aim = ent["aim"][li][3]
        y0, u0 = aim_infinite(aim["field"], disc(n, 20 + li), aim["z"], aim["p"], ent["object_angle"])
        d = (eng.to_device(y0, dtype), eng.to_device(u0, dtype))
        rays.append(d)
        ref = [eng.empty((S, ld, 3), dtype) for _ in range(3)] + [eng.empty((S, ld), dtype)]
        eng.trace_device(ent["tables"][li], d[0], d[1], *ref, N=n, ld=ld, clip=True)
        single.append(ref)
        outs.append([eng.empty((S, ld, 3), dtype) for _ in range(3)] + [eng.empty((S, ld), dtype)])
    eng.trace_device_batch(ent["tables"][:3], [r[0] for r in rays], [r[1] for r in rays],
                           [o[0] for o in outs], [o[1] for o in outs], [o[2] for o in outs],
                           [o[3] for o in outs], Ns=ns, ld=ld, clip=True)
    eng.sync()
    for n, a, b in zip(ns, single, outs):
        for x, y in zip(a, b):
            assert np.array_equal(x.download()[:, :n], y.download()[:, :n], equal_nan=True)
    for group in single + outs:
        for a in group:
            a.free()


def test_device_ray_generation_finite(eng):
    """rtx_aim_finite vs the host restatement of FiniteConjugate.aim (which is
    bit-identical to the reference): to the last ulps of tan()"""
    from rayopt_b200.rays import aim_finite, hexapolar
    p = np.array(((-3., -2.5), (3., 2.5)))
    for z in (50., -40.):
        yp = disc(4001, 8)
        hy, hu = aim_finite((.3, -.4), yp, z, p, 5.)
        dy, du = eng.aim_finite_device((.3, -.4), z, p, 5., yp=eng.to_device(yp))
        eng.sync()
        assert np.array_equal(dy.download(), hy)
        np.testing.assert_allclose(du.download(), hu, rtol=0, atol=4e-16)
        rings, xy = hexapolar(3000)
        hy, hu = aim_finite((0, .7), xy, z, p, 5.)
        dy, du = eng.aim_finite_device((0, .7), z, p, 5., nrays=3000)
        eng.sync()
        np.testing.assert_allclose(du.download(), hu, rtol=0, atol=5e-15)
        assert np.allclose(np.square(du.download()).sum(1), 1, rtol=0, atol=2e-15)
