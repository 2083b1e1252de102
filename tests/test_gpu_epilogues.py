"""The fused trace epilogues (rtx_trace_reduce, rtx_trace_opd) and the moment
reductions on stored rows (rtx_moments, rtx_focus_moments) against an exact
restatement of their contracts (oracle/epi_oracle.py).  Needs a GPU.

The epilogue kernel is a second copy of the march.  Its per-ray state at the
last surface is the state rtx_trace stores, which the parity and cluster tests
pin bit for bit across kernel configurations.  So each case traces the same
launch rays with rtx_trace and checks the epilogues against the stored rows:

* moments: the counts m[4], m[5], m[8] exactly; every sum within
  (L + 64) eps sum|term| of the exact sum, L the longest serial chain of the
  kernel's summation (tiles per CTA, or rays per thread, plus the CTAs that
  meet in the atomics), 64 covering the warp and CTA trees and the rounding
  of the terms themselves; the derived rms and focus shift to 1e-12 / 1e-10;
* OPD: A and P bit for bit, since the epilogue uses only separately rounded
  operations on the stored state and rtx_set_path_sum_output's sum.

The reduce sums through atomicAdd, so it is not asserted to repeat bit for bit.

This holds for Newton (aspheric) systems in fast FP64 and FP32 mode too, with
no per-ray allowance.  The one-ray-per-thread trace kernel used to differ
there from the two- and four-ray kernels and from the epilogue by a few ulps
for a few rays in a thousand: the Newton slope's r2 = x*x + y*y (and the
normal's q_x^2 + q_y^2 + 1) were plain expressions, and the compiler fused a
different one of the two products in that kernel.  Both are now written with
one explicit rounded product and one FMA (rtx_device.cuh, sumsq2_fast);
tests/test_gpu_config_invariance.py pins every configuration to the same bits.
"""
import ctypes as C

import numpy as np
import pytest

import epi_oracle
import np_oracle
from conftest import load_golden
from rayopt_b200.rays import aim_infinite, disc

pytestmark = pytest.mark.gpu

EPS = 2.0**-52
NS = [0, 1, 31, 32, 33, 63, 64, 65, 511, 512, 513, 70001, 1000003]
MODES = {"f64_exact": (np.float64, True), "f64_fast": (np.float64, False),
         "f32": (np.float32, False)}
SYSTEMS = ["double_gauss", "cooke_asph", "mirror", "tilted_start3", "zoom", "plates256", "s1"]


@pytest.fixture(scope="module")
def eng():
    from rayopt_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def _plates(S=256):
    """a stack of thin plane-parallel plates (alternating n): its FP64 table
    (92 KB) and its FP32 table (48 KB + 16 bytes) are both over 48 KB, so
    the epilogue launch opts into more shared memory in both dtypes"""
    from rayopt_b200.surface_table import SURFACE_DTYPE
    big = np.zeros(S, SURFACE_DTYPE)
    big["rot"] = np.eye(3).reshape(9)
    big["offset"][:, 2] = .01
    big["radius2"] = np.inf
    big["n_asph"] = -1
    nn = np.where(np.arange(S) % 2 == 0, 1.5, 1.0)
    n0 = np.r_[1.0, nn[:-1]]
    big["n0"], big["n"] = n0, nn
    big["mu"] = n0/nn
    big["muf"], big["sgn"], big["mu2m1"] = np.abs(big["mu"]), np.sign(big["mu"]), big["mu"]**2 - 1
    return big


def _system(name, systems):
    """(table, rot0, clip, rays(n, seed) -> (y0, u0) float64)"""
    if name == "plates256":
        def rays(n, seed):
            rng = np.random.default_rng(seed)
            u = rng.normal(0, .1, (n, 2))
            return np.c_[rng.normal(0, 1, (n, 2)), np.zeros(n)], \
                np.c_[u, np.sqrt(1 - np.square(u).sum(1))]
        return _plates(), None, False, rays
    if name == "tilted_start3":
        c = load_golden(name)

        def rays(n, seed):
            k = np.random.default_rng(seed).integers(0, len(c["y0"]), n)
            return c["y0"][k], c["u0"][k]
        return c["table"], c["rot0"], c["clip"], rays
    key, fi, clip = {"double_gauss": ("double_gauss", 3, True),      # field 0.7, vignetted
                     "cooke_asph": ("cooke_asph", 3, True),
                     "mirror": ("mirror", 3, False),                  # last surface rotated
                     "zoom": ("zoom", 3, True),
                     "s1": ("cooke", 3, False)}[name]
    ent = systems[key]
    table, aim = ent["tables"][0], ent["aim"][0][fi]
    if name == "s1":
        table = table[:1]

    def rays(n, seed):
        return aim_infinite(aim["field"], disc(n, seed), aim["z"], aim["p"], ent["object_angle"])
    return table, None, clip, rays


def _L_epi(eng, N):
    """longest serial chain of epi_kernel's sum: tiles per CTA + CTAs (any
    occupancy up to 8 CTAs of 256 threads per SM)"""
    tiles = max(-(-N//512), 1)
    return -(-tiles//min(eng.sm_count, tiles)) + min(8*eng.sm_count, tiles)


def _L_mom(eng, N):
    """same for moments_kernel / focus_moments_kernel: rays per thread + CTAs"""
    blocks = max(min(-(-N//256), 8*eng.sm_count), 1)
    return -(-N//(256*blocks)) + blocks


def _within(got, want, scale, L, what):
    """|got - want| <= (L + 64) eps scale elementwise (NaN where want is NaN).
    Returns the worst ratio to the bound"""
    got, want, scale = (np.asarray(a, np.float64) for a in (got, want, scale))
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan), (what, got, want)
    tol = (L + 64)*EPS*scale[~nan]
    err = np.abs(got[~nan] - want[~nan])
    assert np.all(err <= tol), (what, np.flatnonzero(~nan)[err > tol], got, want)
    return float(np.max(err/np.where(tol > 0, tol, 1), initial=0.))


def _rel(a, b, rtol, what):
    if np.isnan(b):
        assert np.isnan(a), (what, a, b)
    else:
        assert abs(a - b) <= rtol*abs(b), (what, a, b, abs(a - b)/abs(b))


def _derived(m, s, a, unit_weights, center, rtol_rms, rtol_shift, what):
    """rms_from_moments and focus_shift_from_moments of m against those of the
    exact sums s.  Only about the chief ray's centre, where the one-pass
    formulas are cancellation free (about the origin they lose (|mean| /
    rms)^2 ulps), and only where the quantity is defined to that accuracy:
    a spot wider than rounding (not a single ray), slopes that differ (not a
    bundle of parallel rays, whose shift is 0/0)"""
    from rayopt_b200.engine import Engine
    if center is None:
        return
    if s[5] >= 64:
        _rel(Engine.rms_from_moments(m, unit_weights=unit_weights),
             Engine.rms_from_moments(s, unit_weights=unit_weights), rtol_rms, "rms " + what)
    G = s[8]
    if G >= 64:
        bu = s[11:13]/G
        den = s[19] - 2*bu.dot(s[16:18]) + bu.dot(bu)*s[13]
        if abs(den) > 1e-6*a[19]:
            _rel(Engine.focus_shift_from_moments(m), Engine.focus_shift_from_moments(s),
                 rtol_shift, "shift " + what)


def _focus_moments(eng, y, inc, w, N, center):
    """the raw 8 sums of rtx_focus_moments"""
    from rayopt_b200._lib import check
    m = np.zeros(8)
    c = None if center is None else np.ascontiguousarray(center, np.float64)
    check(eng.lib.rtx_focus_moments(eng.ctx, 0 if y.dtype == np.float64 else 1, N, y.ptr, inc.ptr,
                                    None if w is None else w.ptr,
                                    None if c is None else c.ctypes.data_as(C.c_void_p),
                                    m.ctypes.data_as(C.c_void_p)))
    return m


def _stored(eng, table, dy0, du0, N, dtype, exact, clip, rot0, rows="last", path_sum=False):
    """rtx_trace of the same launch rays: host y, u, i rows (last or all) and
    the path sum over all marched surfaces"""
    S = len(table)
    ld = (max(N, 1) + 63)//64*64
    R = 1 if rows == "last" else S
    Y, U, I = (eng.empty((R, ld, 3), dtype) for _ in range(3))
    ps = eng.empty((max(N, 1),), dtype) if path_sum else None
    eng.trace_device(table, dy0, du0, Y, U, I, None, N=N, ld=ld, clip=clip,
                     keep_last=rows == "last", rot0=rot0, exact=exact, path_sum=ps)
    eng.sync()
    out = [a.download()[:, :N] for a in (Y, U, I)]
    p = ps.download()[:N] if path_sum else None
    for a in (Y, U, I) + ((ps,) if path_sum else ()):
        a.free()
    return out + [p]


def _check_reduce(eng, table, dy0, du0, N, dtype, exact, clip, rot0, w, center, y, inc):
    """rtx_trace_reduce and rtx_moments / rtx_focus_moments on the stored rows
    against the exact sums of the stored rows; returns the worst ratio"""
    m = eng.trace_reduce(table, dy0, du0, N=N, clip=clip, rot0=rot0, exact=exact,
                         w=w, center=center)
    wh = None if w is None else w.download()[:N]
    s, a = epi_oracle.reduce_sums(y, inc, wh, center)
    for k in (4, 5, 8):
        assert m[k] == s[k], (k, m[k], s[k])
    worst = _within(m, s, a, _L_epi(eng, N), "trace_reduce")
    _derived(m, s, a, w is None, center, 1e-12, 1e-10, "vs stored rows")
    # the same sums from the stored rows by the two stand-alone kernels
    if N:
        dy, di = eng.to_device(y, dtype), eng.to_device(inc, dtype)
        cy = None if center is None else np.asarray(center)[:2]
        mm = eng.moments(dy, w, N=N, center=cy)
        assert mm[4] == s[4] and mm[5] == s[5]
        worst = max(worst, _within(mm, s[:8], a[:8], _L_mom(eng, N), "moments"))
        fm = _focus_moments(eng, dy, di, w, N, center)
        fs = np.r_[s[8], s[5], s[9:13], s[18:20]]
        fa = np.r_[a[8], a[5], a[9:13], a[18:20]]
        assert fm[0] == fs[0] and fm[1] == fs[1]
        worst = max(worst, _within(fm, fs, fa, _L_mom(eng, N), "focus_moments"))
        dy.free(), di.free()
    return m, s, worst


def _spec(y0, u0, y_last, n0, n_after, infinite, tilt):
    """an rtx_opd record for a table without a System: the sphere centred on
    ray 0's intercept, optionally seen through a tilted frame M"""
    ca, sa = np.cos(tilt), np.sin(tilt)
    M = np.array([[1, 0, 0], [0, ca, sa], [0, -sa, ca]])
    ref = np.nan_to_num(np.asarray(y_last[0], np.float64))
    return dict(y0_ref=np.asarray(y0[0], np.float64), u0_ref=np.asarray(u0[0], np.float64),
                n0=n0, n_after=n_after, M=M.reshape(9), d=-(ref @ M) + (.01, -.02, .03),
                radius=-60.0 if infinite else 45.0, infinite=int(infinite))


LAMBDA = 587.56e-6    # l/scale of the d line in mm: OPD in waves


def _check_opd(eng, table, dy0, du0, y0, u0, N, dtype, exact, clip, rot0, k):
    """A and P of rtx_trace_opd bit for bit against opd_epilogue of the stored
    rows and path sum (the tilted input plane and the tilted frame M every
    other case); in FP64 also the reference's operation order, to 1e-9 waves
    (eps |A| / l is about 1e-10 for paths of ~100 mm)"""
    if N:
        Y, U, _, ps = _stored(eng, table, dy0, du0, N, dtype, exact, clip, rot0, path_sum=True)
    spec = _spec(y0, u0, Y[0] if N else np.zeros((1, 3)), 1.0, float(table["n"][-1]) or 1.0,
                 k % 2 == 0, .02*(k % 3))
    A, P = eng.empty((max(N, 1),), dtype), eng.empty((max(N, 1), 3), dtype)
    eng.memset(A, 0x7f)
    eng.memset(P, 0x7f)
    sentinel = A.download(), P.download()
    n0 = eng.launch_count()
    eng.trace_opd(table, dy0, du0, spec, A, P, N=N, clip=clip, rot0=rot0, exact=exact)
    eng.sync()
    a, p = A.download(), P.download()
    A.free(), P.free()
    if N == 0:
        assert eng.launch_count() == n0
        assert np.array_equal(a, sentinel[0]) and np.array_equal(p, sentinel[1])
        return
    wa, wp = epi_oracle.opd_epilogue(y0[:N].astype(dtype), Y[0], U[0], ps, spec)
    assert a.dtype == wa.dtype
    assert np.array_equal(a[:N], wa, equal_nan=True), np.flatnonzero(
        ~((a[:N] == wa) | (np.isnan(a[:N]) & np.isnan(wa))))[:8]
    assert np.array_equal(p[:N], wp, equal_nan=True)
    if dtype == np.float64 and N <= 70001:
        T = eng.trace(table, y0[:N], u0[:N], clip=clip, rot0=rot0, exact=exact, want=("t",))[3]
        T = np.vstack([np.zeros((1, N)), T])            # row 0: the launch, t = 0
        x, yy, t = epi_oracle.opd_reference_order(
            T, 0, y0[:N], u0[:N], spec["n0"], spec["n_after"], Y[0], U[0],
            np.reshape(spec["M"], (3, 3)), None, np.asarray(spec["d"]), np.zeros(3), np.zeros(3),
            spec["radius"], spec["infinite"], LAMBDA)
        got = -(a[:N] - a[0])/LAMBDA
        assert np.array_equal(np.isnan(got), np.isnan(t))
        ok = ~np.isnan(t)
        assert np.all(np.abs(got[ok] - t[ok]) <= 1e-9), np.abs(got[ok] - t[ok]).max()
        pp = p[:N] - p[0]
        assert np.all(np.abs(pp[ok, 0] - x[ok]) <= 1e-12)
        assert np.all(np.abs(pp[ok, 1] - yy[ok]) <= 1e-12)


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("name", SYSTEMS)
def test_epilogues_match_stored_rows(eng, systems, name, mode):
    """rtx_trace_reduce, rtx_moments, rtx_focus_moments and rtx_trace_opd
    against the exact restatement applied to what rtx_trace stores for the same
    rays, over N = 0 .. 1e6 (below a warp, around warp and tile edges),
    weights absent / random positive (of the ray dtype), centre absent / the
    chief ray's; at N <= 1e5 in FP64 also the derived rms and focus shift
    against np_oracle's trace"""
    dtype, exact = MODES[mode]
    table, rot0, clip, rays = _system(name, systems)
    rng = np.random.default_rng(7)
    worst = 0.
    for k, N in enumerate(NS):
        y0, u0 = rays(max(N, 1), 100 + k)
        dy0, du0 = eng.to_device(y0, dtype), eng.to_device(u0, dtype)
        y = inc = np.zeros((0, 3), dtype)
        if N:
            Y, _, I, _ = _stored(eng, table, dy0, du0, N, dtype, exact, clip, rot0)
            y, inc = Y[0], I[0]
        w = eng.to_device(rng.uniform(.5, 2., max(N, 1)), dtype) if k % 2 else None
        center = None
        if (k//2) % 2 and N:
            c = np.r_[y[0, :2], inc[0, :2]/inc[0, 2]].astype(np.float64)
            center = c if np.all(np.isfinite(c)) else np.zeros(4)
        n0 = eng.launch_count()
        m, s, r = _check_reduce(eng, table, dy0, du0, N, dtype, exact, clip, rot0, w, center,
                                y, inc)
        worst = max(worst, r)
        if N == 0:
            assert np.array_equal(m, np.zeros(20))
            assert eng.launch_count() == n0
        elif name == "double_gauss" and N > 1000:
            assert 0 < m[4] < m[5]                         # clipped rays in the bundle
        if N in (65, 70001) and dtype == np.float64:
            Yo, _, Io, _ = np_oracle.trace(table, y0[:N], u0[:N], clip=clip, rot0=rot0)
            so, ao = epi_oracle.reduce_sums(Yo[-1], Io[-1], None if w is None else
                                            w.download()[:N], center)
            tol = 1e-12 if exact else 1e-10
            _derived(m, so, ao, w is None, center, tol, 1e-10, "vs np_oracle")
        _check_opd(eng, table, dy0, du0, y0, u0, N, dtype, exact, clip, rot0, k)
        for a in (dy0, du0, w):
            if a is not None:
                a.free()
    print("%s %s: worst |sum - exact| / bound = %.3g" % (name, mode, worst))


@pytest.mark.parametrize("mode", list(MODES))
def test_sub_ranges_and_restarts(eng, systems, mode):
    """the march to an inner surface (at < last: 3 and 5 surfaces) equals the
    full trace's stored row there; a march restarted from the stored row k-1
    of a rotated system (rot0 = that surface's rotation back to the axis
    frame) equals the full trace's last row"""
    dtype, exact = MODES[mode]
    ent = systems["double_gauss"]
    table, aim = ent["tables"][0], ent["aim"][0][3]
    N = 4099
    y0, u0 = aim_infinite(aim["field"], disc(N, 5), aim["z"], aim["p"], ent["object_angle"])
    dy0, du0 = eng.to_device(y0, dtype), eng.to_device(u0, dtype)
    Y, U, I, _ = _stored(eng, table, dy0, du0, N, dtype, exact, True, None, rows="all")
    for at in (2, 4):
        _check_reduce(eng, table[:at + 1], dy0, du0, N, dtype, exact, True, None, None, None,
                      Y[at], I[at])
        _check_opd(eng, table[:at + 1], dy0, du0, y0, u0, N, dtype, exact, True, None, at)
    c = load_golden("tilted_clip0")
    table = c["table"]
    y0, u0 = c["y0"], c["u0"]
    N = len(y0)
    dy0, du0 = eng.to_device(y0, dtype), eng.to_device(u0, dtype)
    Y, U, I, _ = _stored(eng, table, dy0, du0, N, dtype, exact, c["clip"], None, rows="all")
    assert table["flags"][1] & 1
    full = eng.trace_reduce(table, dy0, du0, N=N, clip=c["clip"], exact=exact)
    ry, ru = eng.to_device(Y[1], dtype), eng.to_device(U[1], dtype)
    rot0 = np.asarray(table["rot"][1], np.float64).reshape(9)
    m, s, _ = _check_reduce(eng, table[2:], ry, ru, N, dtype, exact, c["clip"], rot0, None, None,
                            Y[-1], I[-1])
    assert m[4] == full[4] == N and m[8] == full[8]
    _within(m, full, epi_oracle.reduce_sums(Y[-1], I[-1])[1], 2*_L_epi(eng, N), "restart")


@pytest.mark.parametrize("mode", list(MODES))
def test_degenerate_bundles(eng, systems, mode):
    """rays clipped at the first surface: nothing is finite at the last, both
    derived quantities are NaN (no exception); rays clipped only at the last
    surface keep a finite y and i there and count, as in the reference"""
    from rayopt_b200.engine import Engine
    dtype, exact = MODES[mode]
    ent = systems["double_gauss"]
    table, aim = ent["tables"][0], ent["aim"][0][0]
    N = 777
    y0, u0 = aim_infinite(aim["field"], disc(N, 9), aim["z"], aim["p"], ent["object_angle"])
    out = y0.copy()
    out[:, 0] += 100.                                      # outside the first aperture
    dy0, du0 = eng.to_device(out, dtype), eng.to_device(u0, dtype)
    Y, _, I, _ = _stored(eng, table, dy0, du0, N, dtype, exact, True, None)
    m, _, _ = _check_reduce(eng, table, dy0, du0, N, dtype, exact, True, None, None, None,
                            Y[0], I[0])
    assert m[4] == 0 and m[8] == 0 and m[5] == N
    assert np.isnan(Engine.rms_from_moments(m)) and np.isnan(Engine.focus_shift_from_moments(m))
    last = table.copy()
    last["radius2"][-1] = 1e-12                            # clips (almost) every ray there
    dy0 = eng.to_device(y0, dtype)
    Y, _, I, _ = _stored(eng, last, dy0, du0, N, dtype, exact, True, None)
    want = np_oracle.trace(last, y0, u0, clip=True)
    assert np.isfinite(want[0][-1]).all() and np.isnan(want[1][-1]).all()
    m, _, _ = _check_reduce(eng, last, dy0, du0, N, dtype, exact, True, None, None, None,
                            Y[0], I[0])
    assert m[4] == N and m[8] == N


def test_long_table_keep_last_large_bundle(eng):
    """rtx_trace of a 256-surface FP64 table, keep-LAST, above the small-bundle
    size: the default kernel for that case stages 164 KB besides the 92 KB
    table, more than a CTA can have, so the launch steps down to a smaller
    staged kernel instead of refusing the table.  Same rows as the
    small-bundle kernel gives for the first rays."""
    table, _, _, rays = _system("plates256", None)
    N = 200003
    y0, u0 = rays(N, 17)
    dy0, du0 = eng.to_device(y0), eng.to_device(u0)
    Y, _, I, _ = _stored(eng, table, dy0, du0, N, np.float64, False, False, None)
    Ys, _, Is, _ = _stored(eng, table, dy0, du0, 100000, np.float64, False, False, None)
    assert np.isfinite(Y).all()
    assert np.array_equal(Y[:, :100000], Ys) and np.array_equal(I[:, :100000], Is)


@pytest.mark.parametrize("mode", ["f64_fast", "f32"])
def test_large_ragged_bundle_accumulation(eng, systems, mode):
    """2e7 + 33 rays through rtx_trace_reduce: every sum within
    (L + 64) eps sum|term| of the exact sum of the stored rows, L about 1400
    here; two runs give the same counts and sums within that bound"""
    dtype, exact = MODES[mode]
    ent = systems["double_gauss"]
    table, aim = ent["tables"][0], ent["aim"][0][3]
    N = 20_000_033
    y0, u0 = aim_infinite(aim["field"], disc(N, 13), aim["z"], aim["p"], ent["object_angle"])
    dy0, du0 = eng.to_device(y0, dtype), eng.to_device(u0, dtype)
    del y0, u0
    ld = (N + 63)//64*64
    Y, I = eng.empty((1, ld, 3), dtype), eng.empty((1, ld, 3), dtype)
    eng.trace_device(table, dy0, du0, Y, None, I, None, N=N, ld=ld, clip=True, keep_last=True,
                     exact=exact)
    eng.sync()
    y, inc = Y.download()[0, :N], I.download()[0, :N]
    Y.free(), I.free()
    center = np.r_[y[0, :2], inc[0, :2]/inc[0, 2]].astype(np.float64)
    s, a = epi_oracle.reduce_sums(y, inc, None, center)
    L = _L_epi(eng, N)
    runs = [eng.trace_reduce(table, dy0, du0, N=N, clip=True, exact=exact, center=center)
            for _ in range(2)]
    worst = 0.
    for m in runs:
        for k in (4, 5, 8):
            assert m[k] == s[k]
        worst = max(worst, _within(m, s, a, L, "2e7"))
    assert 0 < s[4] < N
    _within(runs[0], runs[1], a, 2*L, "repeat")
    print("%s N=%d L=%d: worst |sum - exact| / bound = %.3g, max |err|/sum|term| = %.3g" % (
        mode, N, L, worst, max(abs(runs[0] - s)/np.where(a > 0, a, 1))))
