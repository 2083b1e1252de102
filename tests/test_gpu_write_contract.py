"""What every trace call writes, and what it leaves alone.

include/rtx.h promises more than the values of the stored rows:
- bulk (staged) stores write whole groups of 32 x rays-per-thread rays, so
  nothing at or after column up(N, 32 rpt) of a row; per-ray stores touch only
  columns < N; keep-LAST writes one row; a NULL output is skipped;
- the warp-ballot mask (rtx_set_mask_output) is ceil(N/32) words whose bit k
  of word w is isfinite(u[last][32 w + k]), 0 for rays >= N; the path sum
  (rtx_set_path_sum_output) is N values, the left-to-right sum of the stored
  t rows 0..upto;
- rtx_trace_batch, rtx_trace_host and rtx_trace_batch_host switch both side
  outputs off and restore the registration afterwards;
- a gather writes exactly rays dst_offset .. dst_offset + N - 1 of every
  destination; the host front ends write exactly the caller's (rows, N, k);
  inputs are never modified; the epilogues and generators write exactly
  their outputs.

Every output here is a view into one allocation [guard | payload | guard]
with guards of 64 KB (more than one CTA tile of the largest kernel, 2048
FP64 rays x 24 bytes), pre-filled with a NaN whose payload no kernel makes
(0x7FF4A5A5A5A5A5A5 in FP64, 0x7FA5A5A5 in FP32 and in 32-bit words).
After each call the regions that must stay untouched are compared bytewise
with that sentinel.  The kernel configurations are those of
test_gpu_config_invariance.py; every trace case asserts, through
Engine.last_launch_config(), the configuration it ran.  Mask and path sum
are also compared with the values derived from the per-thread store
kernel's rows (`canon`), so they are bit-identical across configurations.
Needs a GPU: `pytest -m gpu`.
"""
import ctypes as C

import numpy as np
import pytest

import np_oracle
from rayopt_b200._lib import check, ptr
from rayopt_b200.engine import _code
from rayopt_b200.rays import aim_record, grid_spec
from test_gpu_config_invariance import (  # noqa: F401  (fixtures)
    CTA, DIRECT, FORCED, FP32_ONLY, FP64_ONLY, GATHERS, LAYOUTS, MIN_FORCED, MODES, PER_RAY,
    R1W8, SIZES32, SIZES64, WARP, _bad, _by_size, _chunk, _host_tiled, _tiled, _up, canon, eng,
    forced, sysdb)
from test_gpu_aim import P as AIM_P, conj, surf
from test_gpu_epilogues import _spec

pytestmark = pytest.mark.gpu

GUARD = 64 << 10
UINT = {8: np.uint64, 4: np.uint32}
SENTINEL = {8: np.uint64(0x7FF4A5A5A5A5A5A5), 4: np.uint32(0x7FA5A5A5)}
_FILL_CHUNK = 1 << 20


def _sentinel(raw, isz):
    """True where the (element-aligned) bytes `raw` hold the sentinel"""
    return raw.view(UINT[isz]) == SENTINEL[isz]


def _fill(e, p, nbytes, isz):
    """fill device bytes [p, p + nbytes) with the sentinel (one upload, then
    doubling device-to-device copies)"""
    pat = np.full(_FILL_CHUNK//isz, SENTINEL[isz], UINT[isz])
    done = min(_FILL_CHUNK, nbytes)
    check(e.lib.rtx_memcpy_h2d(e.ctx, p, pat.ctypes.data, done))
    e.sync()
    while done < nbytes:
        n = min(done, nbytes - done)
        check(e.lib.rtx_memcpy_d2d(e.ctx, p + done, p, n))
        done += n
    e.sync()


def _typed_view(base, byte_off, shape, dtype):
    from rayopt_b200.engine import DeviceArray
    v = object.__new__(DeviceArray)
    v.engine, v.dtype, v.shape = base.engine, np.dtype(dtype), tuple(int(s) for s in shape)
    v.nbytes = int(np.prod(v.shape, dtype=np.int64))*v.dtype.itemsize
    v.ptr = base.ptr + byte_off
    v.free = lambda: None
    v._parent = base
    return v


class Guarded:
    """`a`: a (shape, dtype) DeviceArray view that starts `offset` bytes after
    a 64 KB guard and is followed by one, all filled with the sentinel"""

    def __init__(self, e, shape, dtype, offset=0):
        self.e, self.dtype = e, np.dtype(dtype)
        self.isz = self.dtype.itemsize
        self.shape = tuple(int(s) for s in shape)
        self.lo = GUARD + int(offset)
        self.pbytes = int(np.prod(self.shape, dtype=np.int64))*self.isz
        self.total = self.lo + self.pbytes + GUARD
        self.base = e.empty((self.total,), np.uint8)
        self.refill()
        self.a = _typed_view(self.base, self.lo, self.shape, self.dtype)

    def refill(self):
        _fill(self.e, self.base.ptr, self.total, self.isz)

    def free(self):
        self.base.free()

    def raw(self, off, n):
        out = np.empty(n, np.uint8)
        if n:
            check(self.e.lib.rtx_memcpy_d2h(self.e.ctx, out.ctypes.data, self.base.ptr + off, n))
            self.e.sync()
        return out

    def guards_ok(self):
        return bool(_sentinel(self.raw(0, self.lo), self.isz).all()
                    and _sentinel(self.raw(self.lo + self.pbytes, GUARD), self.isz).all())

    def untouched(self):
        """guards and payload all sentinel"""
        return bool(_sentinel(self.raw(0, self.total), self.isz).all())

    def payload(self):
        return self.a.download()

    def tail_ok(self, ld, k, c0, rows_written):
        """columns c0 .. ld-1 of the rows < rows_written, and every later row
        of a (rows, ld, k) payload, still hold the sentinel"""
        rb = ld*k*self.isz
        ok = True
        w = (ld - c0)*k*self.isz
        if w and rows_written:
            out = np.empty(w*rows_written, np.uint8)
            check(self.e.lib.rtx_memcpy2d_d2h(self.e.ctx, out.ctypes.data, w,
                                              self.base.ptr + self.lo + c0*k*self.isz, rb, w,
                                              rows_written))
            self.e.sync()
            ok = bool(_sentinel(out, self.isz).all())
        rest = self.raw(self.lo + rows_written*rb, self.pbytes - rows_written*rb)
        return ok and bool(_sentinel(rest, self.isz).all())

    def row(self, r, n, k):
        """the first n rays of row r of a (rows, ld, k) payload"""
        ld = self.shape[1]
        out = np.empty((n, k) if k > 1 else (n,), self.dtype)
        check(self.e.lib.rtx_memcpy_d2h(self.e.ctx, out.ctypes.data,
                                        self.a.ptr + r*ld*k*self.isz, out.nbytes))
        self.e.sync()
        return out


def _free(items):
    for a in items:
        if a is not None:
            a.free()


def _lr_sum(rows, upto):
    """sum of rows 0..upto (all for upto < 0), left to right, in their dtype"""
    k = len(rows) if upto < 0 else min(upto + 1, len(rows))
    acc = np.zeros(rows.shape[1], rows.dtype)
    for j in range(k):
        acc = acc + rows[j]
    return acc


def _same(got, want, what):
    bad = _bad(got.reshape(len(got), -1), want.reshape(len(want), -1))
    assert not bad.any(), "%s: %d of %d rays differ, first %d" % (
        what, int(bad.sum()), len(bad), int(np.flatnonzero(bad)[0]))


def _mask_bits(words, N):
    bits = np.unpackbits(words.view(np.uint8), bitorder="little").astype(bool)
    assert not bits[N:].any(), "mask bits of rays >= N set"
    return bits[:N]


def _canon_side(canon, name, mode, N, upto=-1):
    """mask and path sum of N tiled probe rays from the per-thread store
    kernel's rows"""
    Y, U, I, T = canon(name, mode)
    k = np.arange(N) % U.shape[1]
    return np.isfinite(U[-1][:, 0])[k], _lr_sum(T, upto)[k]


def _inputs_ok(dy, du, hy, hu):
    for d, h in ((dy, hy), (du, hu)):
        assert np.array_equal(d.download().view(UINT[h.itemsize]), h.view(UINT[h.itemsize])), \
            "launch rays modified"


# ---- device traces over the whole configuration matrix ---------------------
def _store_end(cfg, N):
    """first column a launch in configuration `cfg` may not write"""
    return N if cfg[1] == DIRECT else _up(N, 32*cfg[0])


def _device_case(e, s, canon, name, mode, N, ld, want_cfg, label, keep_last=False, offset=0,
                 rpt=0, direct=False, drop=None):
    """one trace of N tiled probe rays into guarded Y, U, I, T (all S rows even
    for keep-LAST: the rows after the first are guards too), mask and path
    sum; then path-sum-only launches for every `upto` and a mask-only launch.
    `drop`: the index of the output passed as NULL.  Returns the host rows
    [:N] of the outputs."""
    dtype, exact = MODES[mode]
    isz = np.dtype(dtype).itemsize
    table = s["tables"][0]
    tab0 = table.copy()
    S = len(table)
    rows = 1 if keep_last else S
    dy, du = _tiled(e, s, dtype, N)
    hy, hu = (np.ascontiguousarray(a, dtype) for a in _host_tiled(s, N))
    ks = (3, 3, 3, 1)
    outs = [None if j == drop else Guarded(e, (S, ld, k) if k == 3 else (S, ld), dtype,
                                            offset*isz) for j, k in enumerate(ks)]
    mask = Guarded(e, ((N + 31)//32,), np.uint32)
    ps = Guarded(e, (N,), dtype)
    kw = dict(N=N, ld=ld, clip=s["clip"], rot0=s["rot0"], exact=exact, keep_last=keep_last,
              rpt=rpt, direct=direct)
    try:
        e.trace_device(table, dy, du, *[None if g is None else g.a for g in outs], mask=mask.a,
                       path_sum=ps.a, **kw)
        e.sync()
        cfg = e.last_launch_config()
        assert cfg == want_cfg, (label, cfg)
        c0 = _store_end(cfg, N)
        got = []
        for g, k, nm in zip(outs, ks, "YUIT"):
            if g is None:
                got.append(None)
                continue
            assert g.guards_ok(), "%s: write outside %s" % (label, nm)
            assert g.tail_ok(ld, k, c0, rows), "%s: %s written at or after column %d or row %d" % (
                label, nm, c0, rows)
            got.append([g.row(r, N, k) for r in range(rows)])
        _inputs_ok(dy, du, hy, hu)
        assert table.tobytes() == tab0.tobytes()
        want_mask, want_sum = _canon_side(canon, name, mode, N)
        # mask: the launch's own last row, and the per-thread kernel's
        assert mask.guards_ok(), "%s: mask written past ceil(N/32) words" % label
        bits = _mask_bits(mask.payload(), N)
        if got[1] is not None:
            assert np.array_equal(bits, np.isfinite(got[1][-1][:, 0])), "%s: mask" % label
        assert np.array_equal(bits, want_mask), "%s: mask differs from the per-thread kernel's" % label
        # path sum: the launch's own T rows (keep-ALL), and the per-thread kernel's
        assert ps.guards_ok(), "%s: path sum written past N" % label
        if got[3] is not None and not keep_last:
            _same(ps.payload(), _lr_sum(np.array(got[3]), -1), "%s: path sum vs its own T" % label)
        _same(ps.payload(), want_sum, "%s: path sum vs the per-thread kernel's T" % label)
        if mode == "exact" and s["bit"]:
            _same(ps.payload(), _oracle_sum(s, N), "%s: path sum vs the oracle" % label)
        # side outputs alone (nothing else stored), every `upto`; without
        # outputs nothing is misaligned, so an offset layout's per-ray
        # kernel is requested explicitly
        side = dict(kw, direct=direct or offset != 0)
        for upto in (0, S//2, S - 1, S + 2):
            ps.refill()
            e.trace_device(table, dy, du, None, None, None, None, path_sum=ps.a,
                           path_sum_upto=upto, **side)
            e.sync()
            assert e.last_launch_config() == want_cfg, (label, "path sum only")
            assert ps.guards_ok(), "%s: path sum only (upto %d) past N" % (label, upto)
            _same(ps.payload(), _canon_side(canon, name, mode, N, upto)[1],
                  "%s: path sum only, upto %d" % (label, upto))
            if got[3] is not None and not keep_last:
                _same(ps.payload(), _lr_sum(np.array(got[3]), upto),
                      "%s: path sum only vs its own T, upto %d" % (label, upto))
        mask.refill()
        e.trace_device(table, dy, du, None, None, None, None, mask=mask.a, **side)
        e.sync()
        assert e.last_launch_config() == want_cfg, (label, "mask only")
        assert mask.guards_ok()
        assert np.array_equal(_mask_bits(mask.payload(), N), want_mask), "%s: mask only" % label
        _inputs_ok(dy, du, hy, hu)
        return got
    finally:
        check(e.lib.rtx_set_mask_output(e.ctx, None))
        check(e.lib.rtx_set_path_sum_output(e.ctx, None, -1))
        _free(outs + [mask, ps, dy, du])


_oracle_cache = {}


def _oracle_sum(s, N):
    key = id(s)
    if key not in _oracle_cache:
        T = np_oracle.trace(s["tables"][0], s["y0"], s["u0"], clip=s["clip"], rot0=s["rot0"])[3]
        _oracle_cache[key] = _lr_sum(T, -1)
    return _oracle_cache[key][np.arange(N) % len(s["y0"])]


MATRIX_SYSTEMS = ["cooke_asph", "double_gauss"]      # one Newton, one analytic


def _forced_cases():
    for mode in MODES:
        for cfg in FORCED:
            if cfg in (FP64_ONLY if mode == "fp32" else FP32_ONLY):
                continue
            for name in MATRIX_SYSTEMS:
                yield pytest.param(name, mode, cfg, id="%s-%s-%s" % (name, mode, cfg))


@pytest.mark.parametrize("name,mode,cfg", list(_forced_cases()))
def test_forced_configuration(sysdb, canon, forced, name, mode, cfg):
    s = sysdb(name)
    # a ragged bundle (N % 32 = 9: a last mask word and a last ray group with
    # dead lanes) and a pitch with spare columns whose tail must stay untouched
    N = max(len(s["y0"]), MIN_FORCED) + 1001
    _device_case(forced(cfg), s, canon, name, mode, N, _up(N, 128) + 128, FORCED[cfg][0],
                 "%s %s %s" % (name, mode, cfg))


def _size_cases():
    for mode in MODES:
        for N in (SIZES32 if mode == "fp32" else SIZES64):
            for name in MATRIX_SYSTEMS:
                yield pytest.param(name, mode, N, id="%s-%s-N%d" % (name, mode, N))


@pytest.mark.parametrize("name,mode,N", list(_size_cases()))
def test_default_choice_by_size(eng, sysdb, canon, name, mode, N):
    s = sysdb(name)
    _device_case(eng, s, canon, name, mode, N, _up(N, 128) + 128,
                 _by_size(MODES[mode][0], s["newton"], N), "%s %s N=%d" % (name, mode, N))


@pytest.mark.parametrize("case", LAYOUTS)
def test_layout(eng, sysdb, canon, case):
    name, mode, N, ld, off, keep_last, rpt, want_cfg = LAYOUTS[case]
    _device_case(eng, sysdb(name), canon, name, mode, N, ld, want_cfg, case, keep_last=keep_last,
                 offset=off, rpt=rpt)


# (engine: None = the default one, else a FORCED name; mode; direct)
NULL_CASES = {
    "per_ray-fast": (None, "fast", True, PER_RAY),
    "per_ray-exact": (None, "exact", True, PER_RAY),
    "r1w8-fp32": ("r1w8", "fp32", False, R1W8),
    "r2w16-fast": ("r2w16", "fast", False, (2, WARP, 16, 2, 1)),
    "r2c16-exact": ("r2c16", "exact", False, (2, CTA, 16, 1, 1)),
    "r4c16-fp32": ("r4c16", "fp32", False, (4, CTA, 16, 1, 1)),
    "r4w16-fp32": ("r4w16", "fp32", False, (4, WARP, 16, 1, 1)),
    "cluster16-fast": ("cluster16", "fast", False, (2, CTA, 16, 1, 16)),
}


@pytest.mark.parametrize("case", NULL_CASES)
def test_null_outputs(eng, forced, sysdb, canon, case):
    """each of Y, U, I, T passed as NULL in turn: the other three are the
    rows of the launch that stores all four, and nothing else is written"""
    cfg_name, mode, direct, want_cfg = NULL_CASES[case]
    e = eng if cfg_name is None else forced(cfg_name)
    s = sysdb("cooke_asph")
    N = len(s["y0"]) + 1001
    ld = _up(N, 128) + 128
    full = _device_case(e, s, canon, "cooke_asph", mode, N, ld, want_cfg, case, direct=direct)
    for drop in range(4):
        got = _device_case(e, s, canon, "cooke_asph", mode, N, ld, want_cfg,
                           "%s without %s" % (case, "YUIT"[drop]), direct=direct, drop=drop)
        for j in range(4):
            if j != drop:
                for r in range(len(full[j])):
                    assert np.array_equal(got[j][r].view(UINT[got[j][r].itemsize]),
                                          full[j][r].view(UINT[full[j][r].itemsize])), (
                        case, "YUIT"[drop], "YUIT"[j], r)


# ---- the registration across the calls that switch it off ------------------
def _raw_trace(e, table, dy, du, N, ld, T, s, dtype, exact):
    """rtx_trace as a C caller issues it: the registered side outputs stay as
    they are"""
    table = np.ascontiguousarray(table)
    r0 = None if s["rot0"] is None else np.ascontiguousarray(s["rot0"], np.float64).reshape(9)
    check(e.lib.rtx_trace(e.ctx, ptr(table), len(table), ptr(r0), _code(dtype), N, dy.ptr, du.ptr,
                          int(s["clip"]), 0, ld, None, None, None, T.ptr, 1 if exact else 0))


@pytest.mark.parametrize("mode", ["fast", "fp32"])
def test_registration_survives_other_calls(eng, sysdb, canon, mode):
    """guarded mask and path-sum buffers registered, then every call that must
    not use them: they stay at the sentinel, and the next rtx_trace fills them"""
    name = "cooke_asph"
    s = sysdb(name)
    dtype, exact = MODES[mode]
    table = s["tables"][0]
    S = len(table)
    Cn = _chunk(S, dtype)
    cap = 2*Cn + 100_017             # room for the largest call below: no write can escape
    mask = Guarded(eng, ((cap + 31)//32,), np.uint32)
    ps = Guarded(eng, (cap,), dtype)
    kw = dict(clip=s["clip"], rot0=s["rot0"], exact=exact)
    held = []
    try:
        check(eng.lib.rtx_set_mask_output(eng.ctx, mask.a.ptr))
        check(eng.lib.rtx_set_path_sum_output(eng.ctx, ps.a.ptr, -1))

        def untouched(what):
            eng.sync()
            assert mask.untouched(), "%s wrote the registered mask" % what
            assert ps.untouched(), "%s wrote the registered path sum" % what

        Ns = [20_000, 15_000, 77]
        ld = _up(max(Ns), 128)
        ins = [_tiled(eng, s, dtype, n) for n in Ns]
        outs = [[eng.empty((S, ld, 3), dtype) for _ in range(3)] + [eng.empty((S, ld), dtype)]
                for _ in Ns]
        held += [a for x in ins + outs for a in x]
        eng.trace_device_batch([table]*3, [a[0] for a in ins], [a[1] for a in ins],
                               *[[o[k] for o in outs] for k in range(4)], Ns=Ns, ld=ld, **kw)
        untouched("rtx_trace_batch")
        for n in (7, 1000):
            eng.trace(table, s["y0"][:n], s["u0"][:n], dtype=dtype, **kw)
            untouched("rtx_trace_host n=%d" % n)
        y, u = _host_tiled(s, cap)
        eng.trace(table, y, u, dtype=dtype, keep_last=True, **kw)
        untouched("rtx_trace_host, three chunks")
        del y, u
        for Nb in ([200 + 97*b for b in range(11)], [100_000, 77_777, 100_001]):
            rays = [_host_tiled(s, n) for n in Nb]
            eng.trace_bundles([table]*len(Nb), [r[0] for r in rays], [r[1] for r in rays],
                              dtype=dtype, **kw)
            untouched("rtx_trace_batch_host, %d bundles" % len(Nb))
        N = 50_001
        dy, du = _tiled(eng, s, dtype, N)
        held += [dy, du]
        eng.trace_reduce(table, dy, du, N=N, **kw)
        untouched("rtx_trace_reduce")
        A, Pp = eng.empty((N,), dtype), eng.empty((N, 3), dtype)
        held += [A, Pp]
        spec = _spec(s["y0"], s["u0"], np.zeros((1, 3)), 1.0, float(table["n"][-1]) or 1.0, True,
                     0.)
        eng.trace_opd(table, dy, du, spec, A, Pp, N=N, **kw)
        untouched("rtx_trace_opd")
        # the registration is back: the next rtx_trace writes both, N values
        T = eng.empty((S, _up(N, 128)), dtype)
        held.append(T)
        _raw_trace(eng, table, dy, du, N, _up(N, 128), T, s, dtype, exact)
        eng.sync()
        want_mask, want_sum = _canon_side(canon, name, mode, N)
        words = (N + 31)//32
        assert np.array_equal(_mask_bits(mask.payload()[:words], N), want_mask)
        assert _sentinel(mask.payload()[words:], 4).all() and mask.guards_ok()
        p = ps.payload()
        _same(p[:N], want_sum, "path sum after the other calls")
        _same(p[:N], _lr_sum(T.download()[:, :N], -1), "path sum vs its own T")
        assert _sentinel(p[N:], np.dtype(dtype).itemsize).all() and ps.guards_ok()
    finally:
        check(eng.lib.rtx_set_mask_output(eng.ctx, None))
        check(eng.lib.rtx_set_path_sum_output(eng.ctx, None, -1))
        _free(held + [mask, ps])


def test_gather_does_not_write_earlier_registration(eng, sysdb):
    """Engine.trace_gather without side outputs leaves the buffers an earlier
    trace_device registered alone"""
    s = sysdb("double_gauss")
    N = 20_000
    dy, du = _tiled(eng, s, np.float64, N)
    mask = Guarded(eng, ((N + 31)//32,), np.uint32)
    ps = Guarded(eng, (N,), np.float64)
    dst = eng.empty((N, 3))
    try:
        eng.trace_device(s["tables"][0], dy, du, None, None, None, None, N=N, clip=True,
                         mask=mask.a, path_sum=ps.a)
        eng.sync()
        mask.refill()
        ps.refill()
        eng.trace_gather(s["tables"][0], dy, du, [dst.ptr], 0, N=N, clip=True)
        eng.sync()
        assert mask.untouched() and ps.untouched()
    finally:
        _free([dy, du, mask, ps, dst])


# ---- host front ends ----------------------------------------------------------
class HostGuarded:
    """a (shape, dtype) numpy view between two 64 KB guards of one pageable or
    page-locked array filled with the sentinel"""

    def __init__(self, shape, dtype, e=None):
        dtype = np.dtype(dtype)
        self.isz = dtype.itemsize
        self.g, self.n = GUARD//self.isz, int(np.prod(shape, dtype=np.int64))
        n = self.n + 2*self.g
        self.buf = e.pinned_empty((n,), dtype) if e is not None else np.empty(n, dtype)
        self.buf.view(UINT[self.isz])[:] = SENTINEL[self.isz]
        self.a = self.buf[self.g:self.g + self.n].reshape(shape)

    def guards_ok(self):
        u = self.buf.view(UINT[self.isz])
        return bool((u[:self.g] == SENTINEL[self.isz]).all()
                    and (u[self.g + self.n:] == SENTINEL[self.isz]).all())


def _host_outputs(rows, N, dtype, e=None):
    return [HostGuarded((rows, N, 3), dtype, e) for _ in range(3)] + \
        [HostGuarded((rows, N), dtype, e)]


def _check_host(outs, want, keep_last, label):
    S = want[0].shape[0]
    P = want[0].shape[1]
    for g, w, nm in zip(outs, want, "yuit"):
        assert g.guards_ok(), "%s: write outside the caller's %s" % (label, nm)
        for r in range(g.a.shape[0]):
            ref = w[S - 1 if keep_last else r]
            N = g.a.shape[1]
            _same(g.a[r], ref[np.arange(N) % P], "%s %s[%d]" % (label, nm, r))


@pytest.mark.parametrize("mode", MODES)
def test_host_front_end(eng, sysdb, canon, mode):
    """rtx_trace_host (zero-copy, DMA, three chunks, keep-LAST) into guarded
    pageable and page-locked views; the caller's rays and table unchanged"""
    name = "cooke_asph"
    s = sysdb(name)
    dtype, exact = MODES[mode]
    table = s["tables"][0]
    tab0 = table.copy()
    S = len(table)
    want = canon(name, mode)
    kw = dict(clip=s["clip"], rot0=s["rot0"], dtype=dtype, exact=exact)
    Cn = _chunk(S, dtype)
    for N, keep_last, pinned in ((7, False, False), (7, False, True), (1000, False, False),
                                 (1000, True, True), (2*Cn + 100_017, False, False),
                                 (2*Cn + 100_017, True, True)):
        label = "%s host N=%d keep_last=%s pinned=%s" % (mode, N, keep_last, pinned)
        y, u = (np.ascontiguousarray(a, dtype) for a in _host_tiled(s, N))
        y1, u1 = y.copy(), u.copy()
        outs = _host_outputs(1 if keep_last else S, N, dtype, eng if pinned else None)
        eng.trace(table, y, u, keep_last=keep_last,
                  out=dict(zip("yuit", [g.a for g in outs])), **kw)
        assert np.array_equal(y.view(UINT[y.itemsize]), y1.view(UINT[y.itemsize]))
        assert np.array_equal(u.view(UINT[u.itemsize]), u1.view(UINT[u.itemsize]))
        assert table.tobytes() == tab0.tobytes()
        _check_host(outs, want, keep_last, label)
        del outs


def _batch_host(e, tables, ys, us, outs, keep_last, s, dtype, exact):
    """rtx_trace_batch_host into the caller's arrays"""
    nb = len(tables)
    vp = C.c_void_p
    tabs = [np.ascontiguousarray(t) for t in tables]

    def arr(items):
        return C.cast((vp*nb)(*[vp(a.ctypes.data) for a in items]), vp)
    keep = [arr(tabs), arr(ys), arr(us)] + [arr([o[k] for o in outs]) for k in range(4)]
    r0 = None if s["rot0"] is None else np.ascontiguousarray(s["rot0"], np.float64).reshape(9)
    check(e.lib.rtx_trace_batch_host(
        e.ctx, nb, keep[0], len(tabs[0]), ptr(r0), _code(dtype),
        C.cast((C.c_int64*nb)(*[len(y) for y in ys]), vp), keep[1], keep[2], int(s["clip"]),
        1 if keep_last else 0, keep[3], keep[4], keep[5], keep[6], 1 if exact else 0))


@pytest.mark.parametrize("mode", MODES)
def test_batch_host_front_end(eng, sysdb, canon, mode):
    """rtx_trace_batch_host: 11 small bundles (one staging buffer) and three
    bundles beyond its 64 MB (one host trace each), into guarded views"""
    name = "cooke_asph"
    s = sysdb(name)
    dtype, exact = MODES[mode]
    table = s["tables"][0]
    S = len(table)
    want = canon(name, mode)
    for Ns in ([200 + 97*b for b in range(11)], [100_000, 77_777, 100_001]):
        for keep_last in (False, True):
            rays = [[np.ascontiguousarray(a, dtype) for a in _host_tiled(s, n)] for n in Ns]
            copies = [[a.copy() for a in r] for r in rays]
            gouts = [_host_outputs(1 if keep_last else S, n, dtype,
                                   eng if (b % 2 and keep_last) else None)
                     for b, n in enumerate(Ns)]
            _batch_host(eng, [table]*len(Ns), [r[0] for r in rays], [r[1] for r in rays],
                        [[g.a for g in o] for o in gouts], keep_last, s, dtype, exact)
            for b, o in enumerate(gouts):
                for a, c in zip(rays[b], copies[b]):
                    assert np.array_equal(a.view(UINT[a.itemsize]), c.view(UINT[c.itemsize]))
                _check_host(o, want, keep_last, "%s %d bundles, bundle %d keep_last=%s" % (
                    mode, len(Ns), b, keep_last))


# ---- gathers --------------------------------------------------------------------
# (name, mode, N, destination offset, expected, {flavour: expected})
GATHER_CASES = {k: v + ({},) for k, v in GATHERS.items()}
GATHER_CASES.update({
    # 5 rays: the (x, y, z) and incidence runs are not 16-byte aligned (per-ray
    # stores); the (x, y) pairs of FP64 are
    "unaligned5": ("cooke_asph", "fast", 200_000, 5, PER_RAY, {"xy": (2, WARP, 16, 2, 1)}),
    # a multiple of 64 rays but not of 128: the four-ray FP32 kernel steps down
    "fp32_n64": ("double_gauss", "fp32", 300_096, 64, (2, CTA, 32, 1, 1), {}),
})
FLAVOURS = {"y_i": (False, True), "xy": (True, False), "xy_i": (True, True)}


@pytest.mark.parametrize("case", GATHER_CASES)
def test_gather(eng, sysdb, canon, case):
    """rtx_trace_gather into two guarded destinations (and two for i[-1]):
    everything outside rays [off, off + N) stays at the sentinel; the (x, y, z)
    + incidence flavour also writes the mask and the path sum"""
    name, mode, N, off, base_cfg, special = GATHER_CASES[case]
    s = sysdb(name)
    dtype, exact = MODES[mode]
    want = canon(name, mode)
    k = np.arange(N) % want[0].shape[1]
    dy, du = _tiled(eng, s, dtype, N)
    hy, hu = (np.ascontiguousarray(a, dtype) for a in _host_tiled(s, N))
    ntot = off + N + 128
    try:
        for flav, (xy, with_i) in FLAVOURS.items():
            kk = 2 if xy else 3
            dst = [Guarded(eng, (ntot, kk), dtype) for _ in range(2)]
            dst_i = [Guarded(eng, (ntot, 3), dtype) for _ in range(2)] if with_i else []
            side = flav == "y_i"
            mask = Guarded(eng, ((N + 31)//32,), np.uint32) if side else None
            ps = Guarded(eng, (N,), dtype) if side else None
            try:
                eng.trace_gather(s["tables"][0], dy, du, [g.a.ptr for g in dst], off, N=N,
                                 clip=s["clip"], rot0=s["rot0"], exact=exact,
                                 dst_i_ptrs=[g.a.ptr for g in dst_i] if with_i else None, xy=xy,
                                 mask=mask.a if side else None, path_sum=ps.a if side else None)
                eng.sync()
                label = "%s %s" % (case, flav)
                assert eng.last_launch_config() == special.get(flav, base_cfg), label
                for group, ref in ((dst, want[0][-1][:, :kk]), (dst_i, want[2][-1])):
                    for g in group:
                        assert g.guards_ok(), "%s: write outside the destination" % label
                        h = g.payload()
                        u = h.view(UINT[h.itemsize])
                        assert (u[:off] == SENTINEL[h.itemsize]).all(), "%s: before the shard" % label
                        assert (u[off + N:] == SENTINEL[h.itemsize]).all(), "%s: after the shard" % label
                        _same(h[off:off + N], ref[k], label)
                if side:
                    want_mask, want_sum = _canon_side(canon, name, mode, N)
                    assert mask.guards_ok() and ps.guards_ok(), label
                    assert np.array_equal(_mask_bits(mask.payload(), N), want_mask), label
                    _same(ps.payload(), want_sum, label + " path sum")
            finally:
                _free(dst + dst_i + [mask, ps])
        _inputs_ok(dy, du, hy, hu)
    finally:
        _free([dy, du])


# ---- epilogues and generators --------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("N", [70_001, 1_001])
def test_trace_opd_writes_n_rays(eng, sysdb, N, mode):
    """rtx_trace_opd writes A and P of exactly N rays"""
    s = sysdb("cooke_asph")
    dtype, exact = MODES[mode]
    table = s["tables"][0]
    dy, du = _tiled(eng, s, dtype, N)
    hy, hu = (np.ascontiguousarray(a, dtype) for a in _host_tiled(s, N))
    A, Pp = Guarded(eng, (N,), dtype), Guarded(eng, (N, 3), dtype)
    try:
        spec = _spec(s["y0"], s["u0"], np.zeros((1, 3)), 1.0, float(table["n"][-1]) or 1.0,
                     N % 2 == 1, .02)
        eng.trace_opd(table, dy, du, spec, A.a, Pp.a, N=N, clip=s["clip"], rot0=s["rot0"],
                      exact=exact)
        eng.sync()
        for g in (A, Pp):
            assert g.guards_ok()
            assert not _sentinel(g.payload(), g.isz).any(), "a ray left unwritten"
        _inputs_ok(dy, du, hy, hu)
    finally:
        _free([dy, du, A, Pp])


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_aim_rays_sub_ranges(eng, dtype):
    """rtx_aim_rays writes rays first .. first + count - 1 into y0, u0 and the
    pupil output, and nothing else"""
    rec = aim_record(conj(angle=.35, projection="stereographic"), (-.4, .9), 25., AIM_P,
                     grid_spec("hexapolar", 4000)[1], True, surf())
    spec = np.ascontiguousarray(rec)
    y, u, p = eng.aim_rays(rec, dtype, want_pupil=True)
    eng.sync()
    full = [a.download() for a in (y, u, p)]
    _free([y, u, p])
    total = len(full[0])
    for first, count in ((0, total), (17, 1000), (total - 33, 33), (5, 1)):
        outs = [Guarded(eng, (count, 3), dtype), Guarded(eng, (count, 3), dtype),
                Guarded(eng, (count, 2), np.float64)]
        try:
            check(eng.lib.rtx_aim_rays(eng.ctx, ptr(spec), 0, None, _code(dtype), first, count,
                                       outs[0].a.ptr, outs[1].a.ptr, outs[2].a.ptr))
            eng.sync()
            for g, f, nm in zip(outs, full, ("y0", "u0", "pupil")):
                assert g.guards_ok(), (first, count, nm)
                _same(g.payload(), f[first:first + count], "%s [%d, +%d)" % (nm, first, count))
        finally:
            _free(outs)


def test_grid_linear_writes_grid(eng):
    """rtx_grid_linear writes exactly its (n, n) values and winners"""
    from scipy.spatial import Delaunay
    rng = np.random.default_rng(11)
    m, n = 3000, 97
    r, phi = np.sqrt(rng.random(m)), 2*np.pi*rng.random(m)
    pts = np.stack([r*np.cos(phi), r*np.sin(phi)], -1)
    vals = np.cos(3*pts[:, 0])*pts[:, 1]
    tri = Delaunay(pts)
    gh = np.linspace(-1.05, 1.05, n)
    want, wwin = eng.grid_linear(pts, vals, tri, n, gh, winner=True)
    wwin[wwin < 0] = np.iinfo(np.int32).max
    ins = [eng.to_device(a) for a in (pts, vals, np.ascontiguousarray(tri.simplices, np.int32),
                                      tri.transform, gh)]
    out, win = Guarded(eng, (n, n), np.float64), Guarded(eng, (n, n), np.int32)
    try:
        check(eng.lib.rtx_grid_linear(eng.ctx, 0, m, ins[0].ptr, ins[1].ptr, len(tri.simplices),
                                      ins[2].ptr, ins[3].ptr, n, ins[4].ptr, out.a.ptr, win.a.ptr))
        eng.sync()
        assert out.guards_ok() and win.guards_ok()
        assert np.array_equal(out.payload(), want, equal_nan=True)
        assert np.array_equal(win.payload(), wwin)
    finally:
        _free(ins + [out, win])


def test_psf_writes_padded_grid(eng):
    """rtx_psf writes exactly its (pad n)^2 output"""
    n, pad = 126, 3
    xs = np.linspace(-1, 1, n)[:, None]*np.ones(n)
    ys = xs.T
    o = 0.3*(xs*xs + ys*ys) + 0.1*xs*ys
    o[xs*xs + ys*ys > 1] = np.nan
    od = eng.to_device(o)
    want, _ = eng.psf(od, pad)
    out = Guarded(eng, (n*pad, n*pad), np.float64)
    try:
        check(eng.lib.rtx_psf(eng.ctx, 0, n, od.ptr, pad, out.a.ptr, None))
        eng.sync()
        assert out.guards_ok()
        assert np.array_equal(out.payload(), want.download())
    finally:
        _free([od, want, out])
