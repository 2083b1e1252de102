"""The argument refusals of the C entry points (include/rtx.h): the exact
RTX_E_* code of every bad argument, of pairs whose code depends on the order
of the checks, and -- with a real context -- that a refusal launches nothing
and allocates nothing.  A NULL context is refused without a device."""
import ctypes as C

import numpy as np
import pytest

from rayopt_b200 import _lib, build
from rayopt_b200.engine import OPD_DTYPE
from rayopt_b200.rays import GRID_GIVEN, GRID_HEXAPOLAR, infinite_record
from rayopt_b200.surface_table import SURFACE_DTYPE

BAD, UNSUP = -1, -2
N = 64                    # rays of the valid base call
S = 3
MAX_ASPH, MAX_SURFACES, MAX_BATCH = 10, 256, 8

ARGS = {
    "rtx_trace": "ctx surf S rot0 dtype N y0 u0 clip keep ld Y U I T flags",
    "rtx_trace_batch": "ctx nb surf S rot0 dtype N y0 u0 clip keep ld Y U I T flags",
    "rtx_trace_batch_host": "ctx nb surf S rot0 dtype N y0 u0 clip keep Y U I T flags",
    "rtx_trace_host": "ctx surf S rot0 dtype N y0 u0 clip keep Y U I T flags",
    "rtx_trace_gather": "ctx surf S rot0 dtype N y0 u0 clip npeers dst dst_i dst_offset flags",
    "rtx_trace_reduce": "ctx surf S rot0 dtype N y0 u0 clip w center m flags",
    "rtx_trace_opd": "ctx surf S rot0 dtype N y0 u0 clip opd A P flags",
    "rtx_moments": "ctx dtype N y w center m",
    "rtx_focus_moments": "ctx dtype N y inc w center m",
    "rtx_aim_plan": "ctx spec n_given yp n_rays",
    "rtx_aim_rays": "ctx spec n_given yp dtype first count y0 u0 yp_out",
    "rtx_grid_linear": "ctx dtype M pts vals T simplices transform n gh out winner",
    "rtx_psf": "ctx dtype n o pad psf stats",
    "rtx_grid_range": "ctx dtype n o count lo hi",
}
ARGS = {k: v.split() for k, v in ARGS.items()}


def table(n_asph=None):
    t = np.zeros(S, SURFACE_DTYPE)
    t["n_asph"] = -1
    t["mu"] = 1.
    t["c"] = 0.01
    if n_asph is not None:
        t["n_asph"][1] = n_asph
    return t


def vp(a):
    return None if a is None else C.c_void_p(a if isinstance(a, int) else a.ctypes.data)


def parr(items):
    """a void* array of the pointers of `items` (ints or numpy arrays)"""
    return C.cast((C.c_void_p*len(items))(*[vp(x) for x in items]), C.c_void_p)


class Operands:
    """The operands of a valid call of every entry point.  `dev(shape,
    dtype)` returns the address of a device buffer: a real allocation with a
    context, a never-dereferenced dummy without one."""

    def __init__(self, dev):
        self.keep = []                          # host arrays the pointers refer to
        self.tab, self.tab_asph = table(), table(MAX_ASPH + 1)
        self.tab_neg = table(-2)
        self.y0, self.u0 = dev((N, 3)), dev((N, 3))
        self.Y, self.U, self.I = (dev((S, N, 3)) for _ in range(3))
        self.T = dev((S, N))
        self.hy0, self.hu0 = np.zeros((N, 3)), np.zeros((N, 3))
        self.hu0[:, 2] = 1.
        self.hY = [np.empty((S, N, 3)) for _ in range(3)]
        self.hT = np.empty((S, N))
        self.m = np.zeros(20)
        self.opd = np.zeros(1, OPD_DTYPE)
        self.opd["radius"] = 1.
        self.opd["n0"] = self.opd["n_after"] = 1.
        self.A, self.P = dev((N,)), dev((N, 3))
        self.aim = infinite_record((0., 0.), 10., ((-1., -1.), (1., 1.)), 0.1,
                                   grid=dict(grid=GRID_HEXAPOLAR, n=2))
        self.given = infinite_record((0., 0.), 10., ((-1., -1.), (1., 1.)), 0.1,
                                     grid=dict(grid=GRID_GIVEN))
        self.aim_asph = self.aim.copy()
        self.aim_asph["curved"] = 1
        self.aim_asph["surface"]["n_asph"] = MAX_ASPH + 1
        self.aim_asph["surface"]["c"] = 0.01
        self.n_rays = C.c_int64()
        self.gh, self.grid_out = dev((4,)), dev((4, 4))
        self.psf_o, self.psf_out = dev((4, 4)), dev((8, 8))
        self.count, self.lo, self.hi = C.c_int64(), C.c_double(), C.c_double()

    def keep_arr(self, rec, **fields):
        """a copy of the record `rec` with `fields` changed"""
        r = rec.copy()
        for k, v in fields.items():
            r[k] = v
        self.keep.append(r)
        return r

    def batch(self, tabs=None, Ns=None, y0s=None, u0s=None):
        tabs = tabs or [self.tab, self.tab]
        Ns = np.asarray(Ns or [N]*len(tabs), np.int64)
        y0s = y0s or [self.y0]*len(tabs)
        u0s = u0s or [self.u0]*len(tabs)
        self.keep.append((tabs, Ns))
        return dict(nb=len(tabs), surf=parr(tabs), N=vp(Ns), y0=parr(y0s), u0=parr(u0s))

    def base(self, name):
        tr = dict(surf=vp(self.tab), S=S, rot0=None, dtype=0, N=N, clip=0)
        if name == "rtx_trace":
            return dict(tr, y0=self.y0, u0=self.u0, keep=0, ld=N, Y=self.Y, U=self.U, I=self.I,
                        T=self.T, flags=0)
        if name == "rtx_trace_batch":
            return dict(tr, **self.batch(), keep=0, ld=N, Y=parr([self.Y]*2), U=None, I=None,
                        T=None, flags=0)
        if name == "rtx_trace_batch_host":
            b = self.batch(y0s=[self.hy0]*2, u0s=[self.hu0]*2)
            return dict(tr, **b, keep=0, Y=parr([self.hY[0]]*2), U=None, I=None, T=None,
                        flags=0)
        if name == "rtx_trace_host":
            return dict(tr, y0=vp(self.hy0), u0=vp(self.hu0), keep=0, Y=vp(self.hY[0]),
                        U=vp(self.hY[1]), I=vp(self.hY[2]), T=vp(self.hT), flags=0)
        if name == "rtx_trace_gather":
            return dict(tr, y0=self.y0, u0=self.u0, npeers=1, dst=parr([self.Y]), dst_i=None,
                        dst_offset=0, flags=0)
        if name == "rtx_trace_reduce":
            return dict(tr, y0=self.y0, u0=self.u0, w=None, center=None, m=vp(self.m), flags=0)
        if name == "rtx_trace_opd":
            return dict(tr, y0=self.y0, u0=self.u0, opd=vp(self.opd), A=self.A, P=self.P,
                        flags=0)
        if name == "rtx_moments":
            return dict(dtype=0, N=N, y=self.y0, w=None, center=None, m=vp(self.m))
        if name == "rtx_focus_moments":
            return dict(dtype=0, N=N, y=self.y0, inc=self.u0, w=None, center=None, m=vp(self.m))
        if name == "rtx_aim_plan":
            return dict(spec=vp(self.aim), n_given=0, yp=None, n_rays=C.byref(self.n_rays))
        if name == "rtx_aim_rays":
            return dict(spec=vp(self.aim), n_given=0, yp=None, dtype=0, first=0, count=7,
                        y0=self.y0, u0=self.u0, yp_out=None)
        if name == "rtx_grid_linear":
            return dict(dtype=0, M=0, pts=None, vals=None, T=0, simplices=None, transform=None,
                        n=4, gh=self.gh, out=self.grid_out, winner=None)
        if name == "rtx_psf":
            return dict(dtype=0, n=4, o=self.psf_o, pad=2, psf=self.psf_out, stats=None)
        if name == "rtx_grid_range":
            return dict(dtype=0, n=16, o=self.psf_o, count=C.byref(self.count),
                        lo=C.byref(self.lo), hi=C.byref(self.hi))
        raise KeyError(name)


def call(lib, ops, ctx, name, **over):
    kw = dict(ops.base(name), ctx=ctx)
    kw.update(over)
    return getattr(lib, name)(*[kw[a] for a in ARGS[name]])


TRACES = ["rtx_trace", "rtx_trace_host", "rtx_trace_gather", "rtx_trace_reduce",
          "rtx_trace_opd"]
BATCHES = ["rtx_trace_batch", "rtx_trace_batch_host"]
FP64_ONLY = ["rtx_grid_linear", "rtx_psf", "rtx_grid_range"]


def _cases():
    """(entry point, what, overrides(ops), expected code)"""
    for name in TRACES:
        yield name, "NULL table", lambda o: dict(surf=None), BAD
        yield name, "S = 0", lambda o: dict(S=0), BAD
        yield name, "S > RTX_MAX_SURFACES", lambda o: dict(S=MAX_SURFACES + 1), BAD
        yield name, "n_asph > RTX_MAX_ASPH", lambda o: dict(surf=vp(o.tab_asph)), UNSUP
        yield name, "n_asph < -1", lambda o: dict(surf=vp(o.tab_neg)), BAD
        yield name, "N < 0", lambda o: dict(N=-1), BAD
        yield name, "NULL y0", lambda o: dict(y0=None), BAD
        yield name, "NULL u0", lambda o: dict(u0=None), BAD
        yield name, "dtype 2", lambda o: dict(dtype=2), BAD
        # the table is checked before the element type
        yield name, "n_asph > RTX_MAX_ASPH and dtype 2", \
            lambda o: dict(surf=vp(o.tab_asph), dtype=2), UNSUP
        yield name, "n_asph > RTX_MAX_ASPH and N < 0", \
            lambda o: dict(surf=vp(o.tab_asph), N=-1), UNSUP
        yield name, "NULL table and dtype 2", lambda o: dict(surf=None, dtype=2), BAD
    for name in ("rtx_trace", "rtx_trace_host"):
        yield name, "keep 2", lambda o: dict(keep=2), BAD
        yield name, "n_asph > RTX_MAX_ASPH and keep 2", \
            lambda o: dict(surf=vp(o.tab_asph), keep=2), UNSUP
    yield "rtx_trace", "ld < N", lambda o: dict(ld=N - 1), BAD
    yield "rtx_trace", "n_asph > RTX_MAX_ASPH and ld < N", \
        lambda o: dict(surf=vp(o.tab_asph), ld=N - 1), UNSUP
    for name in BATCHES:
        yield name, "nb 0", lambda o: dict(nb=0), BAD
        yield name, "NULL tables", lambda o: dict(surf=None), BAD
        yield name, "NULL N", lambda o: dict(N=None), BAD
        yield name, "NULL y0", lambda o: dict(y0=None), BAD
        yield name, "NULL u0", lambda o: dict(u0=None), BAD
        yield name, "NULL table of bundle 1", lambda o: o.batch(tabs=[o.tab, None]), BAD
        yield name, "S = 0", lambda o: dict(S=0), BAD
        yield name, "S > RTX_MAX_SURFACES", lambda o: dict(S=MAX_SURFACES + 1), BAD
        yield name, "n_asph > RTX_MAX_ASPH in bundle 1", \
            lambda o: o.batch(tabs=[o.tab, o.tab_asph]), UNSUP
        yield name, "N[1] < 0", lambda o: o.batch(Ns=[N, -1]), BAD
        yield name, "dtype 2", lambda o: dict(dtype=2), BAD
        yield name, "keep 2", lambda o: dict(keep=2), BAD
        # the batch calls check the element type and keep before the tables
        yield name, "dtype 2 and n_asph > RTX_MAX_ASPH", \
            lambda o: dict(o.batch(tabs=[o.tab, o.tab_asph]), dtype=2), BAD
        yield name, "keep 2 and n_asph > RTX_MAX_ASPH", \
            lambda o: dict(o.batch(tabs=[o.tab_asph, o.tab]), keep=2), BAD
        yield name, "n_asph > RTX_MAX_ASPH in bundle 0 and N[1] < 0", \
            lambda o: o.batch(tabs=[o.tab_asph, o.tab], Ns=[N, -1]), UNSUP
        yield name, "N[0] < 0 and n_asph > RTX_MAX_ASPH in bundle 1", \
            lambda o: o.batch(tabs=[o.tab, o.tab_asph], Ns=[-1, N]), BAD
    yield "rtx_trace_batch", "nb > RTX_MAX_BATCH", lambda o: dict(nb=MAX_BATCH + 1), BAD
    yield "rtx_trace_batch", "N[1] = 0", lambda o: o.batch(Ns=[N, 0]), BAD
    yield "rtx_trace_batch", "ld < N[1]", lambda o: dict(ld=N - 1), BAD
    yield "rtx_trace_batch", "NULL y0[1]", lambda o: o.batch(y0s=[o.y0, None]), BAD
    yield "rtx_trace_batch_host", "NULL u0[1]", lambda o: o.batch(u0s=[o.hu0, None]), BAD
    g = "rtx_trace_gather"
    yield g, "npeers 0", lambda o: dict(npeers=0), BAD
    yield g, "npeers 9", lambda o: dict(npeers=9), BAD
    yield g, "NULL dst", lambda o: dict(dst=None), BAD
    yield g, "NULL dst[0]", lambda o: dict(dst=parr([None])), BAD
    yield g, "NULL dst_i[0]", lambda o: dict(dst_i=parr([None])), BAD
    yield g, "dst_offset < 0", lambda o: dict(dst_offset=-1), BAD
    yield g, "n_asph > RTX_MAX_ASPH and npeers 0", \
        lambda o: dict(surf=vp(o.tab_asph), npeers=0), UNSUP
    # no ray: done before the destinations are looked at
    yield g, "N = 0 and NULL dst[0]", lambda o: dict(N=0, dst=parr([None])), 0
    yield "rtx_trace_reduce", "NULL m", lambda o: dict(m=None), BAD
    yield "rtx_trace_reduce", "NULL m and n_asph > RTX_MAX_ASPH", \
        lambda o: dict(m=None, surf=vp(o.tab_asph)), BAD
    yield "rtx_trace_opd", "NULL opd", lambda o: dict(opd=None), BAD
    yield "rtx_trace_opd", "NULL A", lambda o: dict(A=None), BAD
    yield "rtx_trace_opd", "NULL P", lambda o: dict(P=None), BAD
    yield "rtx_trace_opd", "radius 0", lambda o: dict(opd=vp(o.keep_arr(o.opd, radius=0.))), BAD
    yield "rtx_trace_opd", "n_asph > RTX_MAX_ASPH and radius 0", \
        lambda o: dict(surf=vp(o.tab_asph), opd=vp(o.keep_arr(o.opd, radius=0.))), UNSUP
    for name in ("rtx_moments", "rtx_focus_moments"):
        yield name, "N < 0", lambda o: dict(N=-1), BAD
        yield name, "NULL y", lambda o: dict(y=None), BAD
        yield name, "NULL m", lambda o: dict(m=None), BAD
        yield name, "dtype 2", lambda o: dict(dtype=2), BAD
        yield name, "dtype 2 and N < 0", lambda o: dict(dtype=2, N=-1), BAD
    yield "rtx_focus_moments", "NULL inc", lambda o: dict(inc=None), BAD
    for name in ("rtx_aim_plan", "rtx_aim_rays"):
        yield name, "NULL spec", lambda o: dict(spec=None), BAD
        yield name, "n_given < 0", lambda o: dict(n_given=-1), BAD
        yield name, "curved surface with n_asph > RTX_MAX_ASPH", \
            lambda o: dict(spec=vp(o.aim_asph)), UNSUP
        yield name, "GIVEN grid without pupil coordinates", \
            lambda o: dict(spec=vp(o.given), n_given=5), BAD
        yield name, "grid 9", lambda o: dict(spec=vp(o.keep_arr(o.aim, grid=9))), BAD
    yield "rtx_aim_plan", "NULL n_rays", lambda o: dict(n_rays=None), BAD
    a = "rtx_aim_rays"
    yield a, "dtype 2", lambda o: dict(dtype=2), BAD
    yield a, "NULL y0", lambda o: dict(y0=None), BAD
    yield a, "first < 0", lambda o: dict(first=-1), BAD
    yield a, "count < 0", lambda o: dict(count=-1), BAD
    yield a, "first + count > rays", lambda o: dict(first=13, count=7), BAD
    yield a, "dtype 2 and n_asph > RTX_MAX_ASPH", \
        lambda o: dict(dtype=2, spec=vp(o.aim_asph)), BAD
    yield a, "n_asph > RTX_MAX_ASPH and first + count > rays", \
        lambda o: dict(spec=vp(o.aim_asph), first=13, count=7), UNSUP
    for name in FP64_ONLY:
        yield name, "FP32", lambda o: dict(dtype=1), UNSUP
        yield name, "dtype 2", lambda o: dict(dtype=2), BAD
    gl = "rtx_grid_linear"
    yield gl, "M < 0", lambda o: dict(M=-1), BAD
    yield gl, "T < 0", lambda o: dict(T=-1), BAD
    yield gl, "n = 1", lambda o: dict(n=1), BAD
    yield gl, "n = 46341", lambda o: dict(n=46341), BAD
    yield gl, "NULL gh", lambda o: dict(gh=None), BAD
    yield gl, "M > 0 and NULL pts", lambda o: dict(M=3, vals=o.gh), BAD
    yield gl, "T > 0 and NULL simplices", lambda o: dict(T=1, transform=o.gh), BAD
    yield gl, "n = 1 and FP32", lambda o: dict(n=1, dtype=1), BAD
    yield gl, "M > 0, NULL pts and FP32", lambda o: dict(M=3, dtype=1), BAD
    yield "rtx_psf", "n = 0", lambda o: dict(n=0), BAD
    yield "rtx_psf", "pad = 0", lambda o: dict(pad=0), BAD
    yield "rtx_psf", "NULL o", lambda o: dict(o=None), BAD
    yield "rtx_psf", "n = 0 and FP32", lambda o: dict(n=0, dtype=1), BAD
    yield "rtx_grid_range", "n = 0", lambda o: dict(n=0), BAD
    yield "rtx_grid_range", "NULL lo", lambda o: dict(lo=None), BAD
    yield "rtx_grid_range", "n = 0 and FP32", lambda o: dict(n=0, dtype=1), BAD


CASES = list(_cases())


@pytest.fixture(scope="module")
def lib():
    build.build()
    return _lib.load()


@pytest.mark.parametrize("name", list(ARGS))
def test_null_context_is_refused(lib, name):
    ops = Operands(lambda shape, dtype=np.float64: 0x1000)   # never dereferenced
    assert call(lib, ops, None, name) == BAD


@pytest.fixture(scope="module")
def eng():
    from rayopt_b200.engine import Engine
    _lib.preload_cufft()              # the valid rtx_psf call
    e = Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def dev_ops(eng):
    held = []

    def dev(shape, dtype=np.float64):
        a = eng.empty(shape, dtype)
        eng.memset(a)
        held.append(a)
        return a.ptr
    ops = Operands(dev)
    eng.sync()
    yield ops
    for a in held:
        a.free()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(ARGS))
def test_valid_base_call_is_accepted(eng, dev_ops, name):
    """the operands the refusals start from are a valid call"""
    assert call(eng.lib, dev_ops, eng.ctx, name) == 0, name
    eng.sync()


@pytest.mark.gpu
@pytest.mark.parametrize("name,what,over,code", CASES,
                         ids=["%s: %s" % (c[0], c[1]) for c in CASES])
def test_refusal_code_and_no_device_work(eng, dev_ops, name, what, over, code):
    eng.sync()
    launches, free = eng.launch_count(), eng.free_bytes()
    assert call(eng.lib, dev_ops, eng.ctx, name, **over(dev_ops)) == code, (name, what)
    assert eng.launch_count() == launches, (name, what)
    assert eng.free_bytes() == free, (name, what)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["rtx_moments", "rtx_focus_moments"])
def test_moments_refuse_a_bad_dtype_without_rays(eng, dev_ops, name):
    """the element type is checked whatever N is, as rtx_spot_rows does"""
    launches, free = eng.launch_count(), eng.free_bytes()
    assert call(eng.lib, dev_ops, eng.ctx, name, N=0, dtype=7) == BAD
    assert eng.launch_count() == launches and eng.free_bytes() == free
    assert call(eng.lib, dev_ops, eng.ctx, name, N=0) == 0


@pytest.mark.gpu
def test_failed_timed_call_reports_no_kernel_time(eng, dev_ops):
    """a call that fails after its timing started (RTX_EXACT with FP32 is
    refused at the launch) leaves no span for rtx_last_kernel_ms: the
    chunk-event sum of no chunk, 0"""
    eng.trace(table(), np.zeros((2, 3)), np.tile((0., 0., 1.), (2, 1)))  # clears the chunk events
    assert call(eng.lib, dev_ops, eng.ctx, "rtx_trace") == 0
    eng.sync()
    assert eng.last_kernel_ms() > 0
    for name in ("rtx_trace", "rtx_trace_reduce"):
        assert call(eng.lib, dev_ops, eng.ctx, name, dtype=1, flags=_lib.RTX_EXACT) == UNSUP
        eng.sync()
        assert eng.last_kernel_ms() == 0, name
