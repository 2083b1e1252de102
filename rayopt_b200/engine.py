"""Host-side handle of one GPU context of the ray-trace engine.

Thin, torch-free layer over the C ABI (include/rtx.h): device / pinned memory,
the trace call with host or device buffers, CUDA-event timing.  One `Engine`
per GPU (one process per GPU in multi-GPU runs).
"""
import ctypes as C
import weakref

import numpy as np

from . import _lib
from ._lib import (RTX_F32, RTX_F64, RTX_KEEP_ALL, RTX_KEEP_LAST, RTX_EXACT,
                   RTX_STORE_DIRECT, RTX_RPT1, RTX_RPT2, RtxError, check, ptr)
from .surface_table import SURFACE_DTYPE

_DTYPES = {np.dtype(np.float64): RTX_F64, np.dtype(np.float32): RTX_F32}

# mirrors `struct rtx_opd` (include/rtx.h)
OPD_DTYPE = np.dtype([("y0_ref", "<f8", (3,)), ("u0_ref", "<f8", (3,)), ("n0", "<f8"),
                      ("n_after", "<f8"), ("M", "<f8", (9,)), ("d", "<f8", (3,)),
                      ("radius", "<f8"), ("infinite", "<i4"), ("reserved", "<i4")], align=True)


def _code(dtype):
    try:
        return _DTYPES[np.dtype(dtype)]
    except KeyError:
        raise TypeError("dtype must be float64 or float32, got %r" % (dtype,))


def _check_operands(dtype, N, **arrays):
    """The reductions and epilogues take their element type from the rays and
    read N rays from every other array: each (DeviceArray, values per ray)
    in `arrays` (None entries are skipped) must have that dtype and room for N
    rays.  Raises ValueError before anything is launched."""
    dtype = np.dtype(dtype)
    if N < 0:
        raise ValueError("N must be >= 0, got %d" % N)
    for name, (a, per_ray) in arrays.items():
        if a is None:
            continue
        if np.dtype(a.dtype) != dtype:
            raise ValueError("%s is %s but the rays are %s" % (name, np.dtype(a.dtype), dtype))
        room = a.nbytes//(dtype.itemsize*per_ray)
        if N > room:
            raise ValueError("N = %d rays but %s holds only %d" % (N, name, room))


def _check_trace_operands(dtype, N, rows, ld, outputs, mask=None, path_sum=None):
    """A trace writes rows x ld rays into each of Y, U, I (3 values per ray)
    and T (1), N values of the rays' dtype into `path_sum` and ceil(N/32)
    32-bit words into `mask`: refuse (ValueError, before anything is
    launched) an operand of another element type or one too small for that."""
    dtype = np.dtype(dtype)
    _check_operands(dtype, N, path_sum=(path_sum, 1))
    for name, (a, per_ray) in outputs.items():
        if a is None:
            continue
        if np.dtype(a.dtype) != dtype:
            raise ValueError("%s is %s but the rays are %s" % (name, np.dtype(a.dtype), dtype))
        room = a.nbytes//(dtype.itemsize*per_ray)
        if room < rows*ld:
            raise ValueError("%s holds %d rays but %d rows of pitch %d need %d"
                             % (name, room, rows, ld, rows*ld))
    if mask is not None:
        words = (N + 31)//32
        if np.dtype(mask.dtype).itemsize != 4:
            raise ValueError("mask must be 32-bit words, got %s" % np.dtype(mask.dtype))
        if mask.nbytes//4 < words:
            raise ValueError("N = %d rays need %d mask words but mask holds only %d"
                             % (N, words, mask.nbytes//4))


def _given(yp):
    """(n_given, pointer) of the DEVICE pupil coordinates of a GRID_GIVEN
    bundle, which the generator reads as (n, 2) FP64 whatever the rays' type"""
    if yp is None:
        return 0, None
    if np.dtype(yp.dtype) != np.float64:
        raise ValueError("given pupil coordinates must be float64, got %s" % np.dtype(yp.dtype))
    return yp.shape[0], yp.ptr


class DeviceArray:
    """A typed block of HBM owned by an Engine (freed with it or on .free())."""

    def __init__(self, engine, shape, dtype):
        self.engine = engine
        self.shape = tuple(int(s) for s in shape)
        self.dtype = np.dtype(dtype)
        self.nbytes = int(np.prod(self.shape, dtype=np.int64))*self.dtype.itemsize
        p = C.c_void_p()
        check(engine.lib.rtx_malloc(engine.ctx, self.nbytes, C.byref(p)))
        self.ptr = p.value
        engine._live[id(self)] = self.ptr

    def free(self):
        eng = self.engine
        if self.ptr is not None and eng.ctx is not None and id(self) in eng._live:
            eng._live.pop(id(self), None)
            check(eng.lib.rtx_free_device(eng.ctx, self.ptr))
        self.ptr = None

    def __del__(self):              # dropped without free(): give the HBM back
        try:
            if self.ptr is not None and id(self) in self.engine._live:
                self.free()
        except Exception:
            pass

    def upload(self, a):
        a = np.ascontiguousarray(a, self.dtype)
        assert a.nbytes <= self.nbytes
        check(self.engine.lib.rtx_memcpy_h2d(self.engine.ctx, self.ptr, ptr(a), a.nbytes))
        self.engine.sync()          # `a` may be a temporary
        return self

    def download(self, out=None):
        if out is None:
            out = np.empty(self.shape, self.dtype)
        check(self.engine.lib.rtx_memcpy_d2h(self.engine.ctx, ptr(out), self.ptr, out.nbytes))
        self.engine.sync()
        return out

    def copy_from(self, other, nbytes=None):
        """device-to-device copy (asynchronous on the engine stream)"""
        n = min(self.nbytes, other.nbytes) if nbytes is None else int(nbytes)
        check(self.engine.lib.rtx_memcpy_d2d(self.engine.ctx, self.ptr, other.ptr, n))
        return self

    def rows(self, r0, r1=None):
        """byte-offset view of leading-axis rows (no copy)"""
        v = object.__new__(DeviceArray)
        r1 = r0 + 1 if r1 is None else r1
        row_bytes = self.nbytes//self.shape[0]
        v.engine, v.dtype = self.engine, self.dtype
        v.shape = (r1 - r0,) + self.shape[1:]
        v.nbytes = row_bytes*(r1 - r0)
        v.ptr = self.ptr + r0*row_bytes
        v.free = lambda: None
        v._parent = self            # keeps the allocation alive
        return v


class DeviceTriangulation:
    """A Delaunay triangulation in HBM (Engine.delaunay): T triangles in
    scipy.spatial.Delaunay's layout -- simplices (T,3) int32 counter-clockwise,
    neighbors (T,3) int32 (-1 on the hull), transform (T,3,2) FP64 -- as
    DeviceArrays with room for 2M triangles."""

    def __init__(self, T, simplices, neighbors, transform):
        self.T = T
        self.simplices, self.neighbors, self.transform = simplices, neighbors, transform

    def free(self):
        for a in (self.simplices, self.neighbors, self.transform):
            a.free()

    def download(self):
        """(simplices, neighbors, transform) as numpy arrays of T rows"""
        return tuple(a.download(np.empty((self.T,) + a.shape[1:], a.dtype))
                     for a in (self.simplices, self.neighbors, self.transform))


class _PinnedBlock:
    """owner of one page-locked allocation: the numpy arrays handed out by
    Engine.pinned_empty are views of its buffer, so the memory is released
    (cudaFreeHost) only when the LAST view has died -- never under a live
    array, whatever happens to the trace object or the engine"""

    def __init__(self, lib, address, nbytes):
        self.address = address
        self.buf = (C.c_char*nbytes).from_address(address)
        weakref.finalize(self.buf, lib.rtx_host_free, None, address)


class Engine:
    def __init__(self, device=0, numa=None):
        """`numa`: pin this process to the CPUs / memory of the GPU's NUMA
        node (rtx_numa_bind) so that page-locked buffers are local to the
        GPU's PCIe root; default: only in one-process-per-GPU launches
        (LOCAL_RANK set)."""
        self.lib = _lib.load()
        self.ctx = None
        if self.lib.rtx_device_count() < 1:
            raise RtxError("no CUDA device visible: the rayopt_b200 engine has "
                           "no CPU fallback")
        ctx = C.c_void_p()
        check(self.lib.rtx_init(int(device), C.byref(ctx)))
        self.ctx = ctx
        self.device = int(device)
        self._live = {}
        self.numa_node = None
        import os
        if numa is None:
            numa = "LOCAL_RANK" in os.environ
        if numa:
            self.numa_bind(True)
        sm, fr, tot = C.c_int(), C.c_size_t(), C.c_size_t()
        name = C.create_string_buffer(128)
        check(self.lib.rtx_device_info(self.ctx, C.byref(sm), C.byref(fr), C.byref(tot), name, 128))
        self.sm_count, self.total_bytes = sm.value, tot.value
        self.name = name.value.decode()
        self._fin = weakref.finalize(self, Engine._finalize, self.lib, self.ctx, self._live)

    @staticmethod
    def _finalize(lib, ctx, live):
        # (also runs at interpreter exit) `live` is emptied first so that a
        # DeviceArray collected later sees "not mine any more" and never hands
        # the dangling context back to the library
        try:
            live.clear()
            lib.rtx_free(ctx)
        except Exception:
            pass

    def close(self):
        """Release the context and every DeviceArray still alive.  Page-locked
        arrays from pinned_empty stay valid: they are freed when their last
        numpy view dies."""
        if self.ctx is not None:
            for p in list(self._live.values()):     # device arrays still alive
                self.lib.rtx_free_device(self.ctx, p)
            self._live.clear()
            self._fin.detach()
            self.lib.rtx_free(self.ctx)
            self.ctx = None

    def numa_bind(self, enable=True):
        """rtx_numa_bind: returns the NUMA node (or -1 if not reported)"""
        node = C.c_int(-1)
        check(self.lib.rtx_numa_bind(self.ctx, int(bool(enable)), C.byref(node)))
        self.numa_node = node.value if enable else None
        return node.value

    # ---- memory -------------------------------------------------------
    def empty(self, shape, dtype=np.float64):
        return DeviceArray(self, shape, dtype)

    def to_device(self, a, dtype=None):
        a = np.ascontiguousarray(a, dtype)
        return DeviceArray(self, a.shape, a.dtype).upload(a)

    def pinned_empty(self, shape, dtype=np.float64):
        """numpy array backed by page-locked host memory (full-rate PCIe)"""
        dtype = np.dtype(dtype)
        n = int(np.prod(shape, dtype=np.int64))*dtype.itemsize
        p = C.c_void_p()
        check(self.lib.rtx_host_alloc(self.ctx, max(n, 16), C.byref(p)))
        block = _PinnedBlock(self.lib, p.value, max(n, 16))
        # the array's base chain holds block.buf: freed with the last view
        return np.frombuffer(block.buf, dtype=dtype, count=n//dtype.itemsize).reshape(shape)

    def memset(self, darray, value=0):
        check(self.lib.rtx_memset(self.ctx, darray.ptr, int(value), darray.nbytes))

    def free_bytes(self):
        fr = C.c_size_t()
        check(self.lib.rtx_device_info(self.ctx, None, C.byref(fr), None, None, 0))
        return fr.value

    def sync(self):
        check(self.lib.rtx_sync(self.ctx))

    # ---- timing -------------------------------------------------------
    def timer_start(self):
        check(self.lib.rtx_timer_start(self.ctx))

    def timer_stop(self):
        ms = C.c_float()
        check(self.lib.rtx_timer_stop(self.ctx, C.byref(ms)))
        return ms.value

    def last_kernel_ms(self):
        ms = C.c_float()
        check(self.lib.rtx_last_kernel_ms(self.ctx, C.byref(ms)))
        return ms.value

    def launch_count(self):
        return int(self.lib.rtx_launch_count(self.ctx))

    def last_launch_ctas(self):
        """CTAs the most recent trace kernel launch ran with"""
        n = C.c_int()
        check(self.lib.rtx_last_launch_ctas(self.ctx, C.byref(n)))
        return n.value

    def last_launch_config(self):
        """(rpt, store, warps, nbuf, cluster) of the most recent trace kernel
        launch: rays per thread, store path (0 per-thread, 1 per-warp bulk,
        2 per-CTA bulk), warps per CTA, staging buffers, CTAs per cluster as
        launched"""
        cfg = (C.c_int*5)()
        check(self.lib.rtx_last_launch_config(self.ctx, cfg))
        return tuple(cfg)

    # ---- the hot path -------------------------------------------------
    @staticmethod
    def _table(table):
        table = np.ascontiguousarray(table, SURFACE_DTYPE)
        if table.ndim != 1 or len(table) < 1:
            raise ValueError("surface table must be a non-empty 1-d record array")
        return table

    @staticmethod
    def _flags(exact, direct, rpt=0):
        return ((RTX_EXACT if exact else 0) | (RTX_STORE_DIRECT if direct else 0)
                | {0: 0, 1: RTX_RPT1, 2: RTX_RPT2}[rpt])

    def trace_device(self, table, y0, u0, Y, U, I, T, N=None, ld=None, clip=False,
                     keep_last=False, rot0=None, exact=False, direct=False, rpt=0, mask=None,
                     path_sum=None, path_sum_upto=-1):
        """One launch on DEVICE arrays (DeviceArray or None for outputs).
        Asynchronous on the engine stream.  `mask`: optional uint32
        DeviceArray of ceil(N/32) words receiving the warp-ballot vignetting
        mask (bit set = the ray survives the last surface).  `path_sum`:
        optional (N,) DeviceArray receiving sum_{s <= path_sum_upto} t[s],
        the left-to-right sum of the stored t.  Operands of another dtype
        than the rays, or too small for rows x ld rays (N for path_sum,
        ceil(N/32) words for mask), raise ValueError."""
        table = self._table(table)
        dt = _code(y0.dtype)
        N = y0.shape[0] if N is None else int(N)
        first = next((a for a in (Y, U, I, T) if a is not None), None)
        if ld is None:
            ld = first.shape[1] if first is not None else (N + 63)//64*64
        r0 = None if rot0 is None else np.ascontiguousarray(rot0, np.float64).reshape(9)
        dp = lambda a: None if a is None else a.ptr  # noqa: E731
        if mask is None and path_sum is None and all(a is None for a in (Y, U, I, T)):
            raise ValueError("nothing to store: pass an output array, a mask or a path sum")
        _check_operands(y0.dtype, N, y0=(y0, 3), u0=(u0, 3))
        _check_trace_operands(y0.dtype, N, 1 if keep_last else len(table), int(ld),
                              dict(Y=(Y, 3), U=(U, 3), I=(I, 3), T=(T, 1)), mask, path_sum)
        check(self.lib.rtx_set_mask_output(self.ctx, dp(mask)))
        check(self.lib.rtx_set_path_sum_output(self.ctx, dp(path_sum), int(path_sum_upto)))
        check(self.lib.rtx_trace(
            self.ctx, ptr(table), len(table), ptr(r0), dt, N, y0.ptr, u0.ptr,
            int(bool(clip)), RTX_KEEP_LAST if keep_last else RTX_KEEP_ALL, ld,
            dp(Y), dp(U), dp(I), dp(T), self._flags(exact, direct, rpt)))

    def trace_device_batch(self, tables, y0s, u0s, Ys, Us, Is, Ts, Ns=None, ld=None, clip=False,
                           keep_last=False, rot0=None, exact=False):
        """rtx_trace_batch: several bundles of the same lens (one table each,
        e.g. one per wavelength) in ONE launch.  Lists of DeviceArrays (any of
        Ys/Us/Is/Ts may be None as a whole)."""
        nb = len(tables)
        tabs = [self._table(t) for t in tables]
        S = len(tabs[0])
        if any(len(t) != S for t in tabs):
            raise ValueError("all bundles of a batch must have the same number of surfaces")
        dt = _code(y0s[0].dtype)
        Ns = [a.shape[0] for a in y0s] if Ns is None else [int(n) for n in Ns]
        first = next(a for a in (Ys, Us, Is, Ts) if a is not None)[0]
        ld = first.shape[1] if ld is None else int(ld)
        rows = 1 if keep_last else S
        for b in range(nb):
            pick = lambda xs: None if xs is None else xs[b]  # noqa: E731
            _check_operands(y0s[0].dtype, Ns[b], y0=(y0s[b], 3), u0=(u0s[b], 3))
            _check_trace_operands(y0s[0].dtype, Ns[b], rows, ld,
                                  dict(Y=(pick(Ys), 3), U=(pick(Us), 3), I=(pick(Is), 3),
                                       T=(pick(Ts), 1)))
        vp = C.c_void_p

        def arr(items, get):
            if items is None:
                return None
            return (vp*nb)(*[vp(get(x)) for x in items])
        a_tab = arr(tabs, lambda t: t.ctypes.data)
        a_n = (C.c_int64*nb)(*Ns)
        r0 = None if rot0 is None else np.ascontiguousarray(rot0, np.float64).reshape(9)
        check(self.lib.rtx_trace_batch(
            self.ctx, nb, C.cast(a_tab, vp), S, ptr(r0), dt, C.cast(a_n, vp),
            C.cast(arr(y0s, lambda a: a.ptr), vp), C.cast(arr(u0s, lambda a: a.ptr), vp),
            int(bool(clip)), RTX_KEEP_LAST if keep_last else RTX_KEEP_ALL, ld,
            *[None if x is None else C.cast(arr(x, lambda a: a.ptr), vp) for x in (Ys, Us, Is, Ts)],
            self._flags(exact, False)))

    def trace(self, table, y0, u0, clip=False, keep_last=False, rot0=None,
              dtype=np.float64, exact=False, direct=False, rpt=0, out=None,
              want=("y", "u", "i", "t")):
        """Host arrays in, host arrays out (reference layout): returns
        Y,U,I (rows,N,3), T (rows,N); rows = S or 1.  H2D, kernel and D2H are
        pipelined over ray chunks inside the library."""
        table = self._table(table)
        dtype = np.dtype(dtype)
        dt = _code(dtype)
        y0 = np.ascontiguousarray(y0, dtype)
        u0 = np.ascontiguousarray(u0, dtype)
        if y0.ndim != 2 or y0.shape[1] != 3 or u0.shape != y0.shape:
            raise ValueError("y0, u0 must both be (N, 3)")
        N = y0.shape[0]
        rows = 1 if keep_last else len(table)
        if out is None:
            out = {}
        res = []
        for k, shape in (("y", (rows, N, 3)), ("u", (rows, N, 3)),
                         ("i", (rows, N, 3)), ("t", (rows, N))):
            if k not in want:
                res.append(None)
                continue
            a = out.get(k)
            if a is None:
                a = np.empty(shape, dtype)
            if a.shape != shape or a.dtype != dtype or not a.flags.c_contiguous:
                raise ValueError("output %r must be C-contiguous %s %r" % (k, dtype, shape))
            res.append(a)
        r0 = None if rot0 is None else np.ascontiguousarray(rot0, np.float64).reshape(9)
        check(self.lib.rtx_trace_host(
            self.ctx, ptr(table), len(table), ptr(r0), dt, N, ptr(y0), ptr(u0),
            int(bool(clip)), RTX_KEEP_LAST if keep_last else RTX_KEEP_ALL,
            ptr(res[0]), ptr(res[1]), ptr(res[2]), ptr(res[3]),
            self._flags(exact, direct, rpt)))
        return tuple(res)

    def trace_bundles(self, tables, y0s, u0s, clip=False, keep_last=False, rot0=None,
                      dtype=np.float64, exact=False, want=("y", "u", "i", "t")):
        """rtx_trace_batch_host: many (small) bundles of ONE lens, host arrays
        in and out, one H2D + launches of 8 bundles + one D2H.  `tables[b]`
        the table of bundle b (same number of surfaces), `y0s[b]`, `u0s[b]`
        its (N_b,3) launch rays.  Returns a list of (Y, U, I, T) per bundle
        (None for arrays not in `want`)."""
        nb = len(tables)
        tabs = [self._table(t) for t in tables]
        S = len(tabs[0])
        if any(len(t) != S for t in tabs):
            raise ValueError("all bundles of a batch must have the same number of surfaces")
        dtype = np.dtype(dtype)
        y0s = [np.ascontiguousarray(np.atleast_2d(a), dtype) for a in y0s]
        u0s = [np.ascontiguousarray(np.atleast_2d(a), dtype) for a in u0s]
        Ns = [a.shape[0] for a in y0s]
        rows = 1 if keep_last else S
        outs = {k: ([np.empty((rows, n, 3) if k != "t" else (rows, n), dtype) for n in Ns]
                    if k in want else None) for k in "yuit"}
        vp = C.c_void_p

        def arr(items):
            if items is None:
                return None
            return C.cast((vp*nb)(*[vp(a.ctypes.data) for a in items]), vp)
        keep = [arr(tabs), arr(y0s), arr(u0s)] + [arr(outs[k]) for k in "yuit"]
        r0 = None if rot0 is None else np.ascontiguousarray(rot0, np.float64).reshape(9)
        check(self.lib.rtx_trace_batch_host(
            self.ctx, nb, keep[0], S, ptr(r0), _code(dtype), C.cast((C.c_int64*nb)(*Ns), vp),
            keep[1], keep[2], int(bool(clip)), RTX_KEEP_LAST if keep_last else RTX_KEEP_ALL,
            keep[3], keep[4], keep[5], keep[6], self._flags(exact, False)))
        return [tuple(None if outs[k] is None else outs[k][b] for k in "yuit") for b in range(nb)]

    def trace_gather(self, table, y0, u0, dst_ptrs, dst_offset, N=None, clip=False,
                     rot0=None, exact=False, dst_i_ptrs=None, xy=False, mask=None,
                     path_sum=None, path_sum_upto=-1):
        """rtx_trace_gather: trace the local shard (DEVICE y0,u0) and store
        the last surface's intercepts into every buffer of `dst_ptrs` (raw
        device pointers: local or peer memory) at ray offset `dst_offset`;
        `dst_i_ptrs`: a second set of buffers for the incidence directions;
        `xy`: the intercept buffers are (Ntotal, 2) and receive x,y only.
        `mask`, `path_sum`: the side outputs of trace_device for the shard's
        N rays; without them both are switched off, so that a gather never
        writes into buffers an earlier trace_device registered."""
        table = self._table(table)
        N = y0.shape[0] if N is None else int(N)
        _check_operands(y0.dtype, N, y0=(y0, 3), u0=(u0, 3))
        _check_trace_operands(y0.dtype, N, 1, N, {}, mask, path_sum)
        dp = lambda a: None if a is None else a.ptr  # noqa: E731
        check(self.lib.rtx_set_mask_output(self.ctx, dp(mask)))
        check(self.lib.rtx_set_path_sum_output(self.ctx, dp(path_sum), int(path_sum_upto)))
        r0 = None if rot0 is None else np.ascontiguousarray(rot0, np.float64).reshape(9)
        arr = (C.c_void_p*len(dst_ptrs))(*[C.c_void_p(int(p)) for p in dst_ptrs])
        arr_i = None
        if dst_i_ptrs is not None:
            if len(dst_i_ptrs) != len(dst_ptrs):
                raise ValueError("dst_i_ptrs must match dst_ptrs")
            arr_i = C.cast((C.c_void_p*len(dst_ptrs))(*[C.c_void_p(int(p)) for p in dst_i_ptrs]),
                           C.c_void_p)
        check(self.lib.rtx_trace_gather(
            self.ctx, ptr(table), len(table), ptr(r0), _code(y0.dtype), N, y0.ptr, u0.ptr,
            int(bool(clip)), len(dst_ptrs), C.cast(arr, C.c_void_p), arr_i, int(dst_offset),
            self._flags(exact, False) | (_lib.RTX_GATHER_XY if xy else 0)))

    # ---- fused epilogues (no per-surface stores) -------------------------
    def trace_reduce(self, table, y0, u0, N=None, clip=False, rot0=None, exact=False, w=None,
                     center=None):
        """rtx_trace_reduce: march the DEVICE launch rays to the last surface
        of `table` and return the 20 rms / refocus moments of that surface
        (include/rtx.h) -- one launch, no intercept is stored.  `center`:
        (y_x, y_y, u_x, u_y) guess centres (e.g. the chief ray's)."""
        table = self._table(table)
        N = y0.shape[0] if N is None else int(N)
        _check_operands(y0.dtype, N, y0=(y0, 3), u0=(u0, 3), w=(w, 1))
        r0 = None if rot0 is None else np.ascontiguousarray(rot0, np.float64).reshape(9)
        c = None if center is None else np.ascontiguousarray(center, np.float64).reshape(4)
        m = np.zeros(20)
        check(self.lib.rtx_trace_reduce(
            self.ctx, ptr(table), len(table), ptr(r0), _code(y0.dtype), N, y0.ptr, u0.ptr,
            int(bool(clip)), None if w is None else w.ptr, ptr(c), ptr(m),
            self._flags(exact, False)))
        return m

    @staticmethod
    def rms_from_moments(m, unit_weights=False, about_center=False):
        """GeometricTrace.rms (rayopt/geometric_trace.py:171-183) from the
        moments of ONE pass about a guess centre c: the spot is re-centred on
        the unweighted mean analytically, sum w |y - ybar|^2 = m3 - 2 ybar.(m1,
        m2) + |ybar|^2 m0 with ybar = (m6, m7)/N relative to c (cancellation
        free when c is within the spot).  Not NaN-masked, like the reference.
        `about_center`: rms about c itself (the reference's `ref` ray).
        `unit_weights`: the moments were taken with w = 1 -> default 1/N."""
        if m[4] != m[5] or m[5] == 0:
            return float("nan")
        if about_center:
            r2 = m[3]
        else:
            bx, by = m[6]/m[5], m[7]/m[5]
            r2 = m[3] - 2*(bx*m[1] + by*m[2]) + (bx*bx + by*by)*m[0]
        if unit_weights:
            r2 /= m[5]
        return float(np.sqrt(max(r2, 0.)))

    @staticmethod
    def focus_shift_from_moments(m):
        """the shift of GeometricTrace.refocus (rayopt/geometric_trace.py:82-99),
        t = -<w dy, du>/<w du, du> about the unweighted means of the rays
        with finite slope, from the one-pass sums m[8..19]"""
        G = m[8]
        if G == 0:
            return float("nan")
        by, bu = m[9:11]/G, m[11:13]/G
        W, Wy, Wu = m[13], m[14:16], m[16:18]
        num = m[18] - by.dot(Wu) - bu.dot(Wy) + by.dot(bu)*W
        den = m[19] - 2*bu.dot(Wu) + bu.dot(bu)*W
        return float(-num/den)

    def trace_opd(self, table, y0, u0, spec, A, P, N=None, clip=False, rot0=None, exact=False):
        """rtx_trace_opd: `spec` a dict with the members of `struct rtx_opd`
        (include/rtx.h); A (N,), P (N,3) DeviceArrays.  Asynchronous."""
        table = self._table(table)
        N = y0.shape[0] if N is None else int(N)
        _check_operands(y0.dtype, N, y0=(y0, 3), u0=(u0, 3), A=(A, 1), P=(P, 3))
        r0 = None if rot0 is None else np.ascontiguousarray(rot0, np.float64).reshape(9)
        rec = np.zeros(1, OPD_DTYPE)
        for k in ("y0_ref", "u0_ref", "M", "d"):
            rec[k] = np.asarray(spec[k], float).reshape(rec[k].shape[1:])
        for k in ("n0", "n_after", "radius"):
            rec[k] = float(spec[k])
        rec["infinite"] = int(bool(spec["infinite"]))
        check(self.lib.rtx_trace_opd(
            self.ctx, ptr(table), len(table), ptr(r0), _code(y0.dtype), N, y0.ptr, u0.ptr,
            int(bool(clip)), ptr(rec), A.ptr, P.ptr, self._flags(exact, False)))

    def ipc_export(self, darray):
        h = (C.c_ubyte*64)()
        check(self.lib.rtx_ipc_export(self.ctx, darray.ptr, C.cast(h, C.c_void_p)))
        return bytes(h)

    def ipc_open(self, handle):
        h = (C.c_ubyte*64).from_buffer_copy(handle)
        p = C.c_void_p()
        check(self.lib.rtx_ipc_open(self.ctx, C.cast(h, C.c_void_p), C.byref(p)))
        return p.value

    def ipc_close(self, p):
        check(self.lib.rtx_ipc_close(self.ctx, p))

    def download_rays(self, darray, idx):
        """host copy of rays `idx` (1-d integer array) of a device array whose
        trailing axes are (rays, 3) -- a row view (1, ld, 3) or an (N, 3)
        array: one strided D2H when `idx` is an arithmetic progression, else one
        24-byte copy per ray (samples for parity checks)"""
        idx = np.asarray(idx, np.int64).reshape(-1)
        item = darray.dtype.itemsize*3
        out = np.empty((len(idx), 3), darray.dtype)
        if len(idx) == 0:
            return out
        step = int(idx[1] - idx[0]) if len(idx) > 1 else 1
        if len(idx) > 1 and step > 0 and np.all(np.diff(idx) == step):
            check(self.lib.rtx_memcpy2d_d2h(self.ctx, ptr(out), item, darray.ptr + int(idx[0])*item,
                                            step*item, item, len(idx)))
        else:
            for j, i in enumerate(idx):
                check(self.lib.rtx_memcpy_d2h(self.ctx, out[j].ctypes.data_as(C.c_void_p),
                                              darray.ptr + int(i)*item, item))
        self.sync()
        return out

    def aim_infinite_device(self, yo, z, p, angle, yp=None, nrays=None, dtype=np.float64,
                            rings=None):
        """Launch rays of an aimed bundle for an infinite object (rectilinear
        projection, plane object surface) generated in HBM: `yp` a DEVICE
        (N,2) FP64 array of pupil coordinates, or None for the hexapolar grid
        with about `nrays` rays (or exactly `rings` rings).  Host
        restatement: rays.aim_infinite.  Returns DeviceArrays (y0, u0)."""
        from .rays import infinite_record, pupil_grid
        return self.aim_rays(infinite_record(yo, z, p, angle, grid=pupil_grid(yp, nrays, rings)),
                             dtype, yp=yp)

    def aim_finite_device(self, yo, z, p, radius, yp=None, nrays=None, dtype=np.float64):
        """Launch rays of an aimed bundle from a FINITE object (non-telecentric
        pupil, plane object surface) generated in HBM, `yp` and `nrays` as in
        aim_infinite_device.  Host restatement: rays.aim_finite.  Returns
        (y0, u0)."""
        from .rays import finite_record, pupil_grid
        return self.aim_rays(finite_record(yo, z, p, radius, grid=pupil_grid(yp, nrays)),
                             dtype, yp=yp)

    def aim_rays(self, spec, dtype=np.float64, first=0, count=None, yp=None, want_pupil=False):
        """rtx_aim_plan + rtx_aim_rays: launch rays `first .. first+count-1` of
        the bundle a `rtx_aim` record (rays.aim_record) describes, generated in
        HBM.  `yp`: DEVICE (n,2) FP64 pupil coordinates for GRID_GIVEN.
        Returns (y0, u0) DeviceArrays, plus the (count,2) pupil coordinates
        when `want_pupil`."""
        spec = np.ascontiguousarray(spec)
        n_given, ypp = _given(yp)
        total = C.c_int64()
        check(self.lib.rtx_aim_plan(self.ctx, ptr(spec), n_given, ypp, C.byref(total)))
        count = total.value - first if count is None else int(count)
        y0, u0 = self.empty((count, 3), dtype), self.empty((count, 3), dtype)
        po = self.empty((count, 2), np.float64) if want_pupil else None
        check(self.lib.rtx_aim_rays(self.ctx, ptr(spec), n_given, ypp, _code(dtype), int(first),
                                    count, y0.ptr, u0.ptr, None if po is None else po.ptr))
        return (y0, u0, po) if want_pupil else (y0, u0)

    def aim_rays_into(self, spec, y_dst, u_dst, count, first=0, yp=None):
        """rtx_aim_rays into existing device rows (DeviceArray views)"""
        spec = np.ascontiguousarray(spec)
        n_given, ypp = _given(yp)
        check(self.lib.rtx_aim_rays(self.ctx, ptr(spec), n_given, ypp, _code(y_dst.dtype),
                                    int(first), int(count), y_dst.ptr, u_dst.ptr, None))

    def aim_count(self, spec, yp=None):
        """number of rays the record generates (after clipping / filtering)"""
        spec = np.ascontiguousarray(spec)
        n_given, ypp = _given(yp)
        total = C.c_int64()
        check(self.lib.rtx_aim_plan(self.ctx, ptr(spec), n_given, ypp, C.byref(total)))
        return total.value

    def selftest_math(self, a, b):
        """(6, n): engine a/b, IEEE a/b, engine sqrt(a), IEEE sqrt(a),
        engine 1/sqrt(a), IEEE 1/sqrt(a)"""
        a = np.ascontiguousarray(a, np.float64)
        b = np.ascontiguousarray(b, np.float64)
        out = np.empty((6, a.size))
        check(self.lib.rtx_selftest_math(self.ctx, a.size, ptr(a), ptr(b), ptr(out)))
        return out

    def selftest_math2(self, a, b, c):
        """(7, n): shared-reciprocal a/b and c/b, IEEE a/b and c/b, fast 1/b,
        fast sqrt(a) and 1/sqrt(a)"""
        a, b, c = (np.ascontiguousarray(x, np.float64) for x in (a, b, c))
        if not a.shape == b.shape == c.shape:
            raise ValueError("a, b, c must have one shape")
        out = np.empty((7, a.size))
        check(self.lib.rtx_selftest_math2(self.ctx, a.size, ptr(a), ptr(b), ptr(c), ptr(out)))
        return out

    def moments(self, y, w=None, N=None, center=None):
        """Weighted moments of device intercepts about `center`
        (include/rtx.h rtx_moments): 8 doubles."""
        m = np.zeros(8)
        N = y.shape[-2] if N is None else int(N)
        _check_operands(y.dtype, N, y=(y, 3), w=(w, 1))
        c = None if center is None else np.ascontiguousarray(center, np.float64)
        check(self.lib.rtx_moments(self.ctx, _code(y.dtype), N, y.ptr,
                                   None if w is None else w.ptr, ptr(c), ptr(m)))
        return m

    def rms(self, y, w=None, N=None, ref_point=None, comm_sum=None):
        """GeometricTrace.rms (rayopt/geometric_trace.py:171-183) of device
        intercepts `y` (N,3) without a D2H of the rays: centre = unweighted
        mean (or `ref_point`), rms = sqrt(sum w |y - y0|^2) with the
        reference's default weights 1/N when `w` is None.  Like the
        reference it is NOT NaN-masked: any non-finite ray gives NaN.
        `comm_sum` (callable: 8-vector -> summed 8-vector) makes it the rms of
        a ray-sharded bundle (one all-reduce per pass)."""
        red = comm_sum or (lambda v: v)
        if ref_point is None:
            m = red(self.moments(y, w, N))
            if m[4] != m[5]:
                return float("nan")
            ref_point = (m[6]/m[5], m[7]/m[5])
        m = red(self.moments(y, w, N, center=ref_point))
        if m[4] != m[5]:
            return float("nan")
        return float(np.sqrt(m[3]/m[5] if w is None else m[3]))


    def refocus_shift(self, y, inc, w=None, N=None, comm_sum=None):
        """The focus shift of GeometricTrace.refocus (rayopt/geometric_trace.py:
        82-99), t = -<w y, u>/<w u, u> about the means of the finite rays, from
        DEVICE arrays y (N,3) and inc (N,3) of the surface -- no D2H of the rays.
        `comm_sum` all-reduces the 8 moments for ray-sharded bundles."""
        red = comm_sum or (lambda v: v)
        N = y.shape[-2] if N is None else int(N)
        _check_operands(y.dtype, N, y=(y, 3), inc=(inc, 3), w=(w, 1))

        def mom(center):
            m = np.zeros(8)
            c = None if center is None else np.ascontiguousarray(center, np.float64)
            check(self.lib.rtx_focus_moments(self.ctx, _code(y.dtype), N, y.ptr, inc.ptr,
                                             None if w is None else w.ptr, ptr(c), ptr(m)))
            return red(m)
        m = mom(None)
        if m[0] == 0:
            return float("nan")
        m = mom(m[2:6]/m[0])
        return float(-m[6]/m[7])

    # ---- diffraction PSF (GeometricTrace.psf, rayopt/geometric_trace.py:133-169)
    def grid_linear(self, points, values, tri, n, gh, download=True, winner=False):
        """rtx_grid_linear: griddata(points, values, (xs, ys), method="linear",
        fill_value=nan) on the grid node (i, j) = (gh[i], gh[j]), with the
        triangulation `tri` of `points`: scipy.spatial.Delaunay on the host,
        or a DeviceTriangulation (``delaunay``), whose arrays are used in place;
        `points` may be a DeviceArray, used in place too.
        Returns the (n, n) values -- numpy, or a DeviceArray when not
        `download` -- and with `winner` also the covering simplex per node
        (numpy int32, -1 where none covers it, like find_simplex)."""
        dev_points = isinstance(points, DeviceArray)
        if not dev_points:
            points = np.ascontiguousarray(points, np.float64)
        values = np.ascontiguousarray(values, np.float64)
        gh = np.ascontiguousarray(gh, np.float64)
        if len(points.shape) != 2 or points.shape[1] != 2 or values.shape != points.shape[:1] \
                or np.dtype(points.dtype) != np.float64:
            raise ValueError("points must be (M, 2) FP64 and values (M,)")
        if gh.shape != (int(n),):
            raise ValueError("gh must be the (n,) grid axis")
        n = int(n)
        ins = [self.to_device(a) for a in (values, gh)]
        if not dev_points:
            ins.append(self.to_device(points))
        pts_ptr = points.ptr if dev_points else ins[-1].ptr
        if isinstance(tri, DeviceTriangulation):
            ntri, simp_ptr, tr_ptr = tri.T, tri.simplices.ptr, tri.transform.ptr
        else:
            simp = np.ascontiguousarray(tri.simplices, np.int32)
            tr = np.ascontiguousarray(tri.transform, np.float64)
            ins += [self.to_device(simp), self.to_device(tr)]
            ntri, simp_ptr, tr_ptr = len(simp), ins[-2].ptr, ins[-1].ptr
        out = self.empty((n, n))
        win = self.empty((n, n), np.int32) if winner else None
        try:
            check(self.lib.rtx_grid_linear(self.ctx, RTX_F64, points.shape[0], pts_ptr, ins[0].ptr,
                                           ntri, simp_ptr, tr_ptr, n, ins[1].ptr,
                                           out.ptr, None if win is None else win.ptr))
            w = None
            if win is not None:
                w = win.download()
                w[w == np.iinfo(np.int32).max] = -1
                win.free()
            if download:
                o = out.download()
                out.free()
                out = o
            else:
                self.sync()
        finally:
            for a in ins:
                a.free()
        return (out, w) if winner else out

    def selftest_predicates(self, quads):
        """(n, 2) int: the device's exact orient2d(a, b, c) and incircle(a, b,
        c, d) signs of n point quadruples `quads` (n, 4, 2)"""
        q = np.ascontiguousarray(quads, np.float64).reshape(-1, 8)
        out = np.empty((len(q), 2), np.int32)
        check(self.lib.rtx_selftest_predicates(self.ctx, len(q), ptr(q), ptr(out)))
        return out

    def delaunay_bytes(self, m):
        """device bytes of rtx_delaunay's workspace for m points"""
        b = C.c_size_t()
        check(self.lib.rtx_delaunay_bytes(self.ctx, int(m), C.byref(b)))
        return b.value

    def delaunay(self, points):
        """rtx_delaunay: the Delaunay triangulation of `points` (M, 2) FP64,
        numpy or a DeviceArray, computed on the device.  Returns a
        DeviceTriangulation whose simplices, neighbors and transform stay in
        HBM (scipy.spatial.Delaunay's layout)."""
        if isinstance(points, DeviceArray):
            if points.dtype != np.float64 or len(points.shape) != 2 or points.shape[1] != 2:
                raise ValueError("points must be an (M, 2) FP64 device array")
            dp, own = points, None
        else:
            a = np.ascontiguousarray(points, np.float64)
            if a.ndim != 2 or a.shape[1] != 2:
                raise ValueError("points must be (M, 2)")
            dp = own = self.to_device(a)
        m = dp.shape[0]
        cap = max(2*m, 1)
        simp, nbr, tr = self.empty((cap, 3), np.int32), self.empty((cap, 3), np.int32), \
            self.empty((cap, 3, 2))
        T = C.c_int64()
        try:
            check(self.lib.rtx_delaunay(self.ctx, RTX_F64, m, dp.ptr, C.byref(T), simp.ptr,
                                        nbr.ptr, tr.ptr))
        except Exception:
            for a in (simp, nbr, tr):
                a.free()
            raise
        finally:
            if own is not None:
                own.free()
        return DeviceTriangulation(int(T.value), simp, nbr, tr)

    def psf_bytes(self, n, pad):
        """device bytes rtx_psf allocates for itself on an (n, n) grid"""
        _lib.preload_cufft()
        b = C.c_size_t()
        check(self.lib.rtx_psf_bytes(self.ctx, int(n), int(pad), C.byref(b)))
        return b.value

    def psf(self, o, pad):
        """rtx_psf of the regridded OPD `o` (DEVICE (n, n) FP64): the
        (pad n, pad n) PSF |fft2(exp(-2 pi i o)/sqrt(#finite))|^2/(pad n)^2 as
        a DeviceArray, and the device's raw stats (#finite, sum, max,
        sum psf k_p, sum psf k_q; include/rtx.h) for ``psf_stats``.  Raises
        RtxError (RTX_E_NOMEM) before allocating anything when the PSF and
        the library's buffers do not fit in free device memory."""
        n, pad = int(o.shape[0]), int(pad)
        if o.shape != (n, n) or o.dtype != np.float64:
            raise ValueError("o must be a square FP64 device array")
        nx = n*pad
        free = self.free_bytes()
        # the complex grid and the PSF alone, then with cuFFT's work area
        if nx*nx*(16 + 8) > free or self.psf_bytes(n, pad) + nx*nx*8 > free:
            check(_lib.RTX_E_NOMEM)
        out = self.empty((nx, nx))
        raw = np.zeros(5)
        try:
            check(self.lib.rtx_psf(self.ctx, RTX_F64, n, o.ptr, pad, out.ptr, ptr(raw)))
        except Exception:
            out.free()
            raise
        return out, raw

    @staticmethod
    def psf_stats(raw, f):
        """count, sum, peak and the first moments sum psf*p, sum psf*q of a
        PSF on the frequency axis `f` (np.fft.fftfreq(nx, d)) from the raw
        device stats of ``psf``"""
        nx = len(f)
        step = f[1] if nx > 1 else 0.        # fftfreq: f[k] = k/(nx d)
        return dict(count=int(raw[0]), sum=float(raw[1]), max=float(raw[2]),
                    cp=float(raw[3]*step), cq=float(raw[4]*step))

    @staticmethod
    def profile_nbins(shape, center):
        """np.bincount's length for the radial bins of an array of `shape`
        about `center`: 1 + the largest bin, at a corner (polar_sum's
        arithmetic, aspect 1, binsize 1); 0 for a non-finite centre or a
        radius of 2^50 or more, which rtx_psf_profiles refuses"""
        i = np.array([0., shape[0] - 1]) - float(center[0])
        j = np.array([0., shape[1] - 1]) - float(center[1])
        with np.errstate(all="ignore"):
            r = np.sqrt(j[None, :]*j[None, :] + i[:, None]*i[:, None])
        if not (r < 2.**50).all():
            return 0
        return int(r.astype(np.int64).max()) + 1

    def psf_profiles(self, psf, center):
        """rtx_psf_profiles of the PSF `psf` (DEVICE (nx, ny) FP64, the FFT
        order of ``psf``) about `center` (c0, c1) in the fftshifted frame:
        (ee_bins, lsf0, lsf1) as numpy arrays -- polar_sum(fftshift(psf),
        center, "azimuthal") and the column and row sums in the stored order
        (ifftshift(fftshift(psf).sum(i)) for i = 0, 1).  Raises RtxError for a
        negative or non-finite pixel."""
        if len(psf.shape) != 2 or psf.dtype != np.float64:
            raise ValueError("psf must be a 2-d FP64 device array")
        nx, ny = psf.shape
        c0, c1 = float(center[0]), float(center[1])
        nbins = self.profile_nbins(psf.shape, (c0, c1))
        ee, lsf0, lsf1 = np.empty(nbins), np.empty(ny), np.empty(nx)
        check(self.lib.rtx_psf_profiles(self.ctx, RTX_F64, nx, ny, psf.ptr, c0, c1, nbins,
                                        ptr(ee), ptr(lsf0), ptr(lsf1)))
        return ee, lsf0, lsf1


_default = {}


def default_engine(device=0):
    """process-wide engine for `device` (created on first use)"""
    e = _default.get(device)
    if e is None or e.ctx is None:
        e = _default[device] = Engine(device)
    return e
