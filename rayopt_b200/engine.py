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

# mirrors `struct rtx_spot` (include/rtx.h)
SPOT_MAX_PLANES = 16
SPOT_DTYPE = np.dtype([("planes", "<i4"), ("radial", "<i4"), ("nx", "<i8"), ("ny", "<i8"),
                       ("range", "<f8", (2, 2)), ("c", "<f8", (2,)),
                       ("z", "<f8", (SPOT_MAX_PLANES,)), ("o", "<f8", (SPOT_MAX_PLANES, 2))],
                      align=True)


def spot_spec(z, bins, range, center, radial=False, offsets=None):
    """An rtx_spot record: defocus distances `z` (K,), `bins` (nx, ny) (radial:
    nx or (nx,)), `range` ((x_lo, x_hi), (y_lo, y_hi)) (radial: (r_lo, r_hi)),
    the chief intercept `center` (2,) and per-plane `offsets` (K, 2) or None.
    The library checks the values (RtxError); more than 16 planes are passed
    on as a count for it to refuse."""
    z = np.atleast_1d(np.asarray(z, np.float64))
    K = len(z)
    rec = np.zeros(1, SPOT_DTYPE)
    rec["planes"], rec["radial"] = K, int(bool(radial))
    b = np.atleast_1d(np.asarray(bins, np.int64))
    rec["nx"], rec["ny"] = (b[0], b[1]) if len(b) > 1 else (b[0], 1 if radial else b[0])
    r = np.asarray(range, np.float64).reshape(-1, 2)
    rec["range"][0, :len(r)] = r[:2]
    rec["c"] = np.asarray(center, np.float64).reshape(2)
    k = min(K, SPOT_MAX_PLANES)
    rec["z"][0, :k] = z[:k]
    if offsets is not None:
        rec["o"][0, :k] = np.asarray(offsets, np.float64).reshape(K, 2)[:k]
    return rec


# mirrors `struct rtx_otf` (include/rtx.h)
OTF_MAX_PLANES, OTF_MAX_FREQS = 16, 256
WFE_NSUMS = 10      # RTX_WFE_NSUMS: n, sum a, a^2, x, y, x^2, xy, y^2, ax, ay
ZRN_MAX_ORDER = 8   # RTX_ZRN_MAX_ORDER
OTF_SLOT, OTF_BLOCK = 16384, 16      # RTX_OTF_SLOT, RTX_OTF_BLOCK
MAX_PARAMS, JAC_SLOT = 64, 16384     # RTX_MAX_PARAMS, RTX_JAC_SLOT
OTF_DTYPE = np.dtype([("planes", "<i4"), ("nfreq", "<i4"), ("dnu", "<f8"), ("c", "<f8", (2,)),
                      ("z", "<f8", (OTF_MAX_PLANES,)), ("o", "<f8", (OTF_MAX_PLANES, 2))],
                     align=True)


def otf_spec(z, dnu, nfreq, c, offsets=None):
    """An rtx_otf record: defocus distances `z` (K,), frequencies
    ``arange(nfreq)*dnu``, the centre `c` (2,) subtracted from the
    intercepts and per-plane `offsets` (K, 2) or None.  Raises ValueError
    for what rtx_otf_rows refuses: K outside 1..16, nfreq outside 1..256,
    a non-finite dnu, c, z or offset."""
    z = np.atleast_1d(np.asarray(z, np.float64))
    K, F = len(z), int(nfreq)
    if z.ndim != 1 or not 1 <= K <= OTF_MAX_PLANES:
        raise ValueError("need 1..%d planes, got %d" % (OTF_MAX_PLANES, K))
    if not 1 <= F <= OTF_MAX_FREQS:
        raise ValueError("need 1..%d frequencies, got %d" % (OTF_MAX_FREQS, F))
    o = np.zeros((K, 2)) if offsets is None else np.asarray(offsets, np.float64).reshape(K, 2)
    c = np.asarray(c, np.float64).reshape(2)
    dnu = float(dnu)
    if not (np.isfinite(dnu) and np.isfinite(c).all() and np.isfinite(z).all()
            and np.isfinite(o).all()):
        raise ValueError("dnu, c, z and offsets must be finite")
    rec = np.zeros(1, OTF_DTYPE)
    rec["planes"], rec["nfreq"], rec["dnu"], rec["c"] = K, F, dnu, c
    rec["z"][0, :K], rec["o"][0, :K] = z, o
    return rec


# mirrors `struct rtx_pupil` (include/rtx.h)
PUPIL_MAX_PLANES, PUPIL_MAX_PIXELS = 16, 4096
PUPIL_CHUNK, PUPIL_SLOT, PUPIL_MAX_SLOTS = 32, 2048, 16
PUPIL_DTYPE = np.dtype([("planes", "<i4"), ("reserved", "<i4"), ("nx", "<i8"), ("ny", "<i8"),
                        ("a0", "<f8"), ("wavelength", "<f8"), ("kappa", "<f8"), ("radius", "<f8"),
                        ("p0", "<f8"), ("dp", "<f8"), ("q0", "<f8"), ("dq", "<f8"),
                        ("z", "<f8", (PUPIL_MAX_PLANES,))], align=True)


def pupil_spec(z, pixels, p0, dp, q0, dq, a0, wavelength, kappa, radius):
    """An rtx_pupil record: defocus distances `z` (K,), the grid p_a = p0 +
    a dp, q_b = q0 + b dq of `pixels` (nx, ny), the reference path a0, the
    wavelength and kappa = n_image/wavelength in lens units and the sphere
    radius.  Raises ValueError for what rtx_pupil_sum refuses."""
    z = np.atleast_1d(np.asarray(z, np.float64))
    nx, ny = (int(v) for v in pixels)
    if z.ndim != 1 or not 1 <= len(z) <= PUPIL_MAX_PLANES:
        raise ValueError("need 1..%d planes, got %d" % (PUPIL_MAX_PLANES, len(z)))
    if not (1 <= nx <= PUPIL_MAX_PIXELS and 1 <= ny <= PUPIL_MAX_PIXELS):
        raise ValueError("pixels must be in 1..%d, got %r" % (PUPIL_MAX_PIXELS, (nx, ny)))
    v = np.array([p0, dp, q0, dq, a0, wavelength, kappa, radius], np.float64)
    if not (np.isfinite(v).all() and np.isfinite(z).all()) or wavelength == 0 or radius == 0:
        raise ValueError("grid, a0, kappa and z must be finite, wavelength and radius "
                         "finite and non-zero")
    rec = np.zeros(1, PUPIL_DTYPE)
    rec["planes"], rec["nx"], rec["ny"] = len(z), nx, ny
    for k, x in zip(("p0", "dp", "q0", "dq", "a0", "wavelength", "kappa", "radius"), v):
        rec[k] = x
    rec["z"][0, :len(z)] = z
    return rec


def pupil_bound(N, phi, sum_abs_w, chunks=1):
    """The error bound of include/rtx.h on every component of the U one
    rtx_pupil_sum call of N rays adds, ``(D + 24 phi + 40) eps sum|w|``,
    plus ``chunks - 1`` for calls added in order; `phi` the largest phase
    sum of include/rtx.h over the summed rays"""
    L = max(PUPIL_SLOT, -(-int(N)//PUPIL_MAX_SLOTS))
    L = -(-L//PUPIL_CHUNK)*PUPIL_CHUNK
    slots = -(-int(N)//L)
    D = 2*PUPIL_CHUNK + -(-L//PUPIL_CHUNK) + slots + 1 + chunks - 1
    return (D + 24*np.asarray(phi, np.float64) + 40)*2.**-52*np.asarray(sum_abs_w)


def otf_bound(spec, N, count, phi, chunks=1):
    """The error bound of include/rtx.h on every component of S, per plane
    (K,): ``(D + 13 phi + 5 RTX_OTF_BLOCK) eps count`` with the summation
    depth D of N rays in one call, plus ``chunks - 1`` for calls added in
    order; `phi` the largest |nu_j q| over the counted rays"""
    slots = -(-int(N)//OTF_SLOT)
    D = OTF_SLOT//8 + 8 + slots + chunks - 1
    return (D + 13*np.asarray(phi, np.float64) + 5*OTF_BLOCK)*2.**-52*np.asarray(count)


def jacobian_sums_unpack(out, P):
    """rtx_jacobian_sums' row (include/rtx.h) as a dict; rows of several
    calls may be added first"""
    out = np.asarray(out, np.float64)
    K = np.zeros((P, P))
    iu = np.triu_indices(P)
    K[iu] = out[4 + 3*P:4 + 3*P + len(iu[0])]
    K.T[iu] = K[iu]
    return dict(n=out[0], sum_d=out[1:3].copy(), sum_d2=out[3], G=out[4:4 + 2*P].reshape(P, 2),
                H=out[4 + 2*P:4 + 3*P].copy(), K=K, bad=out[-1], out=out)


def wavefront_sums_unpack(out, P):
    """rtx_wavefront_sums' row (include/rtx.h) as a dict; rows of several
    calls may be added first"""
    out = np.asarray(out, np.float64)
    K = np.zeros((P, P))
    iu = np.triu_indices(P)
    K[iu] = out[3 + 2*P:3 + 2*P + len(iu[0])]
    K.T[iu] = K[iu]
    return dict(n=out[0], sum_d=out[1], sum_d2=out[2], G=out[3:3 + P].copy(),
                H=out[3 + P:3 + 2*P].copy(), K=K, bad=out[-1], out=out)


def otf_jacobian_sums_unpack(out, P, F):
    """rtx_otf_jacobian_sums' row (include/rtx.h) as a dict: n, bad, S
    complex (2, F), dS complex (P, 2, F) and the row `out`; rows of several
    calls may be added first"""
    out = np.asarray(out, np.float64)
    S = out[1:1 + 4*F].reshape(2, F, 2)
    dS = out[1 + 4*F:1 + 4*F + 4*P*F].reshape(P, 2, F, 2)
    return dict(n=out[0], bad=out[-1], S=S[..., 0] + 1j*S[..., 1], dS=dS[..., 0] + 1j*dS[..., 1],
                out=out)


def spot_shape(spec):
    """(K, nx, ny) of a 2-D record, (K, nx) of a radial one"""
    s = spec[0]
    K, nx = int(s["planes"]), int(s["nx"])
    return (K, nx) if s["radial"] else (K, nx, int(s["ny"]))


def _code(dtype):
    try:
        return _DTYPES[np.dtype(dtype)]
    except KeyError:
        raise TypeError("dtype must be float64 or float32, got %r" % (dtype,))


def _rooms(dtype, arrays):
    """(name, room in rays) of each (DeviceArray, values per ray) in `arrays`
    (None entries are skipped); ValueError for one of another dtype"""
    for name, (a, per_ray) in arrays.items():
        if a is None:
            continue
        if np.dtype(a.dtype) != dtype:
            raise ValueError("%s is %s but the rays are %s" % (name, np.dtype(a.dtype), dtype))
        yield name, a.nbytes//(dtype.itemsize*per_ray)


def _check_operands(dtype, N, **arrays):
    """The reductions and epilogues take their element type from the rays and
    read N rays from every other array: each (DeviceArray, values per ray)
    in `arrays` (None entries are skipped) must have that dtype and room for N
    rays.  Raises ValueError before anything is launched."""
    dtype = np.dtype(dtype)
    if N < 0:
        raise ValueError("N must be >= 0, got %d" % N)
    for name, room in _rooms(dtype, arrays):
        if N > room:
            raise ValueError("N = %d rays but %s holds only %d" % (N, name, room))


def _check_trace_operands(dtype, N, rows, ld, outputs, mask=None, path_sum=None):
    """A trace writes rows x ld rays into each of Y, U, I (3 values per ray)
    and T (1), N values of the rays' dtype into `path_sum` and ceil(N/32)
    32-bit words into `mask`: refuse (ValueError, before anything is
    launched) an operand of another element type or one too small for that."""
    dtype = np.dtype(dtype)
    _check_operands(dtype, N, path_sum=(path_sum, 1))
    for name, room in _rooms(dtype, outputs):
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


def _rot0(rot0):
    """the optional 3x3 launch rotation as 9 contiguous doubles"""
    return None if rot0 is None else np.ascontiguousarray(rot0, np.float64).reshape(9)


def _opd_record(spec):
    """the rtx_opd record of a dict with its members (lazy.opd_spec)"""
    rec = np.zeros(1, OPD_DTYPE)
    for k in ("y0_ref", "u0_ref", "M", "d"):
        rec[k] = np.asarray(spec[k], float).reshape(rec[k].shape[1:])
    for k in ("n0", "n_after", "radius"):
        rec[k] = float(spec[k])
    rec["infinite"] = int(bool(spec["infinite"]))
    return rec


def _moves(y0, moves, S):
    """(P, param_first, move_row, moves) of the derivative marches from P
    lists of (row, record) on a table of S rows; ValueError for FP32 rays,
    a bad P, a parameter without moves, a row out of range or a move that
    is not one record"""
    if np.dtype(y0.dtype) != np.float64:
        raise ValueError("the Jacobian is FP64 only, got %s rays" % np.dtype(y0.dtype))
    P = len(moves)
    if not 1 <= P <= MAX_PARAMS:
        raise ValueError("need 1..%d parameters, got %d" % (MAX_PARAMS, P))
    rows, recs = [], []
    for p, mv in enumerate(moves):
        if not len(mv):
            raise ValueError("parameter %d has no moves" % p)
        for row, rec in mv:
            if not 0 <= int(row) < S:
                raise ValueError("move row %r is not in 0..%d" % (row, S - 1))
            rows.append(int(row))
            recs.append(rec)
    first = np.cumsum([0] + [len(mv) for mv in moves]).astype(np.int32)
    rows = np.ascontiguousarray(rows, np.int32)
    recs = np.ascontiguousarray(np.array(recs, SURFACE_DTYPE))
    if recs.shape != rows.shape:
        raise ValueError("each move must be one record (a (W, S) table's record_tangents "
                         "gives (W,) records: pick one wavelength), got %s for %d moves"
                         % (recs.shape, len(rows)))
    return P, first, rows, recs


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

    def _march(self, table, y0, u0, N, clip, rot0, **operands):
        """The prologue of the calls that march DEVICE launch rays: checks the
        rays and `operands` as _check_operands does and returns the leading
        arguments (ctx, table, S, rot0, dtype, N, y0, u0, clip) of the C call."""
        table = self._table(table)
        N = y0.shape[0] if N is None else int(N)
        _check_operands(y0.dtype, N, y0=(y0, 3), u0=(u0, 3), **operands)
        return (self.ctx, ptr(table), len(table), ptr(_rot0(rot0)), _code(y0.dtype), N, y0.ptr,
                u0.ptr, int(bool(clip)))

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
        if mask is None and path_sum is None and all(a is None for a in (Y, U, I, T)):
            raise ValueError("nothing to store: pass an output array, a mask or a path sum")
        args = self._march(table, y0, u0, N, clip, rot0)
        S, N = args[2], args[5]
        first = next((a for a in (Y, U, I, T) if a is not None), None)
        if ld is None:
            ld = first.shape[1] if first is not None else (N + 63)//64*64
        dp = lambda a: None if a is None else a.ptr  # noqa: E731
        _check_trace_operands(y0.dtype, N, 1 if keep_last else S, int(ld),
                              dict(Y=(Y, 3), U=(U, 3), I=(I, 3), T=(T, 1)), mask, path_sum)
        check(self.lib.rtx_set_mask_output(self.ctx, dp(mask)))
        check(self.lib.rtx_set_path_sum_output(self.ctx, dp(path_sum), int(path_sum_upto)))
        check(self.lib.rtx_trace(
            *args, RTX_KEEP_LAST if keep_last else RTX_KEEP_ALL, ld,
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
        check(self.lib.rtx_trace_batch(
            self.ctx, nb, C.cast(a_tab, vp), S, ptr(_rot0(rot0)), dt, C.cast(a_n, vp),
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
        check(self.lib.rtx_trace_host(
            self.ctx, ptr(table), len(table), ptr(_rot0(rot0)), dt, N, ptr(y0), ptr(u0),
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
        check(self.lib.rtx_trace_batch_host(
            self.ctx, nb, keep[0], S, ptr(_rot0(rot0)), _code(dtype),
            C.cast((C.c_int64*nb)(*Ns), vp), keep[1], keep[2], int(bool(clip)), RTX_KEEP_LAST if keep_last else RTX_KEEP_ALL,
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
        args = self._march(table, y0, u0, N, clip, rot0)
        N = args[5]
        _check_trace_operands(y0.dtype, N, 1, N, {}, mask, path_sum)
        dp = lambda a: None if a is None else a.ptr  # noqa: E731
        check(self.lib.rtx_set_mask_output(self.ctx, dp(mask)))
        check(self.lib.rtx_set_path_sum_output(self.ctx, dp(path_sum), int(path_sum_upto)))
        arr = (C.c_void_p*len(dst_ptrs))(*[C.c_void_p(int(p)) for p in dst_ptrs])
        arr_i = None
        if dst_i_ptrs is not None:
            if len(dst_i_ptrs) != len(dst_ptrs):
                raise ValueError("dst_i_ptrs must match dst_ptrs")
            arr_i = C.cast((C.c_void_p*len(dst_ptrs))(*[C.c_void_p(int(p)) for p in dst_i_ptrs]),
                           C.c_void_p)
        check(self.lib.rtx_trace_gather(
            *args, len(dst_ptrs), C.cast(arr, C.c_void_p), arr_i, int(dst_offset),
            self._flags(exact, False) | (_lib.RTX_GATHER_XY if xy else 0)))

    # ---- fused epilogues (no per-surface stores) -------------------------
    def trace_reduce(self, table, y0, u0, N=None, clip=False, rot0=None, exact=False, w=None,
                     center=None):
        """rtx_trace_reduce: march the DEVICE launch rays to the last surface
        of `table` and return the 20 rms / refocus moments of that surface
        (include/rtx.h) -- one launch, no intercept is stored.  `center`:
        (y_x, y_y, u_x, u_y) guess centres (e.g. the chief ray's)."""
        args = self._march(table, y0, u0, N, clip, rot0, w=(w, 1))
        c = None if center is None else np.ascontiguousarray(center, np.float64).reshape(4)
        m = np.zeros(20)
        check(self.lib.rtx_trace_reduce(
            *args, None if w is None else w.ptr, ptr(c), ptr(m), self._flags(exact, False)))
        return m

    @staticmethod
    def _many_args(tables, bundles, items):
        """the checked arguments trace_reduce_many, trace_otf_many,
        trace_opd_many and trace_zernike_many share:
        (tables, dtype, items, N, y0s, u0s, item tables, item bundles)"""
        tables = np.ascontiguousarray(tables, SURFACE_DTYPE)
        if tables.ndim != 2 or tables.shape[0] < 1 or tables.shape[1] < 1:
            raise ValueError("tables must be a non-empty (nt, S) record array")
        if not bundles:
            raise ValueError("no bundles")
        dtype = np.dtype(bundles[0][0].dtype)
        Ns = []
        for y0, u0, N in bundles:
            if np.dtype(y0.dtype) != dtype:
                raise ValueError("every bundle must be %s, got %s" % (dtype, np.dtype(y0.dtype)))
            N = y0.shape[0] if N is None else int(N)
            _check_operands(dtype, N, y0=(y0, 3), u0=(u0, 3))
            Ns.append(N)
        items = np.ascontiguousarray(items, np.int64).reshape(-1, 2)
        if len(items) < 1:
            raise ValueError("no items")
        if items.min() < 0 or items[:, 0].max() >= len(tables) or items[:, 1].max() >= len(bundles):
            raise ValueError("an item's table or bundle index is out of range")
        it = np.ascontiguousarray(items[:, 0], np.int32)
        ib = np.ascontiguousarray(items[:, 1], np.int32)
        N = np.ascontiguousarray(Ns, np.int64)
        y0s = (C.c_void_p*len(bundles))(*[b[0].ptr for b in bundles])
        u0s = (C.c_void_p*len(bundles))(*[b[1].ptr for b in bundles])
        return tables, dtype, items, N, y0s, u0s, it, ib

    def trace_reduce_many(self, tables, bundles, items, centers=None, clip=False, rot0=None,
                          exact=False):
        """rtx_trace_reduce_many: `tables` (nt, S) records, `bundles` a list
        of (y0, u0, N) DEVICE launch rays (N None: all rows), `items` (nitems,
        2) of (table, bundle) indices, `centers` (nitems, 4) guess centres or
        None.  Returns the (nitems, 20) moments of every item (w = 1) from one
        launch; each row's bits depend on its own item only."""
        tables, dtype, items, N, y0s, u0s, it, ib = self._many_args(tables, bundles, items)
        c = None
        if centers is not None:
            c = np.ascontiguousarray(centers, np.float64).reshape(len(items), 4)
        m = np.zeros((len(items), 20))
        check(self.lib.rtx_trace_reduce_many(
            self.ctx, len(tables), ptr(tables), tables.shape[1], ptr(_rot0(rot0)), _code(dtype),
            len(bundles), ptr(N), y0s, u0s, len(items), ptr(it), ptr(ib), ptr(c), int(bool(clip)),
            ptr(m), self._flags(exact, False)))
        return m

    def trace_otf_many(self, tables, bundles, items, centers=None, z=(0.,), freqs=(0.,),
                       clip=False, rot0=None, exact=False):
        """rtx_trace_otf_many: `tables`, `bundles` and `items` as
        trace_reduce_many, `centers` (nitems, 2) or None, the planes `z` (K,)
        and the frequencies `freqs` (F,) every item shares.  Returns the
        complex OTF sums (nitems, K, 2, F) (axis 0: x, 1: y) and the counts
        (nitems, K) int64 from one launch; each item's bits depend on its own
        item only."""
        tables, dtype, items, N, y0s, u0s, it, ib = self._many_args(tables, bundles, items)
        z = np.ascontiguousarray(np.atleast_1d(np.asarray(z, np.float64)))
        nu = np.ascontiguousarray(np.atleast_1d(np.asarray(freqs, np.float64)))
        K, F = len(z), len(nu)
        if z.ndim != 1 or not 1 <= K <= OTF_MAX_PLANES or not np.isfinite(z).all():
            raise ValueError("need 1..%d finite planes, got %r" % (OTF_MAX_PLANES, z))
        if nu.ndim != 1 or not 1 <= F <= OTF_MAX_FREQS or not np.isfinite(nu).all():
            raise ValueError("need 1..%d finite frequencies, got %r" % (OTF_MAX_FREQS, nu))
        c = None
        if centers is not None:
            c = np.ascontiguousarray(centers, np.float64).reshape(len(items), 2)
            if not np.isfinite(c).all():
                raise ValueError("centres must be finite")
        sums = np.zeros((len(items), K, 2, F, 2))
        count = np.zeros((len(items), K), np.int64)
        check(self.lib.rtx_trace_otf_many(
            self.ctx, len(tables), ptr(tables), tables.shape[1], ptr(_rot0(rot0)), _code(dtype),
            len(bundles), ptr(N), y0s, u0s, len(items), ptr(it), ptr(ib), ptr(c), int(bool(clip)),
            K, ptr(z), F, ptr(nu), ptr(sums), ptr(count), self._flags(exact, False)))
        return sums[..., 0] + 1j*sums[..., 1], count

    @staticmethod
    def _wfe_args(n, specs, a0, centers):
        """the checked per-item arguments trace_opd_many and
        trace_zernike_many share: (spec records, a0, centres)"""
        if isinstance(specs, np.ndarray) and specs.dtype == OPD_DTYPE:
            rec = np.ascontiguousarray(specs.reshape(-1))
        else:
            rec = np.concatenate([_opd_record(s) for s in specs]) if len(specs) else \
                np.zeros(0, OPD_DTYPE)
        if len(rec) != n:
            raise ValueError("need one spec per item: %d specs for %d items" % (len(rec), n))
        a = None if a0 is None else np.ascontiguousarray(a0, np.float64).reshape(n)
        c = None if centers is None else np.ascontiguousarray(centers, np.float64).reshape(n, 2)
        return rec, a, c

    def trace_opd_many(self, tables, bundles, items, specs, a0=None, centers=None, clip=False,
                       rot0=None, exact=False):
        """rtx_trace_opd_many: `tables` (nt, S) records of the march to
        `after` (trace_opd's), `bundles` and `items` as trace_reduce_many,
        `specs` one rtx_opd per item (a list of dicts with its members, or an
        OPD_DTYPE array), `a0` (nitems,) piston guesses and `centers`
        (nitems, 2) pupil centres, or None for 0.  Returns the (nitems, 10)
        sums n, sum a, sum a^2, sum x, sum y, sum x^2, sum xy, sum y^2,
        sum ax, sum ay of a = A - a0, (x, y) = P_xy - c over the rays whose
        a, x, y are finite, from one launch; FP64 only; each row's bits
        depend on its own item only."""
        tables, dtype, items, N, y0s, u0s, it, ib = self._many_args(tables, bundles, items)
        n = len(items)
        rec, a, c = self._wfe_args(n, specs, a0, centers)
        sums = np.zeros((n, WFE_NSUMS))
        check(self.lib.rtx_trace_opd_many(
            self.ctx, len(tables), ptr(tables), tables.shape[1], ptr(_rot0(rot0)), _code(dtype),
            len(bundles), ptr(N), y0s, u0s, n, ptr(it), ptr(ib), ptr(rec), ptr(a), ptr(c),
            int(bool(clip)), ptr(sums), self._flags(exact, False)))
        return sums

    def trace_zernike_many(self, tables, bundles, items, specs, rho, order, a0=None,
                           centers=None, clip=False, rot0=None, exact=False):
        """rtx_trace_zernike_many: trace_opd_many's arguments, the radial
        `order` (0..8) and `rho` (nitems,) each item's normalisation radius.
        Returns (sums (nitems, E), r2max (nitems,)): E = (J+1)(J+2)/2, J =
        (order+1)(order+2)/2, the upper triangle row-major of the Gram sums
        of (a, Z_1 .. Z_J) at (x, y)/rho (Noll's orthonormal Zernikes) over
        the rays whose a, x, y are finite, and the largest x^2 + y^2 of those
        rays; from one launch; FP64 only; each row's bits depend on its own
        item only."""
        tables, dtype, items, N, y0s, u0s, it, ib = self._many_args(tables, bundles, items)
        n = len(items)
        rec, a, c = self._wfe_args(n, specs, a0, centers)
        r = np.ascontiguousarray(rho, np.float64).reshape(n)
        J = (int(order) + 1)*(int(order) + 2)//2
        sums = np.zeros((n, (J + 1)*(J + 2)//2))
        r2max = np.zeros(n)
        check(self.lib.rtx_trace_zernike_many(
            self.ctx, len(tables), ptr(tables), tables.shape[1], ptr(_rot0(rot0)), _code(dtype),
            len(bundles), ptr(N), y0s, u0s, n, ptr(it), ptr(ib), ptr(rec), ptr(a), ptr(c),
            int(bool(clip)), int(order), ptr(r), ptr(sums), ptr(r2max), self._flags(exact, False)))
        return sums, r2max

    @staticmethod
    def rms_finite_from_moments(m):
        """rms about the mean of the rays whose image x, y are finite, from
        w = 1 moments: sqrt((m3 - (m1^2 + m2^2)/m0)/m0), written about the
        guess centre as rms_from_moments is (cancellation free when the
        centre lies within the spot).  Unlike GeometricTrace.rms it is not
        NaN when rays are lost; where none is, it equals
        rms_from_moments(m, unit_weights=True) bit for bit.  NaN when no ray
        is finite.  `m` (20,) or (..., 20): returns a float or an array."""
        m = np.asarray(m, np.float64)
        n = m[..., 0]
        with np.errstate(all="ignore"):
            bx, by = m[..., 1]/n, m[..., 2]/n
            r2 = m[..., 3] - 2*(bx*m[..., 1] + by*m[..., 2]) + (bx*bx + by*by)*n
            r = np.where(n > 0, np.sqrt(np.maximum(r2/n, 0.)), np.nan)
        return float(r) if r.ndim == 0 else r

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
        args = self._march(table, y0, u0, N, clip, rot0, A=(A, 1), P=(P, 3))
        check(self.lib.rtx_trace_opd(*args, ptr(_opd_record(spec)), A.ptr, P.ptr,
                                     self._flags(exact, False)))

    @staticmethod
    def _spot_outputs(spec, counts, extent):
        """the record, host tally / extent buffers and the counts pointer;
        ValueError for a counts array of another type or too small"""
        spec = np.ascontiguousarray(spec, SPOT_DTYPE).reshape(1)
        if counts is not None:
            if np.dtype(counts.dtype) != np.uint64:
                raise ValueError("counts must be uint64, got %s" % np.dtype(counts.dtype))
            need = int(np.prod(spot_shape(spec), dtype=np.int64))
            if 0 < need < 2**31 and counts.nbytes//8 < need:
                raise ValueError("counts holds %d bins but the spec needs %d"
                                 % (counts.nbytes//8, need))
        K = max(int(spec[0]["planes"]), 1)
        tally = np.zeros((K, 2), np.uint64)
        ext = np.zeros((K, 3)) if extent else None
        return spec, tally, ext, None if counts is None else counts.ptr

    def trace_spot(self, table, y0, u0, spec, counts=None, N=None, clip=False, rot0=None,
                   exact=False, extent=False):
        """rtx_trace_spot: march the DEVICE launch rays to the last surface of
        `table` and bin them at the planes of `spec` (spot_spec) into the
        uint64 DeviceArray `counts` (added to; None: extent only) -- one
        launch, nothing per ray is stored.  Returns (tally (K,2): binned,
        non-finite; extent (K,3): max |q_x|, |q_y|, r, or None)."""
        args = self._march(table, y0, u0, N, clip, rot0)
        spec, tally, ext, cp = self._spot_outputs(spec, counts, extent)
        check(self.lib.rtx_trace_spot(*args, ptr(spec), cp, ptr(tally), ptr(ext),
                                      self._flags(exact, False)))
        return tally, ext

    def spot_rows(self, y, inc, spec, counts=None, N=None, extent=False):
        """rtx_spot_rows: the binning of trace_spot on stored DEVICE rows
        y, inc (N,3) (a trace's y[at], i[at]).  Same returns."""
        N = y.shape[0] if N is None else int(N)
        _check_operands(y.dtype, N, y=(y, 3), inc=(inc, 3))
        spec, tally, ext, cp = self._spot_outputs(spec, counts, extent)
        check(self.lib.rtx_spot_rows(self.ctx, _code(y.dtype), N, y.ptr, inc.ptr, ptr(spec), cp,
                                     ptr(tally), ptr(ext)))
        return tally, ext

    otf_spec = staticmethod(otf_spec)

    def otf_rows(self, y, inc, spec, N=None):
        """rtx_otf_rows: the geometric OTF sums of stored DEVICE rows y, inc
        (N,3) (a trace's y[at], i[at]) at the planes and frequencies of
        `spec` (otf_spec).  Returns (S complex128 (K, 2, F): sum over the
        counted rays of exp(-2 pi i nu q) per plane, axis (x, y) and
        frequency; count int64 (K,): the rays with a finite point)."""
        N = y.shape[0] if N is None else int(N)
        _check_operands(y.dtype, N, y=(y, 3), inc=(inc, 3))
        spec = np.ascontiguousarray(spec, OTF_DTYPE).reshape(1)
        K, F = int(spec[0]["planes"]), int(spec[0]["nfreq"])
        sums = np.zeros((max(K, 1), 2, max(F, 1), 2))
        count = np.zeros(max(K, 1), np.int64)
        check(self.lib.rtx_otf_rows(self.ctx, _code(y.dtype), N, y.ptr, inc.ptr, ptr(spec),
                                    ptr(sums), ptr(count)))
        return sums[..., 0] + 1j*sums[..., 1], count

    pupil_spec = staticmethod(pupil_spec)

    def pupil_sum(self, A, P, spec, U, w=None, N=None):
        """rtx_pupil_sum: ADD the Debye sum U_k(a, b) of the DEVICE rays A
        (N,), P (N, 3) (rtx_trace_opd's outputs) with optional DEVICE weights
        w (N,) on the grid and planes of `spec` (pupil_spec) to the complex128
        DeviceArray U (K, nx, ny).  Returns (count, sum_w) of the rays summed."""
        N = A.shape[0] if N is None else int(N)
        _check_operands(np.float64, N, A=(A, 1), P=(P, 3), w=(w, 1))
        spec = np.ascontiguousarray(spec, PUPIL_DTYPE).reshape(1)
        s = spec[0]
        need = int(s["planes"])*int(s["nx"])*int(s["ny"])
        if np.dtype(U.dtype) != np.complex128 or U.nbytes//16 < need:
            raise ValueError("U must be a complex128 device array of %d values" % need)
        count, sumw = C.c_int64(), C.c_double()
        check(self.lib.rtx_pupil_sum(self.ctx, N, A.ptr, P.ptr, None if w is None else w.ptr,
                                     ptr(spec), U.ptr, C.byref(count), C.byref(sumw)))
        return int(count.value), float(sumw.value)

    def pupil_intensity(self, spec, U, psf, scale=1.0):
        """rtx_pupil_intensity: ADD scale |U|^2 of the complex128 DeviceArray
        U (K, nx, ny) to the float64 DeviceArray psf (K, nx, ny).  Returns the
        stats (K, 5) of psf after the addition: sum, max, flat index of the
        first max, sum psf p, sum psf q."""
        spec = np.ascontiguousarray(spec, PUPIL_DTYPE).reshape(1)
        s = spec[0]
        K, need = int(s["planes"]), int(s["planes"])*int(s["nx"])*int(s["ny"])
        if np.dtype(U.dtype) != np.complex128 or U.nbytes//16 < need:
            raise ValueError("U must be a complex128 device array of %d values" % need)
        if np.dtype(psf.dtype) != np.float64 or psf.nbytes//8 < need:
            raise ValueError("psf must be a float64 device array of %d values" % need)
        stats = np.zeros((max(K, 1), 5))
        check(self.lib.rtx_pupil_intensity(self.ctx, ptr(spec), U.ptr, float(scale), psf.ptr,
                                           ptr(stats)))
        return stats

    # ---- lens-parameter derivatives --------------------------------------
    def trace_jacobian(self, table, y0, u0, moves, clip=False, rot0=None, exact=False, N=None):
        """rtx_trace_jacobian: the image point q of every DEVICE launch ray at
        the last surface of `table` and its derivatives with respect to P
        parameters.  `moves`: P lists of (row, record), each record the
        derivative of table[row] (tolerance.record_tangents of this 1-D
        table, or one wavelength's records of a (W, S) table's).  Returns (q
        (N, 2), J (P, 2, ld)) DeviceArrays, ld = N rounded up to 32 rays;
        asynchronous.  q is the last row trace_device stores, bit for bit."""
        args = self._march(table, y0, u0, N, clip, rot0)
        N = args[5]
        P, first, rows, recs = _moves(y0, moves, args[2])
        ld = max(32, -(-N//32)*32)
        q, J = self.empty((N, 2)), self.empty((P, 2, ld))
        check(self.lib.rtx_trace_jacobian(*args, P, ptr(first), ptr(rows), ptr(recs), q.ptr,
                                          J.ptr, ld, self._flags(exact, False)))
        return q, J

    def jacobian_sums(self, q, J, center=None, N=None):
        """rtx_jacobian_sums of trace_jacobian's DEVICE q (N, 2) and J (P, 2,
        ld) about `center` (2,): a dict of n, sum_d (2,), sum_d2, G (P, 2),
        H (P,), K (P, P) (symmetric), bad (rays with a finite q and a
        non-finite derivative) and the raw output row `out`."""
        P, _, ld = J.shape
        N = q.shape[0] if N is None else int(N)
        _check_operands(q.dtype, N, q=(q, 2))
        if np.dtype(J.dtype) != np.float64 or N > ld:
            raise ValueError("J must be float64 (P, 2, ld) with ld >= N")
        c = None if center is None else np.ascontiguousarray(center, np.float64).reshape(2)
        W = 5 + 3*P + P*(P + 1)//2
        out = np.zeros(W)
        check(self.lib.rtx_jacobian_sums(self.ctx, N, P, q.ptr, J.ptr, ld, ptr(c), ptr(out)))
        return jacobian_sums_unpack(out, P)

    def trace_opd_jacobian(self, table, y0, u0, spec, moves, dopd, clip=False, rot0=None,
                           exact=False, N=None):
        """rtx_trace_opd_jacobian: trace_opd's path A of every DEVICE launch
        ray (`table` = system[1:after+1], `spec` as trace_opd's) and its
        derivatives with respect to P parameters.  `moves` as
        trace_jacobian's, on the rows of `table`; `dopd` (P, 4) the
        derivatives of spec's d and n_after.  Returns (A (N,), dA (P, ld))
        DeviceArrays, ld = N rounded up to 32 rays; asynchronous.  A is
        trace_opd's, bit for bit."""
        args = self._march(table, y0, u0, N, clip, rot0)
        N = args[5]
        P, first, rows, recs = _moves(y0, moves, args[2])
        dopd = np.ascontiguousarray(dopd, np.float64)
        if dopd.shape != (P, 4):
            raise ValueError("dopd must be (%d, 4), got %s" % (P, dopd.shape))
        ld = max(32, -(-N//32)*32)
        A, dA = self.empty((N,)), self.empty((P, ld))
        check(self.lib.rtx_trace_opd_jacobian(*args, ptr(_opd_record(spec)), P, ptr(first),
                                              ptr(rows), ptr(recs), ptr(dopd), A.ptr, dA.ptr, ld,
                                              self._flags(exact, False)))
        return A, dA

    def wavefront_sums(self, A, dA, a0=0., N=None):
        """rtx_wavefront_sums of trace_opd_jacobian's DEVICE A (N,) and dA
        (P, ld) (None: P = 0, the sums of A alone) about the piston `a0`: a
        dict of n, sum_d, sum_d2, G (P,), H (P,), K (P, P) (symmetric), bad
        and the raw output row `out`."""
        N = A.shape[0] if N is None else int(N)
        _check_operands(A.dtype, N, A=(A, 1))
        P, ld = (0, max(N, 1)) if dA is None else dA.shape
        if np.dtype(A.dtype) != np.float64 or (dA is not None and np.dtype(dA.dtype) != np.float64) \
                or N > ld:
            raise ValueError("A must be float64 (N,) and dA float64 (P, ld) with ld >= N")
        out = np.zeros(4 + 2*P + P*(P + 1)//2)
        check(self.lib.rtx_wavefront_sums(self.ctx, N, P, A.ptr, None if dA is None else dA.ptr,
                                          ld, float(a0), ptr(out)))
        return wavefront_sums_unpack(out, P)

    def otf_jacobian_sums(self, q, J, freqs, center=None, N=None):
        """rtx_otf_jacobian_sums: the geometric OTF sums of DEVICE image points
        q at the frequencies `freqs` (F,) about `center` (2,) and their
        derivatives from J (trace_jacobian's (P, 2, ld); None: P = 0).  q is
        (N, 2) (trace_jacobian's) or (N, 3) (a keep-LAST row of
        trace_device; its x, y are read).  Returns a
        dict of n, bad (rays with a finite q and a non-finite derivative), S
        complex (2, F), dS complex (P, 2, F) and the raw output row `out`."""
        N = q.shape[0] if N is None else int(N)
        qs = q.shape[-1] if len(q.shape) >= 2 else 0
        if np.dtype(q.dtype) != np.float64 or qs not in (2, 3):
            raise ValueError("q must be float64 (N, 2) or (N, 3), got %s %s"
                             % (np.dtype(q.dtype), q.shape))
        _check_operands(q.dtype, N, q=(q, qs))
        P, ld = (0, max(N, 1)) if J is None else (J.shape[0], J.shape[-1])
        if J is not None and (np.dtype(J.dtype) != np.float64 or len(J.shape) != 3
                              or J.shape[1] != 2 or N > ld):
            raise ValueError("J must be float64 (P, 2, ld) with ld >= N")
        freqs = np.ascontiguousarray(np.atleast_1d(freqs), np.float64)
        F = len(freqs)
        if freqs.ndim != 1 or not 1 <= F <= OTF_MAX_FREQS or not np.isfinite(freqs).all():
            raise ValueError("need 1..%d finite frequencies, got %r" % (OTF_MAX_FREQS, freqs))
        c = None if center is None else np.ascontiguousarray(center, np.float64).reshape(2)
        out = np.zeros(2 + 4*F + 4*P*F)
        check(self.lib.rtx_otf_jacobian_sums(self.ctx, N, P, q.ptr, qs,
                                             None if J is None else J.ptr, ld, ptr(c), F,
                                             ptr(freqs), ptr(out)))
        return otf_jacobian_sums_unpack(out, P, F)

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
        `points` and `values` may be DeviceArrays, used in place too.
        Returns the (n, n) values -- numpy, or a DeviceArray when not
        `download` -- and with `winner` also the covering simplex per node
        (numpy int32, -1 where none covers it, like find_simplex)."""
        dev_points = isinstance(points, DeviceArray)
        dev_values = isinstance(values, DeviceArray)
        if not dev_points:
            points = np.ascontiguousarray(points, np.float64)
        if not dev_values:
            values = np.ascontiguousarray(values, np.float64)
        gh = np.ascontiguousarray(gh, np.float64)
        if len(points.shape) != 2 or points.shape[1] != 2 or values.shape != points.shape[:1] \
                or np.dtype(points.dtype) != np.float64 or np.dtype(values.dtype) != np.float64:
            raise ValueError("points must be (M, 2) FP64 and values (M,)")
        if gh.shape != (int(n),):
            raise ValueError("gh must be the (n,) grid axis")
        step = np.diff(gh)
        if not np.isfinite(gh).all() or not ((step > 0).all() or (step < 0).all()):
            raise ValueError("gh must be finite and strictly monotone")
        n = int(n)
        ins = [values if dev_values else self.to_device(values), self.to_device(gh)]
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
            for a in ins[1:] if dev_values else ins:
                a.free()
        return (out, w) if winner else out

    def opd_points(self, A, P, ref, k):
        """rtx_opd_points: the finite exit-pupil points of rtx_trace_opd's
        DEVICE outputs A (N,), P (N,3) relative to ray `ref`, compacted in
        ray order, with t = -(A - A[ref])/k, k = l/scale.  Returns (pts
        DeviceArray (M, 2), vals DeviceArray (M,), M, h = max |x|, |y|); the
        arrays hold room for N rays, free them when done."""
        N = int(A.shape[0])
        if A.dtype != np.float64 or P.dtype != np.float64 or P.shape[:1] != (N,) or \
                len(P.shape) != 2 or P.shape[1] != 3:
            raise ValueError("A must be (N,) and P (N, 3) FP64 device arrays")
        pts, vals = self.empty((max(N, 1), 2)), self.empty((max(N, 1),))
        M, h = C.c_int64(), C.c_double()
        try:
            check(self.lib.rtx_opd_points(self.ctx, RTX_F64, N, A.ptr, P.ptr, int(ref), float(k),
                                          pts.ptr, vals.ptr, C.byref(M), C.byref(h)))
        except Exception:
            pts.free()
            vals.free()
            raise
        M = int(M.value)
        for a in (pts, vals):               # M rows of the N-ray allocation
            a.shape = (M,) + a.shape[1:]
            a.nbytes = M*a.nbytes//max(N, 1)
        return pts, vals, M, float(h.value)

    def grid_range(self, o):
        """rtx_grid_range of a DEVICE FP64 array: (finite count, min, max)
        over its finite values, NaN min and max when there are none"""
        if o.dtype != np.float64:
            raise ValueError("o must be an FP64 device array")
        count, lo, hi = C.c_int64(), C.c_double(), C.c_double()
        check(self.lib.rtx_grid_range(self.ctx, RTX_F64, int(np.prod(o.shape)), o.ptr,
                                      C.byref(count), C.byref(lo), C.byref(hi)))
        return int(count.value), float(lo.value), float(hi.value)

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
