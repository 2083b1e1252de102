"""Device-resident trace results with lazy host materialisation.

The full trace of 1e7 rays x 12 surfaces is 10 GB; PCIe moves it in 0.2 s while
the kernel needs 1.7 ms.  The consumers of ``GeometricTrace`` mostly read single
rows -- spot diagrams ``y[-1]``, ``i[-1]`` (rayopt/analysis.py:269-280), fans
``y[-1]``, ``y[0]``, ``u[0]`` (:231-245), ``rms`` ``y[i]``
(rayopt/geometric_trace.py:171-183), ``refocus`` ``y[at]``, ``i[at]`` (:82-99)
-- so the resident drop-in keeps ``y,u,i,t`` in HBM and hands out ``LazyRows``
objects that copy a surface row to the host the first time it is indexed (and
the whole array only for ``np.asarray``).

``ResidentMixin`` is the resident flavour of ``PropagateMixin``
(geometric_trace.py): ``bind(rayopt.GeometricTrace, resident=True)`` puts it in
front of the reference class; ``ResidentTrace`` is the standalone class with the
on-device ray generation on top.
"""
import numpy as np

from .engine import default_engine
from .surface_table import pack_system

# rows above this size live in page-locked host buffers (full-rate PCIe)
PINNED_ROW_BYTES = 1 << 20


def opd_spec(system, track, origins, after, image, n0, n_after, y0_ref, u0_ref, y_img_ref,
             radius=None):
    """The `rtx_opd` record of GeometricTrace.opd (rayopt/geometric_trace.py:
    101-131) for surfaces `after` and `image` (indices >= 0): the default
    reference-sphere radius (:110-114, the image pupil's distance, or the
    track between the surfaces for a telecentric pupil), the frame change
    between the surfaces (their rotations and origins) and the reference
    ray's launch ray (y0_ref, u0_ref) and image intercept y_img_ref."""
    s = system
    if radius is None:                                  # :110-114
        if s.image.pupil.telecentric:
            radius = track[image] - track[after]
        else:
            radius = -s.image.pupil.distance
    ea, ei = s[after], s[image]
    eye = np.eye(3)
    Ra = np.asarray(ea.rot_normal, float) if getattr(ea, "rotated", False) else eye
    Ri = np.asarray(ei.rot_normal, float) if getattr(ei, "rotated", False) else eye
    return dict(y0_ref=y0_ref, u0_ref=u0_ref, n0=n0, n_after=n_after, M=Ra @ Ri.T,
                d=(origins[after] - origins[image]) @ Ri.T - y_img_ref,
                radius=radius, infinite=not s.object.finite)


def check_triangulation(triangulation):
    if triangulation not in ("host", "device"):
        raise ValueError("triangulation must be 'host' or 'device', got %r" % (triangulation,))


def regrid(eng, pts, vals, M, h, n, download, triangulation):
    """GeometricTrace.opd's regridding (rayopt/geometric_trace.py:136-143) of
    the M compacted exit-pupil points `pts`, `vals` (Engine.opd_points; freed
    here) on the (n, n) grid of half-width h: Delaunay on the host (the
    points downloaded) or on the device, then rtx_grid_linear.  Returns
    (xs, ys, o) with o numpy, or a DeviceArray when not `download`.
    ValueError when no ray made it through."""
    try:
        if not M:
            raise ValueError("no rays made it through")
        xs, ys = np.mgrid[-1:1:1j*n, -1:1:1j*n]*h
        if triangulation == "host":
            from scipy.spatial import Delaunay
            p, v = pts.download(), vals.download()
            return xs, ys, eng.grid_linear(p, v, Delaunay(p), n, xs[:, 0].copy(),
                                           download=download)
        tri = eng.delaunay(pts)
        try:
            return xs, ys, eng.grid_linear(pts, vals, tri, n, xs[:, 0].copy(), download=download)
        finally:
            tri.free()
    finally:
        pts.free()
        vals.free()


def psf_of_grid(eng, xs, o, pad, wl, radius):
    """GeometricTrace.psf (rayopt/geometric_trace.py:150-161) of the
    regridded OPD `o` (DEVICE (n, n), freed here) on the grid `xs`: rtx_psf
    and the frequency axes for the wavelength wl = l/scale in lens units and
    the sphere's radius.  Returns (p, q, psf DeviceArray, stats)."""
    try:
        out, raw = eng.psf(o, pad)
    finally:
        o.free()
    nx = pad*xs.shape[0]
    dx = xs[1, 0] - xs[0, 0]
    k = 1/wl
    f = np.fft.fftfreq(nx, dx*k/radius)
    p, q = np.broadcast_arrays(f[:, None], f)
    return p, q, out, eng.psf_stats(raw, f)


def psf_profiles(eng, p, out, st):
    """The encircled energy and MTF Analysis.opds (rayopt/analysis.py:
    319-346) takes of the DEVICE PSF `out` (freed here) on the axis `p`,
    with its device stats `st` (ResidentMixin.psf_profiles)"""
    try:
        x0, y0 = st["cp"], st["cq"]
        xs = np.fft.fftshift(p[:, 0])
        dx = (xs[1] - x0) - (xs[0] - x0)
        nx, ny = out.shape
        center = (nx/2 + x0/dx, ny/2 + y0/dx)
        bins, lsf0, lsf1 = eng.psf_profiles(out, center)
    finally:
        out.free()
    size = nx*ny
    mtf = []
    for lsf in (lsf0, lsf1):
        ot = np.fft.ifft(lsf*size**.5)
        mtf.append(np.absolute(ot[:ot.size//2]))
    of = np.fft.fftfreq(lsf0.size, dx)[:lsf0.size//2]
    ee = np.cumsum(bins)
    return dict(stats=st, x0=x0, y0=y0, dx=dx, center=center, xe=np.arange(ee.size)*dx,
                ee=ee, of=of, mtf=tuple(mtf))


class LazyRows:
    """numpy-like view of a device array (rows, ld, k...) restricted to the
    first `n` columns.  Indexing with a leading integer (or a slice of rows)
    downloads just those rows, once; like ``GeometricTrace.y[j]`` in the
    reference the result is a VIEW of the trace's storage: the host buffer of
    a row is reused, so a later ``propagate`` + access refreshes it in place.
    Item assignment writes through to the device."""

    def __init__(self, darray, n, dtype=np.float64):
        self._d = darray
        self._n = int(n)
        self.dtype = np.dtype(dtype)
        self.shape = (darray.shape[0], self._n) + tuple(darray.shape[2:])
        self.ndim = len(self.shape)
        self.size = int(np.prod(self.shape))
        self._rows = {}        # valid host copies
        self._bufs = {}        # host buffers (kept across invalidation)
        self.fetched_bytes = 0

    def __len__(self):
        return self.shape[0]

    def invalidate(self, rows=None):
        if rows is None:
            self._rows.clear()
        else:
            for r in rows:
                self._rows.pop(r, None)

    def _buffer(self, r):
        b = self._bufs.get(r)
        if b is None:
            shape = (self._n,) + self.shape[2:]
            nbytes = int(np.prod(shape))*self._d.dtype.itemsize
            eng = getattr(self._d, "engine", None)
            if nbytes >= PINNED_ROW_BYTES and hasattr(eng, "pinned_empty"):
                b = eng.pinned_empty(shape, self._d.dtype)
            else:
                b = np.empty(shape, self._d.dtype)
            self._bufs[r] = b
        return b

    def set_row(self, r, value):
        """host-side write of one row (e.g. launch rays), mirrored to the
        device; `value` broadcasts to (n, k) or to the padded (ld, k) row"""
        r = range(self.shape[0])[r]
        drow = self._d.rows(r)
        v = np.asarray(value)
        full = drow.shape[1:]
        if v.shape == full:                              # whole padded row
            v = np.ascontiguousarray(v, self._d.dtype)
            drow.upload(v)
            host = v[:self._n]
        else:
            host = np.ascontiguousarray(np.broadcast_to(v, (self._n,) + self.shape[2:]),
                                        self._d.dtype)
            drow.upload(host)                            # the first n columns are contiguous
        b = self._buffer(r)
        b[...] = host
        self._rows[r] = b if b.dtype == self.dtype else b.astype(self.dtype)

    def row(self, r):
        r = range(self.shape[0])[r]
        a = self._rows.get(r)
        if a is None:
            b = self._buffer(r)
            self._d.rows(r).download(out=b)              # first n columns of the row
            a = b if b.dtype == self.dtype else b.astype(self.dtype)
            self._rows[r] = a
            self.fetched_bytes += b.nbytes
        return a

    def __getitem__(self, idx):
        if not isinstance(idx, tuple):
            idx = (idx,)
        head, rest = idx[0], idx[1:]
        if isinstance(head, (int, np.integer)):
            a = self.row(int(head))
            return a[rest] if rest else a
        if isinstance(head, slice):
            rows = range(self.shape[0])[head]
            a = np.stack([self.row(r) for r in rows]) if len(rows) else \
                np.empty((0,) + self.shape[1:], self.dtype)
            return a[(slice(None),) + rest] if rest else a
        return np.asarray(self)[idx]

    def __setitem__(self, idx, value):
        if not isinstance(idx, tuple):
            idx = (idx,)
        head, rest = idx[0], idx[1:]
        rows = [range(self.shape[0])[int(head)]] if isinstance(head, (int, np.integer)) \
            else list(range(self.shape[0])[head])
        value = np.asarray(value)
        for k, r in enumerate(rows):
            v = value if isinstance(head, (int, np.integer)) or value.ndim < self.ndim else value[k]
            if rest:
                host = np.array(self.row(r))
                host[rest] = v
            else:
                host = v
            self.set_row(r, host)

    def __array__(self, dtype=None, copy=None):
        a = np.stack([self.row(r) for r in range(self.shape[0])])
        return a if dtype is None else a.astype(dtype)


class ResidentMixin:
    """``allocate / rays_given / propagate / rms / refocus`` of GeometricTrace
    (rayopt/geometric_trace.py:37-99,171-183) with the results resident in HBM.
    Same signatures and attribute names; ``y, u, i, t`` are ``LazyRows``.
    ``propagate`` moves no ray data over PCIe; ``rms`` and ``refocus`` reduce on
    the device (8 doubles come back)."""

    engine = None
    exact = False
    resident = True

    # the reference's default weights ones(N)/N (geometric_trace.py:57-58) are
    # materialised on first read: at 1e7 rays building them costs more than the
    # trace, and the device reductions never need them (w = None means 1/N)
    @property
    def w(self):
        if self._w is None and getattr(self, "_w_default", False):
            self._w = np.ones(self.nrays)/self.nrays
        return self._w

    @w.setter
    def w(self, value):
        self._w = value
        self._w_default = False
    _w = None
    # i[j] == u[j-1] bit for bit in unrotated systems (system.py:461-463): u and
    # i are then two row-shifted views of ONE (S+2, ld, 3) device buffer and the
    # kernel stores 56 instead of 80 bytes per ray-surface
    alias_incidence = True
    _dev = None

    def _engine(self):
        if self.engine is None:
            self.engine = default_engine()
        return self.engine

    # ---- a1
    def allocate(self, nrays):
        eng = self._engine()
        self.free()
        self.length = L = len(self.system)
        self.nrays = nrays
        self._ld = ld = (nrays + 63)//64*64
        d = {"y": eng.empty((L, ld, 3)), "t": eng.empty((L, ld))}
        if self.alias_incidence:
            d["uext"] = eng.empty((L + 1, ld, 3))
            d["u"], d["i"] = d["uext"].rows(1, L + 1), d["uext"].rows(0, L)
            self._i_alias = True
        else:
            d["u"], d["i"] = eng.empty((L, ld, 3)), eng.empty((L, ld, 3))
            self._i_alias = False
        self._dev = d
        self._wrap()
        self.n = np.empty(L)
        self.w = None
        self.ref = None
        self.l = 1.
        self._w_dev = None

    def _wrap(self):
        d, n = self._dev, self.nrays
        self.y, self.u = LazyRows(d["y"], n), LazyRows(d["u"], n)
        self.i, self.t = LazyRows(d["i"], n), LazyRows(d["t"], n)

    def _materialize_i(self):
        """a rotated element breaks i[j] == u[j-1]: give `i` its own array"""
        eng, d = self._engine(), self._dev
        own = eng.empty((self.length, self._ld, 3))
        own.copy_from(d["i"])
        eng.sync()
        d["i"] = own
        self._i_alias = False
        self.i = LazyRows(own, self.nrays)

    def free(self):
        """give the HBM back now (otherwise: when the object is collected)"""
        if self._dev:
            for a in self._dev.values():
                a.free()
        self._dev = None
        w = getattr(self, "_w_dev", None)
        if w is not None:
            w[1].free()
        self._w_dev = None

    # ---- a2
    def rays_given(self, y, u, l=None, w=None, ref=0):
        """rayopt/geometric_trace.py:49-70: launch rays into row 0 -- straight
        from the caller's arrays into HBM (one H2D per array when they are
        (N,3) float64; page-locked arrays copy at full PCIe rate)."""
        pos, dirn = np.broadcast_arrays(*np.atleast_2d(y, u))
        count, width = pos.shape
        if self._dev is None or self.nrays != count:
            self.allocate(count)
        self.l = self.system.wavelengths[0] if l is None else l
        self.w = w
        self._w_default = w is None
        self._w_dev = None
        self.ref = ref
        if width != 3:
            y0 = np.zeros((count, 3))
            u0 = np.zeros((count, 3))
            y0[:, :width] = pos
            u0[:, :width] = dirn
            if width < 3:                                  # assumes forward rays, :65-67
                u0[:, 2] = np.sqrt(1 - np.square(u0[:, :2]).sum(-1))
            pos, dirn = y0, u0
        d = self._dev
        d["y"].rows(0).upload(pos)
        d["u"].rows(0).upload(dirn)
        d["i"].rows(0).copy_from(d["u"].rows(0), count*24)     # i[0] = u[0], :68
        self._zero_t0()                                        # t[0] = 0, :70
        for a in (self.y, self.u, self.i, self.t):
            a.invalidate()
        self.n[0] = self.system.refractive_index(self.l, 0)

    def _zero_t0(self):
        eng, row = self._engine(), self._dev["t"].rows(0)
        if hasattr(eng, "memset"):
            eng.memset(row, 0)
        else:
            row.upload(np.zeros(row.shape[1:]))

    def _cache_system(self):
        """Trace.propagate, rayopt/raytrace.py:32-36"""
        for name in ("path", "track", "origins", "mirrored"):
            try:
                setattr(self, name, getattr(self.system, name))
            except AttributeError:
                pass

    # ---- a3
    def propagate(self, start=1, stop=None, clip=False):
        """rayopt/geometric_trace.py:72-80 on the resident rows"""
        self._cache_system()
        init = start - 1
        table, n, rot0 = pack_system(self.system, self.l, start, stop, n0=self.n[init])
        rows = len(table)
        if rows == 0:
            return
        if self._i_alias and (rot0 is not None or (table["flags"] & 1).any()):
            self._materialize_i()
        d = self._dev
        sl = (start, start + rows)
        self._engine().trace_device(
            table, d["y"].rows(init), d["u"].rows(init),
            d["y"].rows(*sl), d["u"].rows(*sl),
            None if self._i_alias else d["i"].rows(*sl), d["t"].rows(*sl),
            N=self.nrays, ld=self._ld, clip=clip, rot0=rot0, exact=self.exact)
        self.n[start:start + rows] = n
        self._last_clip = bool(clip)
        touched = range(start, start + rows)
        for a in (self.y, self.u, self.t):
            a.invalidate(touched)
        # an aliased i[j] is u[j-1]: rows start+1 .. start+rows changed
        self.i.invalidate(range(start + 1, start + rows + 1) if self._i_alias else touched)

    # ---- reductions that never bring the rays to the host (SURVEY 8f-1)
    def _weights(self):
        """device copy of self.w, or None for the default 1/N weights"""
        if self._w is None or getattr(self, "_w_default", False):
            return None
        if self._w_dev is None or self._w_dev[0] is not self._w:
            if self._w_dev is not None:
                self._w_dev[1].free()
            self._w_dev = (self._w, self._engine().to_device(np.asarray(self._w, float)))
        return self._w_dev[1]

    def rms(self, i=-1, ref=None):
        """GeometricTrace.rms (rayopt/geometric_trace.py:171-183) on the
        resident intercepts (moment passes on the device, 64 bytes back)."""
        eng = self._engine()
        i = range(self.length)[i]
        ref_point = None if ref is None else \
            eng.download_rays(self._dev["y"].rows(i), [int(ref)])[0, :2]    # 24 bytes, not the row
        return eng.rms(self._dev["y"].rows(i), self._weights(), N=self.nrays,
                       ref_point=ref_point)

    def refocus(self, at=-1):
        """GeometricTrace.refocus (rayopt/geometric_trace.py:82-99): the
        least-squares focus shift from device moments of y[at], i[at]
        (rtx_focus_moments), then the re-trace."""
        eng = self._engine()
        at = range(self.length)[at]
        shift = eng.refocus_shift(self._dev["y"].rows(at), self._dev["i"].rows(at),
                                  self._weights(), N=self.nrays)
        self.system[at].distance += shift
        self.propagate()


    # ---- fused epilogues: the march itself reduces (no rows are stored or read)
    def _chief(self, table, rot0, clip):
        """(y_x, y_y, u_x, u_y) of the `ref` ray at the last surface of `table`
        (a 1-ray trace through the small-bundle path); NaN if it dies"""
        eng, d = self._engine(), self._dev
        ref = 0 if self.ref is None else int(self.ref)
        y0 = eng.download_rays(d["y"].rows(0), [ref])
        u0 = eng.download_rays(d["u"].rows(0), [ref])
        Y, _, I, _ = eng.trace(table, y0, u0, clip=clip, rot0=rot0, keep_last=True,
                               exact=self.exact, want=("y", "i"))
        with np.errstate(all="ignore"):
            return np.r_[Y[0, 0, :2], I[0, 0, :2]/I[0, 0, 2]].astype(np.float64)

    def _guess_center(self, table, rot0, clip):
        """the chief ray's (y_x, y_y, u_x, u_y), zeros if it dies"""
        c = self._chief(table, rot0, clip)
        return c if np.all(np.isfinite(c)) else np.zeros(4)

    def reduce(self, at=-1, clip=False):
        """ONE launch from the launch rays (row 0) to surface `at`: the trace
        kernel accumulates the rms / refocus moments of that surface in
        registers (rtx_trace_reduce) and stores nothing else.  Returns the 20
        moments (include/rtx.h) and the guess centre they refer to."""
        at = range(self.length)[at]
        table, _, rot0 = pack_system(self.system, self.l, 1, at + 1, n0=self.n[0])
        c = self._guess_center(table, rot0, clip)
        d = self._dev
        m = self._engine().trace_reduce(table, d["y"].rows(0), d["u"].rows(0), N=self.nrays,
                                        clip=clip, rot0=rot0, exact=self.exact,
                                        w=self._weights(), center=c)
        return m, c

    def rms_fused(self, at=-1, clip=False):
        """GeometricTrace.rms of surface `at` without a stored trace"""
        m, _ = self.reduce(at, clip)
        return self._engine().rms_from_moments(m, unit_weights=self._weights() is None)

    def refocus_fused(self, at=-1, clip=False):
        """GeometricTrace.refocus (geometric_trace.py:82-99) from one fused
        launch: the focus shift is applied to ``system[at].distance`` and
        returned; nothing is re-traced"""
        m, _ = self.reduce(at, clip)
        shift = self._engine().focus_shift_from_moments(m)
        self.system[at].distance += shift
        return shift

    def _trace_opd(self, radius, after, image):
        """rtx_trace_opd from row 0 to surface `after`: DEVICE A (N,), P (N,3)
        (free them when done).  Needs a propagated trace (the sphere is
        centred on ``y[image, ref]``)."""
        eng, s, d = self._engine(), self.system, self._dev
        after, image = range(self.length)[after], range(self.length)[image]
        ref = int(self.ref)
        spec = opd_spec(s, self.track, self.origins, after, image, self.n[0], self.n[after],
                        eng.download_rays(d["y"].rows(0), [ref])[0],
                        eng.download_rays(d["u"].rows(0), [ref])[0],
                        eng.download_rays(d["y"].rows(image), [ref])[0], radius)
        table, _, rot0 = pack_system(s, self.l, 1, after + 1, n0=self.n[0])
        A, P = eng.empty((self.nrays,)), eng.empty((self.nrays, 3))
        eng.trace_opd(table, d["y"].rows(0), d["u"].rows(0), spec, A, P, N=self.nrays,
                      clip=getattr(self, "_last_clip", False), rot0=rot0, exact=self.exact)
        return A, P

    def opd_rays(self, radius=None, after=-2, image=-1):
        """per-ray part of GeometricTrace.opd (rayopt/geometric_trace.py:
        101-131) as the epilogue of a march from row 0 to surface `after`
        (rtx_trace_opd); the reference ray's terms are subtracted here.
        Returns (x, y, t): exit-pupil coordinates and the OPD in waves -- what
        ``opd(resample=False)`` returns in the reference.  Needs a propagated
        trace (the sphere is centred on ``y[image, ref]``)."""
        A, P = self._trace_opd(radius, after, image)
        a, p = A.download(), P.download()
        A.free()
        P.free()
        ref = int(self.ref)
        t = -(a - a[ref])/(self.l/self.system.scale)        # :125-126
        p -= p[ref]                                         # :131
        return p[:, 0], p[:, 1], t

    def opd(self, radius=None, after=-2, image=-1, resample=4):
        """GeometricTrace.opd with the per-ray part on the device; the
        regridding (scipy griddata, geometric_trace.py:133-144) stays on the host"""
        x, y, t = self.opd_rays(radius, after, image)
        if resample:
            from scipy.interpolate import griddata
            ok = np.isfinite(x) & np.isfinite(y) & np.isfinite(t)
            x, y, t = x[ok], y[ok], t[ok]
            if not t.size:
                raise ValueError("no rays made it through")
            n = int(resample*self.nrays**.5)
            h = np.fabs((x, y)).max()
            xs, ys = np.mgrid[-1:1:1j*n, -1:1:1j*n]*h
            t = griddata((x, y), t, (xs, ys), method="linear", fill_value=np.nan)
            x, y = xs, ys
        return x, y, t

    # ---- diffraction PSF with the regridding and the FFT on the device
    def _opd_grid(self, radius, after, image, resample, download, triangulation="host"):
        """opd's regridding on the device: the per-ray OPD (rtx_trace_opd)
        and its finite exit-pupil points (rtx_opd_points) stay in HBM; they
        are triangulated on the host (scipy.spatial.Delaunay of the M
        downloaded points, griddata's own options) or, with
        ``triangulation="device"``, in HBM (rtx_delaunay); rtx_grid_linear
        interpolates on the reference's grid"""
        check_triangulation(triangulation)
        eng = self._engine()
        A, P = self._trace_opd(radius, after, image)
        try:
            pts = eng.opd_points(A, P, int(self.ref), self.l/self.system.scale)
        finally:
            A.free()
            P.free()
        return regrid(eng, *pts, int(resample*self.nrays**.5), download, triangulation)

    def opd_device(self, radius=None, after=-2, image=-1, resample=4, triangulation="host"):
        """``opd`` (rayopt/geometric_trace.py:101-144) with the regridding on
        the device (rtx_grid_linear on the host's Delaunay triangulation, or
        with ``triangulation="device"`` on rtx_delaunay's): griddata's values
        bit for bit wherever the device picks the simplex scipy's find_simplex
        picks; nodes on shared edges may take the neighbour's value (equal to
        rounding)"""
        if not resample:
            return self.opd_rays(radius, after, image)
        return self._opd_grid(radius, after, image, resample, download=True,
                              triangulation=triangulation)

    def psf_device(self, pad=4, resample=4, download=True, triangulation="host", **kwargs):
        """``psf`` (rayopt/geometric_trace.py:146-169) on the device: the
        regridded OPD stays in HBM, the pupil function, the padded FFT
        (cuFFT) and |.|^2 run there (rtx_psf).  Returns (p, q, psf) like the
        reference; with ``download=False`` psf is a DeviceArray (free it when
        done) and ``self.psf_stats`` holds its count of finite pupil nodes,
        sum, peak and centroid sums (cp, cq) = (sum psf*p, sum psf*q) from a
        device reduction.  ``triangulation="device"`` triangulates the
        exit pupil in HBM too (rtx_delaunay) instead of with scipy on the host"""
        if not resample:
            raise NotImplementedError       # as in the reference
        eng = self._engine()
        radius = self.system[-1].distance
        after, image = kwargs.pop("after", -2), kwargs.pop("image", -1)
        if kwargs:
            raise TypeError("unexpected arguments %s" % sorted(kwargs))
        xs, ys, o = self._opd_grid(radius, after, image, resample, download=False,
                                   triangulation=triangulation)
        p, q, out, self.psf_stats = psf_of_grid(eng, xs, o, pad, self.l/self.system.scale, radius)
        if download:
            psf = out.download()
            out.free()
            return p, q, psf
        return p, q, out

    def psf_profiles(self, pad=4, resample=4, triangulation="host", **kwargs):
        """The encircled energy and MTF Analysis.opds (rayopt/analysis.py:
        319-346) takes from ``psf``, with the PSF kept in HBM: ``psf_device``
        (download=False), its centroid (x0, y0) = (cp, cq) from the device
        stats, dx from the fftshifted p axis after subtracting x0 as Analysis
        does, and rtx_psf_profiles about (nx/2 + x0/dx, ny/2 + y0/dx) (true
        division: for odd sizes half a pixel from the fftshift origin, as in
        Analysis).  Returns a dict: stats, x0, y0, dx, center, xe (bin radii),
        ee (cumulative), of (frequencies) and mtf (axis 0, axis 1); the 1-d
        inverse FFTs of the line sums run on the host.  ``triangulation`` as
        in ``psf_device``."""
        p, q, out = self.psf_device(pad, resample, download=False, triangulation=triangulation,
                                    **kwargs)
        return psf_profiles(self._engine(), p, out, self.psf_stats)

    # ---- diffraction PSF by direct summation over the traced rays
    def psf_direct(self, pixels=(128, 128), pitch=None, center=(0., 0.), defocus=(0.,),
                   radius=None, after=-2, image=-1, weights=None, download=True):
        """The diffraction PSF as the Debye sum of the pupil function over the
        traced rays themselves (rtx_trace_opd, rtx_pupil_sum,
        rtx_pupil_intensity): no regridding and no FFT, so obscured or
        vignetted pupils keep their shape, and the grid is the caller's.  The
        image grid is ``center + (a - nx//2) pitch`` along x and likewise
        along y about the ref ray's image point (``pitch=None``: an eighth
        of the Airy radius at the trace's wavelength), at each `defocus`
        plane; the sphere is ``psf()``'s (``radius=None``:
        ``system[-1].distance``).  `weights` (N,) per ray, numpy or a
        DeviceArray (None: all 1).  Returns (p, q, psf (K, nx, ny)) in
        Strehl units, |U|^2/(sum w)^2, psf a DeviceArray when not
        `download` (free it when done).  ``self.psf_direct_stats`` holds
        count (rays summed), left_out, sum_w, and per plane strehl (at the
        chief point), peak, peak_at (p, q), centroid (p, q) and sum."""
        from .engine import pupil_spec
        eng = self._engine()
        after, image = range(self.length)[after], range(self.length)[image]
        radius = self.system[-1].distance if radius is None else float(radius)
        nx, ny = (int(v) for v in pixels)
        z = np.atleast_1d(np.asarray(defocus, np.float64))
        lam = self.l/self.system.scale
        if pitch is None:
            par = self.system.paraxial
            pitch = par.airy_radius[1]/par.wavelength*self.l/8
        p = float(center[0]) + (np.arange(nx) - nx//2)*float(pitch)
        q = float(center[1]) + (np.arange(ny) - ny//2)*float(pitch)
        p0, q0 = float(center[0]) - (nx//2)*float(pitch), float(center[1]) - (ny//2)*float(pitch)
        pupil_spec(z, (nx, ny), p0, pitch, q0, pitch, 0., lam, 1/lam, radius)   # refuse early
        A, P = self._trace_opd(radius, after, image)
        bufs = [A, P]
        try:
            ref = int(self.ref)
            a0 = float(A.rows(ref).download()[0])
            kappa = self.n[after]/lam
            spec = pupil_spec(z, (nx, ny), p0, pitch, q0, pitch, a0, lam, kappa, radius)
            chief = pupil_spec(z, (1, 1), 0., pitch, 0., pitch, a0, lam, kappa, radius)
            w = weights
            if w is not None and not hasattr(w, "ptr"):
                w = eng.to_device(np.asarray(w, np.float64))
                bufs.append(w)
            U = eng.empty((len(z), nx, ny), np.complex128)
            U1 = eng.empty((len(z), 1, 1), np.complex128)
            bufs += [U, U1]
            eng.memset(U)
            eng.memset(U1)
            count, sw = eng.pupil_sum(A, P, spec, U, w=w, N=self.nrays)
            eng.pupil_sum(A, P, chief, U1, w=w, N=self.nrays)
            if not count or not sw:
                raise ValueError("no rays made it through")
            out = eng.empty((len(z), nx, ny))
            eng.memset(out)
            try:
                st = eng.pupil_intensity(spec, U, out, 1/sw**2)
            except Exception:
                out.free()
                raise
            u1 = U1.download()[:, 0, 0]
        finally:
            for a in bufs:
                a.free()
        at = st[:, 2].astype(np.int64)
        with np.errstate(invalid="ignore", divide="ignore"):
            self.psf_direct_stats = dict(
                count=count, left_out=self.nrays - count, sum_w=sw,
                strehl=np.abs(u1)**2/sw**2, peak=st[:, 1].copy(),
                peak_at=np.stack([p[at//ny], q[at % ny]], -1), sum=st[:, 0].copy(),
                centroid=st[:, 3:5]/st[:, :1])
        pp, qq = np.broadcast_arrays(p[:, None], q[None, :])
        if download:
            psf = out.download()
            out.free()
            return pp, qq, psf
        return pp, qq, out

    # ---- through-focus spot images (Analysis.spots, rayopt/analysis.py:250-283)
    def spot_image(self, defocus=(0.,), bins=(256, 256), range=None, at=-1, radial=False,
                   offsets=None, download=True):
        """Spot images of the stored rows y[at], i[at] at the planes `defocus`
        (rtx_spot_rows): the points ``y - y[ref] + z*tanarcsin(i) - offsets``
        of Analysis.spots (analysis.py:266-280) binned as np.histogram2d
        (radial: their radii as np.histogram) would bin them, exactly.  With
        ``range=None`` an extent pass picks the symmetric range that holds
        every finite point (spot.default_range).  A vignetted ref ray gives
        a NaN centre and counts nothing.  Returns a dict: z, counts (K, nx,
        ny) or (K, nx) uint64 (a DeviceArray when ``download=False``), edges,
        range, tally (K, 2): rays binned, rays with a non-finite point."""
        from .spot import spot_images
        eng, d = self._engine(), self._dev
        at = int(np.arange(self.length)[at])
        ref = 0 if self.ref is None else int(self.ref)
        c = eng.download_rays(d["y"].rows(at), [ref])[0, :2].astype(np.float64)

        def part(spec, counts, extent):
            return eng.spot_rows(d["y"].rows(at), d["i"].rows(at), spec, counts, N=self.nrays,
                                 extent=extent)
        return self._one_image(spot_images(eng, [(c, [part])], defocus, bins, range, radial,
                                           offsets, download))

    def spot_image_fused(self, defocus=(0.,), bins=(256, 256), range=None, at=-1, radial=False,
                         offsets=None, download=True, clip=False):
        """``spot_image`` of a march from the launch rays (row 0) to surface
        `at` with the binning as its epilogue (rtx_trace_spot): no row is
        stored or read.  The centre is the ref ray's, from a 1-ray trace."""
        from .spot import spot_images
        eng, d = self._engine(), self._dev
        at = int(np.arange(self.length)[at])
        table, _, rot0 = pack_system(self.system, self.l, 1, at + 1, n0=self.n[0])
        c = self._chief(table, rot0, clip)[:2]

        def part(spec, counts, extent):
            return eng.trace_spot(table, d["y"].rows(0), d["u"].rows(0), spec, counts,
                                  N=self.nrays, clip=clip, rot0=rot0, exact=self.exact,
                                  extent=extent)
        return self._one_image(spot_images(eng, [(c, [part])], defocus, bins, range, radial,
                                           offsets, download))

    # ---- geometric MTF through focus (the Fourier transform of spot_image)
    def geometric_mtf(self, defocus=(0.,), dnu=None, nfreq=64, at=-1):
        """The geometric OTF of the stored rows y[at], i[at] about y[at, ref]
        at the planes `defocus` (rtx_otf_rows): the mean over the rays with a
        finite point q of exp(-2 pi i nu q), per plane, axis (x, y) and
        frequency ``arange(nfreq)*dnu`` (``dnu=None``: the last frequency is
        1/airy_radius, as mtf.geometric_mtf).  A vignetted ref ray gives a
        NaN centre, counts nothing and gives NaN.  Returns a dict: freq (F,),
        z (K,), otf complex (K, 2, F), mtf = |otf|, count (K,) int64."""
        from .engine import otf_spec
        from .mtf import _otf, default_dnu
        eng, d = self._engine(), self._dev
        at = int(np.arange(self.length)[at])
        ref = 0 if self.ref is None else int(self.ref)
        z = np.atleast_1d(np.asarray(defocus, np.float64))
        F = int(nfreq)
        dnu = default_dnu(self.system, F) if dnu is None else float(dnu)
        c = eng.download_rays(d["y"].rows(at), [ref])[0, :2].astype(np.float64)
        spec = otf_spec(z, dnu, F, np.nan_to_num(c))
        if np.isfinite(c).all():
            S, count = eng.otf_rows(d["y"].rows(at), d["i"].rows(at), spec, N=self.nrays)
        else:
            S, count = np.zeros((len(z), 2, F), np.complex128), np.zeros(len(z), np.int64)
        otf = _otf(S, count)
        return dict(freq=np.arange(F)*dnu, z=z, otf=otf, mtf=np.abs(otf), count=count)

    @staticmethod
    def _one_image(out):
        out["counts"], out["tally"] = out["counts"][0], out["tally"][0]
        return out


class ResidentTrace(ResidentMixin):
    """Standalone resident drop-in (no rayopt import needed) with launch rays
    generated in HBM (SURVEY 8f-2)."""

    def __init__(self, system, engine=None, exact=False, alias_incidence=True):
        self.system = system
        self.engine = engine or default_engine()
        self.exact = exact
        self.alias_incidence = alias_incidence
        self._dev = None

    def rays_infinite(self, yo, z, p, angle, l=None, nrays=None, yp=None, ref=0):
        """Launch rays of an aimed bundle for an infinite conjugate generated
        directly in HBM (as Engine.aim_infinite_device): the hexapolar grid
        with about `nrays` rays, or the DEVICE FP64 pupil coordinates `yp`
        (N,2); (z, p) is the reference's pupil-aiming solution (System.pupil).
        Nothing crosses PCIe."""
        from .rays import infinite_record, pupil_grid
        spec = infinite_record(yo, z, p, angle, grid=pupil_grid(yp, nrays))
        self._generate(spec, yp, self.system.wavelengths[0] if l is None else l, ref)

    def _generate(self, spec, yp, l, ref):
        """the bundle of the `rtx_aim` record `spec` into row 0, at wavelength
        `l` with default weights and reference ray `ref`"""
        eng = self.engine
        count = eng.aim_count(spec, yp)
        if self._dev is None or self.nrays != count:
            self.allocate(count)
        self.l = l
        self.w = None
        self._w_default, self._w_dev = True, None
        self.ref = ref
        d = self._dev
        eng.aim_rays_into(spec, d["y"].rows(0), d["u"].rows(0), count, yp=yp)
        d["i"].rows(0).copy_from(d["u"].rows(0), count*24)   # i[0] = u[0] (geometric_trace.py:68)
        self._zero_t0()
        for a in (self.y, self.u, self.i, self.t):
            a.invalidate()
        self.n[0] = self.system.refractive_index(self.l, 0)

    def rays_device(self, yo, wavelength=None, nrays=11, distribution="hexapolar", filter=False,
                    stop=None, seed=0):
        """Launch rays of ``rays_point`` generated in HBM by the general
        generator (rtx_aim_plan / rtx_aim_rays): the pupil grid (hexapolar,
        square, triangular, random, meridional / sagittal / cross / tee lines),
        Pupil.map with its `filter`, Conjugate.aim for finite and infinite
        objects in every projection, telecentric pupils, curved object
        surfaces.  ``system.pupil`` (the aiming) stays host Python.  Returns
        False (nothing done) for the distributions that stay on the host."""
        from .rays import aim_record, grid_spec
        s = self.system
        ref, grid = grid_spec(distribution, nrays)
        if grid is None:
            return False
        l = s.wavelengths[0] if wavelength is None else wavelength
        z, p = s.pupil(yo, l=wavelength, stop=stop)
        self._generate(aim_record(s.object, yo, z, p, grid, filter, s[0], seed), None, l, ref)
        return True

    def rays_point(self, yo, wavelength=None, nrays=11, distribution="hexapolar",
                   filter=None, stop=None, clip=False):
        """GeometricTrace.rays_point (rayopt/geometric_trace.py:204-209) for a
        rayopt ``System``: the pupil is aimed by the reference on the host
        (``system.pupil``), the launch rays are generated in HBM
        (``rays_device``) -- or by ``system.aim`` on the host and uploaded for
        the quadrature distributions -- and traced with `clip`."""
        s = self.system
        filt = (not clip) if filter is None else filter
        if not self.rays_device(yo, wavelength, nrays, distribution, filt, stop):
            from rayopt.utils import pupil_distribution      # the reference's own helper
            l = s.wavelengths[0] if wavelength is None else wavelength
            z, p = s.pupil(yo, l=wavelength, stop=stop)
            ref, yp, weight = pupil_distribution(distribution, nrays)
            y, u = s.aim(yo, yp, z, p, filter=filt)
            self.rays_given(y, u, l, weight, ref)
        self.propagate(clip=clip)
