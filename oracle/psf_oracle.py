"""numpy / scipy statement of the diffraction PSF of a traced bundle
(rayopt/geometric_trace.py:133-169), the yardstick of the device path
(rtx_grid_linear, rtx_psf).

Two parts:

* ``regrid``: the linear interpolation griddata(method="linear") performs,
  written out on scipy's own triangulation: the simplex of every grid node
  from ``Delaunay.find_simplex``, its barycentric coordinates from
  ``Delaunay.transform`` (c0 and c1 accumulated from zero in index order,
  c2 = (1 - c0) - c1) and the value ((0 + c0 v0) + c1 v1) + c2 v2.  This is
  griddata's own evaluation order, so the result is griddata's bit for bit;
  ``winner`` exposes the simplex per node.
* ``psf``: the pupil function exp(-2 pi i o) over the finite nodes, scaled by
  1/sqrt(#finite), zero-padded at the end to pad*n per axis, its unnormalised
  2-d FFT, |.|^2 over the number of padded nodes, and the frequency axis
  fftfreq(pad*n, dx k / radius) with k = scale / wavelength.
"""
import numpy as np
from scipy.spatial import Delaunay


def grid(n, h):
    """the (n, n) node coordinates of the reference's regridding, and the
    axis gh with node (i, j) = (gh[i], gh[j])"""
    xs, ys = np.mgrid[-1:1:1j*n, -1:1:1j*n]*h
    return xs, ys, xs[:, 0].copy()


def triangulate(x, y):
    """the triangulation griddata makes of the points (default options)"""
    return Delaunay(np.stack([x, y], axis=-1))


def winner(tri, xs, ys):
    """find_simplex of every node, -1 outside the hull"""
    return tri.find_simplex(np.stack([xs.ravel(), ys.ravel()], axis=-1)).reshape(xs.shape)


def barycentric_value(tri, values, s, xs, ys):
    """value of the linear interpolant on simplex s at (xs, ys) (arrays of one
    shape; s >= 0), in scipy's evaluation order"""
    tr = tri.transform[s]                    # (..., 3, 2)
    dx = xs - tr[..., 2, 0]
    dy = ys - tr[..., 2, 1]
    c0 = (0. + tr[..., 0, 0]*dx) + tr[..., 0, 1]*dy
    c1 = (0. + tr[..., 1, 0]*dx) + tr[..., 1, 1]*dy
    c2 = (1. - c0) - c1
    v = values[tri.simplices[s]]             # (..., 3)
    return ((0. + c0*v[..., 0]) + c1*v[..., 1]) + c2*v[..., 2]


def regrid(x, y, t, n, h, tri=None):
    """griddata((x, y), t, (xs, ys), method="linear", fill_value=nan) on the
    reference's grid; returns (xs, ys, o)"""
    xs, ys, _ = grid(n, h)
    tri = triangulate(x, y) if tri is None else tri
    s = winner(tri, xs, ys)
    o = np.full(xs.shape, np.nan)
    hit = s >= 0
    o[hit] = barycentric_value(tri, np.asarray(t, float), s[hit], xs[hit], ys[hit])
    return xs, ys, o


def opd_grid(x, y, t, nrays, resample=4):
    """GeometricTrace.opd's regridding of per-ray (x, y, t) (rays with any
    non-finite coordinate dropped); n from the bundle's ray count"""
    ok = np.isfinite(x) & np.isfinite(y) & np.isfinite(t)
    x, y, t = x[ok], y[ok], t[ok]
    if not t.size:
        raise ValueError("no rays made it through")
    n = int(resample*nrays**.5)
    h = np.fabs((x, y)).max()
    return regrid(x, y, t, n, h)


def psf(xs, o, pad, wavelength, radius):
    """(p, q, psf) of the regridded OPD `o` on the grid `xs`; `wavelength` in
    the system's length unit (l/scale)"""
    good = np.isfinite(o)
    z = np.zeros(o.shape, complex)
    z[good] = np.exp(-2j*np.pi*o[good])
    z = z/np.count_nonzero(good)**.5
    nx, ny = pad*o.shape[0], pad*o.shape[1]
    field = np.fft.fft2(z, (nx, ny))
    intensity = (field*field.conj()).real/field.size
    f = frequencies(xs, nx, wavelength, radius)
    p, q = np.broadcast_arrays(f[:, None], f)
    return p, q, intensity


def frequencies(xs, nx, wavelength, radius):
    """the frequency axis of the PSF of an (n, n) grid padded to nx"""
    dx = xs[1, 0] - xs[0, 0]
    return np.fft.fftfreq(nx, dx*(1/wavelength)/radius)


def stats(p, q, psf):
    """what Analysis takes from a PSF (rayopt/analysis.py:319-322): sum,
    peak and the first moments about the frequency axes"""
    return dict(sum=psf.sum(), max=psf.max(), cp=(psf*p).sum(), cq=(psf*q).sum())
