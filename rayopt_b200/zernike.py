"""Zernike decomposition of the wavefront on the device.

The rms wavefront of ``tolerance_wavefront`` says how large a lens's
aberration is; its Zernike coefficients say which it is: defocus,
astigmatism, coma, spherical.  ``tolerance_zernike`` marches every perturbed
lens as ``tolerance_wavefront`` does and reduces each bundle's rays, in the
same launch, to the Gram sums of a least-squares fit of Noll's orthonormal
Zernike polynomials Z_1 .. Z_J (rtx_trace_zernike_many); the fit is made
here from those sums.  ``zernike`` is the same path for the nominal lens.

Pupil coordinates: the points (x, y) of opd()'s reference sphere in the
image frame, relative to the chief ray's, divided by a radius rho_b that the
NOMINAL lens sets for each (height, wavelength) bundle: the largest
sqrt(x^2 + y^2) of its entering rays.  Every variant of that bundle uses the
same rho_b, so their coefficients are comparable; a variant whose pupil is
larger simply has points at r > 1.  The residual after removing all terms
up to an order does not depend on rho: a polynomial space is invariant
under scaling."""
import math

import numpy as np

from .engine import ZRN_MAX_ORDER

__all__ = ["noll", "zernike_basis", "zernike_fit", "tolerance_zernike", "zernike"]


def nterms(order):
    """J = (order+1)(order+2)/2, the number of terms up to radial `order`"""
    return (order + 1)*(order + 2)//2


def noll(J):
    """(J, 2) int: the (n, m) of Noll's Z_1 .. Z_J; m > 0 is cos(m theta)
    (even j), m < 0 is sin(|m| theta) (odd j)"""
    out, n = [], 0
    while len(out) < J:
        for o in range(n + 1):                                 # j = n(n+1)/2 + 1 + o
            j = n*(n + 1)//2 + 1 + o
            m = 2*(o//2) + 1 if n % 2 else 2*((o + 1)//2)
            out.append((n, m if m == 0 or j % 2 == 0 else -m))
        n += 1
    return np.array(out[:J], np.int64).reshape(J, 2)


def radial_coefficients(n, m):
    """c_k of R_n^|m|(r) = sum_k c_k r^(n-2k), k = 0 .. (n-|m|)/2"""
    m = abs(m)
    return [(-1)**k*math.factorial(n - k)
            // (math.factorial(k)*math.factorial((n + m)//2 - k)*math.factorial((n - m)//2 - k))
            for k in range((n - m)//2 + 1)]


def zernike_basis(J, x, y):
    """(..., J) Z_1 .. Z_J at the pupil points (x, y) (arrays of one shape),
    in closed form: sqrt(n+1) R_n^0, sqrt(2(n+1)) R_n^m cos(m theta) for
    even j, sin for odd j, theta = atan2(y, x).  The dtype follows x and y
    (np.longdouble for an extended-precision reference)."""
    x, y = np.broadcast_arrays(x, y)
    dt = np.result_type(x.dtype, np.float64)
    x, y = x.astype(dt), y.astype(dt)
    r, th = np.hypot(x, y), np.arctan2(y, x)
    out = np.empty(x.shape + (J,), dt)
    for j, (n, m) in enumerate(noll(J)):
        R = sum(dt.type(c)*r**(n - 2*k) for k, c in enumerate(radial_coefficients(n, m)))
        if m == 0:
            out[..., j] = np.sqrt(dt.type(n + 1))*R
        else:
            ang = np.cos(abs(m)*th) if m > 0 else np.sin(abs(m)*th)
            out[..., j] = np.sqrt(dt.type(2*(n + 1)))*R*ang
    return out


def unpack(sums, J):
    """rtx_trace_zernike_many's upper triangle (..., E) -> the symmetric
    (..., J+1, J+1) Gram sums of (a, Z_1 .. Z_J)"""
    sums = np.asarray(sums, np.float64)
    p, q = np.triu_indices(J + 1)
    M = np.zeros((int(np.prod(sums.shape[:-1])), (J + 1)*(J + 1)))
    flat = sums.reshape(len(M), -1)
    M[:, p*(J + 1) + q] = flat
    M[:, q*(J + 1) + p] = flat
    return M.reshape(sums.shape[:-1] + (J + 1, J + 1))


def zernike_fit(sums, J, wl):
    """The least-squares fit of Z_1 .. Z_J to a from the sums (..., E) and
    the wavelength(s) `wl` in lens units (broadcast to sums.shape[:-1]).

    Forms G = Gram/n and b = sum a Z/n and takes the minimum-norm c_a = G+ b
    through eigh, eigenvalues below 1e-12 x the largest taken as zero.
    Returns a dict: coefficients (..., J) = -c_a/wl in waves of opd()'s t =
    -(A - A_ref)/wl, residual = sqrt(max(sum a^2/n - c_a.b, 0))/wl the rms
    after removing the J terms, rms the piston-removed rms (as
    tolerance_wavefront's), rank (...,).  NaN where no ray entered."""
    sums = np.asarray(sums, np.float64)
    shape = sums.shape[:-1]
    if sums.shape[-1] != (J + 1)*(J + 2)//2:
        raise ValueError("sums of %d columns are not those of J = %d" % (sums.shape[-1], J))
    M = unpack(sums, J).reshape(-1, J + 1, J + 1)
    wl = np.broadcast_to(np.asarray(wl, np.float64), shape).reshape(-1)
    n = M[:, 1, 1]
    ok = np.isfinite(M).all((1, 2)) & (n > 0)
    ca = np.full((len(M), J), np.nan)
    resid = np.full(len(M), np.nan)
    rank = np.zeros(len(M), np.int64)
    if ok.any():
        Mo, no = M[ok], n[ok][:, None]
        G, b = Mo[:, 1:, 1:]/no[..., None], Mo[:, 0, 1:]/no
        w, Q = np.linalg.eigh(G)
        keep = w > 1e-12*w[:, -1:]
        inv = np.where(keep, 1/np.where(keep, w, 1), 0.)
        c = np.einsum("ijk,ik->ij", Q, inv*np.einsum("ilk,il->ik", Q, b))   # Q diag(inv) Q^T b
        ca[ok] = c
        resid[ok] = np.sqrt(np.maximum(Mo[:, 0, 0]/no[:, 0] - (c*b).sum(-1), 0.))
        rank[ok] = keep.sum(-1)
    with np.errstate(all="ignore"):
        dbar = M[:, 0, 1]/n                                    # sum a Z_1 = sum a
        rms = np.sqrt(np.maximum((M[:, 0, 0]/n - dbar*dbar)/(wl*wl), 0.))
        rms = np.where(np.isnan(dbar), np.nan, rms)
    return dict(coefficients=(-ca/wl[:, None]).reshape(shape + (J,)),
                residual=(resid/wl).reshape(shape), rms=rms.reshape(shape),
                rank=rank.reshape(shape))


def _check_order(order):
    if isinstance(order, bool) or not isinstance(order, (int, np.integer)) \
            or not 0 <= order <= ZRN_MAX_ORDER:
        raise ValueError("order must be an integer in 0..%d, got %r" % (ZRN_MAX_ORDER, order))
    return int(order)


def tolerance_zernike(system, params, deltas, heights=(0., .707, 1.), wavelengths=None,
                      nrays=1000, distribution="hexapolar", order=6, compensate=None,
                      engine=None, exact=False, chunk=None):
    """The Zernike coefficients of the wavefront of every perturbed lens at
    every field height and wavelength, on the device: the decomposition
    counterpart of ``tolerance_wavefront``.

    `params` [(j, kind)] and `deltas` (V, P) are ``perturbed_tables``'; a
    shape or tilt of the image surface is refused, its distance is not.
    Each (height, wavelength) bundle is aimed once for the NOMINAL lens and
    marched through all V variants with clipping (no re-aiming); each
    variant's rays are referred to its own chief ray and reference sphere
    exactly as in ``tolerance_wavefront``.  Pupil coordinates are (x, y)/rho
    with rho of each bundle set by the nominal lens (see the module
    docstring).  `order` is the radial order 0..8 (J = (order+1)(order+2)/2
    terms, Noll's order).  ``compensate="focus"`` refocuses each variant
    first, as ``tolerance`` does.  `chunk`: variants per launch (default: as
    many as fit in 1 GiB of tables and tile rows); the results do not depend
    on it.  FP64 only.  ``tolerance_zernike(system, params,
    sensitivity_deltas(tol))`` gives each tolerance's Zernike signature.

    Returns a dict: coefficients (V, H, W, J) in waves (lambda =
    l/system.scale) of opd()'s t, residual (V, H, W) the rms after removing
    the J terms, rms (V, H, W) the piston-removed rms (tolerance_wavefront's),
    rank (V, H, W) of the fit, radius (H, W) rho, transmitted (V, H, W),
    chief (V, H, W) true where the chief ray reaches the image (elsewhere
    every value is NaN), noll (J, 2) the (n, m) of each term (m < 0: sine),
    sums (V, H, W, E) rtx_trace_zernike_many's, focus (V,) when compensated,
    heights, wavelengths, params, deltas.  Every argument is checked before
    any device work."""
    from .tolerance import VariantMarch, check_fields, perturbed_tables
    order = _check_order(order)
    J = nterms(order)
    E = (J + 1)*(J + 2)//2
    heights, wavelengths = check_fields(system, heights, wavelengths, compensate, chunk)
    H, W = len(heights), len(wavelengths)
    with VariantMarch(system, params, deltas, heights, wavelengths, nrays, distribution,
                      compensate, chunk, engine, exact, wavefront=True) as r:
        eng, ref, rot0 = r.eng, r.ref, r.rot0
        # rho_b: the nominal lens's largest pupil radius of each bundle (order 0)
        t = perturbed_tables(r.nominal, [], np.zeros((1, 0)))
        march, items, specs, a0, cen = ref.chief(eng, t, rot0, exact)[:5]
        _, r2 = eng.trace_zernike_many(march, r.dev, items, specs, np.ones(H*W), 0, a0, cen,
                                       clip=True, rot0=rot0, exact=exact)
        radius = np.sqrt(r2)
        rho = np.where(radius > 0, radius, 1.)
        sums = np.empty((r.V, H, W, E))
        chief = np.empty((r.V, H, W), bool)
        for v0, t, _ in r.chunks(8*(E + 1), H*W):
            n = len(t)
            march, items, specs, a0, cen, ok = ref.chief(eng, t, rot0, exact)
            s, _ = eng.trace_zernike_many(march, r.dev, items, specs, np.tile(rho, n), order, a0,
                                          cen, clip=True, rot0=rot0, exact=exact)
            sums[v0:v0 + n] = s.reshape(n, H, W, E)
            chief[v0:v0 + n] = ok.reshape(n, H, W)
    wl = np.array([l/system.scale for l in wavelengths])
    out = zernike_result(sums, J, wl, r.counts, chief)
    out["radius"] = np.where(radius > 0, radius, np.nan).reshape(H, W)
    return r.result(out)


def zernike_result(sums, J, wl, N, chief=None):
    """tolerance_zernike's result from the sums (V, H, W, E), the
    wavelengths `wl` (W,) in lens units, the bundles' ray counts N (H, W)
    and `chief` (V, H, W) bool (None: all true); an item whose chief ray is
    lost has NaN for every value"""
    sums = np.array(sums, np.float64)
    V, H, W, _ = sums.shape
    chief = np.ones((V, H, W), bool) if chief is None else np.asarray(chief, bool)
    sums[~chief] = np.nan
    fit = zernike_fit(sums, J, np.asarray(wl, np.float64).reshape(W))
    with np.errstate(all="ignore"):
        fit["transmitted"] = sums[..., 1 + J]/np.asarray(N, np.float64).reshape(H, W)
    fit.update(chief=chief, noll=noll(J), sums=sums)
    return fit


def zernike(system, heights=(0., .707, 1.), wavelengths=None, nrays=10**4,
            distribution="hexapolar", order=6, engine=None, exact=False):
    """The Zernike coefficients of the nominal lens's wavefront at every
    field height and wavelength, on the device: ``tolerance_zernike`` with
    the nominal lens as the only variant and the variant axis dropped.
    Returns its dict without params, deltas and the V axis."""
    out = tolerance_zernike(system, [], np.zeros((1, 0)), heights, wavelengths, nrays,
                            distribution, order, engine=engine, exact=exact)
    for k in ("coefficients", "residual", "rms", "rank", "transmitted", "chief", "sums"):
        out[k] = out[k][0]
    del out["params"], out["deltas"]
    return out
