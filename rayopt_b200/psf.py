"""Diffraction PSF by direct summation over the exit-pupil rays, through
focus, polychromatic and at any image sampling, on the device.

The PSF is the Debye sum of the pupil function over the traced rays
themselves (rtx_pupil_sum, include/rtx.h) on an image grid the caller
chooses: no regridding of the pupil (an obscured or vignetted pupil keeps
its shape), no FFT (the pitch does not depend on the wavelength or the pupil
size), and any defocus.  Every wavelength of a field lands on one grid, so
the polychromatic PSF is a weighted sum in HBM (rtx_pupil_intensity).
"""
import warnings

import numpy as np

from .engine import default_engine, pupil_spec
from .lazy import opd_spec


def psfs(system, heights=(0., .707, 1.), wavelengths=None, nrays=10**5,
         distribution="hexapolar", pixels=(128, 128), pitch=None, defocus=(0.,),
         spectral_weights=None, chunk=2**22, download=True, engine=None, exact=False,
         per_wavelength=False):
    """Diffraction PSFs of a rayopt ``System`` at each height, polychromatic
    and per wavelength, through focus.

    For each height and wavelength the pupil is aimed on the host
    (``system.pupil``), the launch rays are generated in HBM in chunks of at
    most `chunk` rays, each chunk is marched with clipping to the last
    surface before the image with the OPD as the epilogue (rtx_trace_opd,
    ``psf()``'s sphere of radius ``system[-1].distance`` about the
    wavelength's own chief ray) and added to the pupil sum (rtx_pupil_sum).

    The grid is ``(a - nx//2) pitch`` (``pitch=None``: an eighth of the Airy
    radius of ``wavelengths[0]``) about the chief ray of ``wavelengths[0]``
    on the image surface; each wavelength's grid origin is shifted by its
    own chief ray's offset from it, so the polychromatic PSF, the
    `spectral_weights`-weighted mean (equal by default) of the wavelengths
    whose chief ray reaches the image and that sum rays, shows lateral
    colour.  A vignetted chief ray gives NaN for that wavelength.  The pupil
    sums of a height's wavelengths stay in HBM until its polychromatic PSF
    is formed (W K nx ny complex values).  `defocus` are plane distances
    from the image surface along its z.

    Returns a dict: heights, wavelengths, z (K,), p (nx,), q (ny,), poly
    (H, K, nx, ny) in Strehl units (DeviceArrays when not `download`), psf
    (H, W, K, nx, ny) with `per_wavelength`, strehl (H, W, K) at the chief
    point, peak (H, W, K), poly_peak (H, K), centroid (H, W, K, 2) and
    poly_centroid (H, K, 2) on the grid's axes, count (H, W) rays summed,
    sum_w (H, W), chief_offset (H, W, 2) and alias_half_width (H, W), the
    half-width lambda R/(n delta) within which the ray sampling (mean
    spacing delta in the exit pupil) does not alias; a warning is given when
    the grid reaches past half of it."""
    from .rays import grid_spec
    eng = engine or default_engine()
    wavelengths = list(system.wavelengths if wavelengths is None else wavelengths)
    heights = list(heights)
    H, W = len(heights), len(wavelengths)
    z = np.atleast_1d(np.asarray(defocus, np.float64))
    K = len(z)
    nx, ny = (int(v) for v in pixels)
    if pitch is None:
        par = system.paraxial
        pitch = par.airy_radius[1]/par.wavelength*wavelengths[0]/8
    pitch = float(pitch)
    p = (np.arange(nx) - nx//2)*pitch
    q = (np.arange(ny) - ny//2)*pitch
    p0, q0 = -(nx//2)*pitch, -(ny//2)*pitch
    radius = system[-1].distance
    pupil_spec(z, (nx, ny), p0, pitch, q0, pitch, 0., 1., 1., radius)   # refuse before any work
    weights = np.ones(W) if spectral_weights is None else \
        np.asarray(spectral_weights, np.float64).reshape(W)
    ref, grid = grid_spec(distribution, nrays)
    if grid is None:
        raise ValueError("distribution %r with %d rays is not generated on the device"
                         % (distribution, nrays))
    chunk = int(chunk)
    if chunk < 1:
        raise ValueError("chunk must be >= 1")
    L = len(system)
    after, image = L - 2, L - 1
    nan = np.full((H, W, K), np.nan)
    res = dict(heights=heights, wavelengths=wavelengths, z=z, p=p, q=q,
               strehl=nan.copy(), peak=nan.copy(), centroid=np.full((H, W, K, 2), np.nan),
               poly_peak=np.full((H, K), np.nan), poly_centroid=np.full((H, K, 2), np.nan),
               count=np.zeros((H, W), np.int64), sum_w=np.zeros((H, W)),
               chief_offset=np.full((H, W, 2), np.nan), alias_half_width=np.full((H, W), np.nan))
    polys, per = [], []
    try:
        for h in range(H):
            poly = eng.empty((K, nx, ny))
            polys.append(poly)
            per.append([])
            _height(eng, system, res, h, poly, per[h], heights[h], wavelengths, weights, ref,
                    grid, z, (nx, ny), p0, q0, pitch, radius, after, image, chunk, exact,
                    per_wavelength, download)
        res["poly"] = np.stack([a.download() for a in polys]) if download else polys
    except BaseException:
        for a in polys:
            a.free()
        raise
    if download:
        for a in polys:
            a.free()
    if per_wavelength:
        res["psf"] = per if not download else np.stack(
            [np.stack([np.full((K, nx, ny), np.nan) if a is None else a for a in row])
             for row in per])
    return res


def _height(eng, system, res, h, poly, per, height, wavelengths, weights, ref, grid, z, pixels,
            p0, q0, pitch, radius, after, image, chunk, exact, per_wavelength, download):
    """psfs for one height: every wavelength's pupil sum (kept in HBM), its
    PSF and stats, then the polychromatic PSF `poly` over the wavelengths
    that summed rays"""
    from .rays import aim_record
    from .surface_table import pack_system
    K, (nx, ny) = len(z), pixels
    yo = (0, height)
    held = []                                   # device buffers freed on the way out
    try:
        plans = []
        for wl in wavelengths:
            n0 = system.refractive_index(wl, 0)
            table, n_rows, rot0 = pack_system(system, wl, 1, None, n0=n0)
            n = np.r_[n0, n_rows]
            zp, pp = system.pupil(yo, l=wl)
            rec = aim_record(system.object, yo, zp, pp, grid, False, system[0])
            cy, cu = eng.aim_rays(rec, first=ref, count=1)
            held += [cy, cu]
            y0_ref, u0_ref = cy.download()[0], cu.download()[0]
            Y = eng.trace(table, y0_ref[None], u0_ref[None], clip=True, rot0=rot0,
                          keep_last=True, exact=exact, want=("y",))[0][0, 0]
            plans.append((wl, n, rec, cy, cu, y0_ref, u0_ref, Y))
        c0 = plans[0][-1][:2]
        U1, Iw = eng.empty((K, 1, 1), np.complex128), eng.empty((K, nx, ny))
        held += [U1, Iw]
        summed = []                             # (w, spec, U, sum w, off) with rays
        for w, (wl, n, rec, cy, cu, y0_ref, u0_ref, Y) in enumerate(plans):
            if not (np.isfinite(Y).all() and np.isfinite(c0).all()):
                if per_wavelength:
                    per.append(None)
                continue
            lam = wl/system.scale
            kappa = n[after]/lam
            off = Y[:2] - c0
            res["chief_offset"][h, w] = off
            spec_o = opd_spec(system, system.track, system.origins, after, image, n[0],
                              n[after], y0_ref, u0_ref, Y, radius)
            t_after, _, rot_after = pack_system(system, wl, 1, after + 1, n0=n[0])
            A1, P1 = eng.empty((1,)), eng.empty((1, 3))
            try:
                eng.trace_opd(t_after, cy, cu, spec_o, A1, P1, N=1, clip=True,
                              rot0=rot_after, exact=exact)
                a0 = float(A1.download()[0])
            finally:
                A1.free(), P1.free()
            # this wavelength's grid, in the frame of its own chief ray
            spec = pupil_spec(z, (nx, ny), p0 - off[0], pitch, q0 - off[1], pitch, a0, lam,
                              kappa, radius)
            chief = pupil_spec(z, (1, 1), 0., pitch, 0., pitch, a0, lam, kappa, radius)
            U = eng.empty((K, nx, ny), np.complex128)
            held.append(U)
            eng.memset(U)
            eng.memset(U1)
            N = eng.aim_count(rec)
            cap = min(chunk, max(N, 1))
            bufs = [eng.empty((cap, 3)), eng.empty((cap, 3)), eng.empty((cap,)),
                    eng.empty((cap, 3))]
            y0, u0, A, P = bufs
            count, sw, h_pupil = 0, 0., None
            try:
                for first in range(0, N, chunk):
                    m = min(chunk, N - first)
                    eng.aim_rays_into(rec, y0, u0, m, first=first)
                    eng.trace_opd(t_after, y0, u0, spec_o, A, P, N=m, clip=True,
                                  rot0=rot_after, exact=exact)
                    c, s = eng.pupil_sum(A, P, spec, U, N=m)
                    eng.pupil_sum(A, P, chief, U1, N=m)
                    count, sw = count + c, sw + s
                    if h_pupil is None:
                        pts, vals, _, h_pupil = eng.opd_points(A, P, ref if ref < m else 0, lam)
                        pts.free(), vals.free()
            finally:
                for a in bufs:
                    a.free()
            res["count"][h, w], res["sum_w"][h, w] = count, sw
            if not count or not sw:
                if per_wavelength:
                    per.append(None)
                continue
            delta = h_pupil*np.sqrt(np.pi/count) if h_pupil else np.inf
            alias = lam*abs(radius)/(abs(n[after])*delta)
            res["alias_half_width"][h, w] = alias
            s0 = spec[0]
            reach = max(abs(s0["p0"]), abs(s0["p0"] + (nx - 1)*pitch), abs(s0["q0"]),
                        abs(s0["q0"] + (ny - 1)*pitch))   # from this wavelength's chief ray
            if reach > alias/2:
                warnings.warn("the PSF grid reaches %.3g, past half the alias-free "
                              "half-width %.3g of %d rays at height %g, wavelength %g"
                              % (reach, alias, count, height, wl))
            eng.memset(Iw)
            st = eng.pupil_intensity(spec, U, Iw, 1/sw**2)
            u1 = U1.download()[:, 0, 0]
            res["strehl"][h, w] = np.abs(u1)**2/sw**2
            res["peak"][h, w] = st[:, 1]
            res["centroid"][h, w] = st[:, 3:5]/st[:, :1] + off   # on the common grid
            if per_wavelength:
                per.append(Iw.download() if download else _copy(eng, Iw))
            summed.append((w, spec, U, sw, off))
        eng.memset(poly)
        wsum = sum(weights[w] for w, *_ in summed)
        if not summed or wsum <= 0:
            eng.memset(poly, 0xff)              # NaN: no wavelength reaches the image
            return
        for w, spec, U, sw, off in summed:
            pst = eng.pupil_intensity(spec, U, poly, weights[w]/wsum/sw**2)
        res["poly_peak"][h] = pst[:, 1]
        res["poly_centroid"][h] = pst[:, 3:5]/pst[:, :1] + off
    finally:
        for a in held:
            a.free()


def _copy(eng, a):
    b = eng.empty(a.shape, a.dtype)
    b.copy_from(a)
    return b
