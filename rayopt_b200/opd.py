"""OPD, PSF, encircled energy and MTF of every field on the device:
Analysis.opds (rayopt/analysis.py:285-352) for a rayopt ``System``, with the
plots replaced by the numbers they are drawn from.

Per height the launch rays are generated in HBM, the per-ray OPD is the
epilogue of a march that stores no trace (rtx_trace_opd), its finite
exit-pupil points are compacted in HBM (rtx_opd_points), triangulated,
regridded (rtx_grid_linear) and reduced (rtx_grid_range, rtx_psf,
rtx_psf_profiles).  Only the reductions come back unless asked for.
"""
import numpy as np

from .engine import default_engine
from .lazy import check_triangulation, opd_spec, psf_of_grid, psf_profiles, regrid


def scales(results):
    """(mm, rm) of Analysis.opds: the contour half-range max |o| and the PSF
    axis limit 1.5 dx searchsorted(ee, .9), both from the first height with
    rays in Analysis's reversed walk -- the last one here; (None, None) when
    no height has rays"""
    for r in reversed(results):
        if r is not None:
            return r["max_abs"], np.searchsorted(r["ee"], .9)*1.5*r["dx"]
    return None, None


def _points(eng, system, wl, rec, N, n, ref, y_ref, after, image, radius, exact):
    """rtx_trace_opd of the bundle `rec` (generated here) and rtx_opd_points:
    (pts, vals, M, h) with the launch rays and A, P freed"""
    from .surface_table import pack_system
    n0 = n[0]
    spec = opd_spec(system, system.track, system.origins, after, image, n0, n[after],
                    y_ref[0], y_ref[1], y_ref[2], radius)
    t_after, _, rot_after = pack_system(system, wl, 1, after + 1, n0=n0)
    y0, u0 = eng.aim_rays(rec)
    A, P = None, None
    try:
        A, P = eng.empty((N,)), eng.empty((N, 3))
        eng.trace_opd(t_after, y0, u0, spec, A, P, N=N, clip=True, rot0=rot_after, exact=exact)
        return eng.opd_points(A, P, ref, wl/system.scale)
    finally:
        for a in (y0, u0, A, P):
            if a is not None:
                a.free()


def opds(system, heights=(0., .707, 1.), wavelength=None, nrays=1000, distribution="hexapolar",
         pad=4, resample=4, triangulation="device", download=False, engine=None, exact=False):
    """Analysis.opds (rayopt/analysis.py:285-352) on the device for a rayopt
    ``System``.  For each height the pupil is aimed on the host
    (``system.pupil``, the heights in Analysis's order, last to first), the
    launch rays of ``rays_point(clip=True)`` are generated in HBM and
    marched with clipping; no trace is stored.

    - Contour OPD: ``opd()``'s default reference sphere, the finite points
      regridded on ``int(resample*N**.5)`` nodes per axis (N the ray count)
      and reduced to ``ptp`` and ``max_abs`` (max |o|) of the finite nodes.
    - PSF: ``psf()``'s sphere of radius ``system[-1].distance``, then the
      PSF and its encircled energy and MTFs, as
      ``ResidentMixin.psf_profiles`` returns them (stats, x0, y0, dx,
      center, xe, ee, of, mtf).

    Heights run one after another and each frees its device arrays before
    the next.  Returns a dict: heights, wavelength, results (one dict per
    height, None where no ray made it through, as Analysis skips it; with
    `download` each also holds the numpy grids ``opd`` and ``psf``), airy
    (the radius of Analysis's circle), and mm and rm, the contour range and
    PSF axis limit Analysis takes from the last height with rays."""
    from .rays import aim_record, grid_spec
    from .surface_table import pack_system
    check_triangulation(triangulation)
    eng = engine or default_engine()
    wl = system.wavelengths[0] if wavelength is None else wavelength
    ref, grid = grid_spec(distribution, nrays)
    if grid is None:
        raise ValueError("distribution %r with %d rays is not generated on the device"
                         % (distribution, nrays))
    L = len(system)
    after, image = L - 2, L - 1
    n0 = system.refractive_index(wl, 0)
    table, n_rows, rot0 = pack_system(system, wl, 1, None, n0=n0)
    n = np.r_[n0, n_rows]
    results = []
    # Analysis walks the heights from the last to the first, and what
    # System.pupil returns depends on the calls before it: aim in that order
    for height in reversed(heights):
        yo = (0, height)
        zp, p = system.pupil(yo, l=wl)
        rec = aim_record(system.object, yo, zp, p, grid, False, system[0])
        N = eng.aim_count(rec)
        cy, cu = eng.aim_rays(rec, first=ref, count=1)
        try:
            y0_ref, u0_ref = cy.download()[0], cu.download()[0]
        finally:
            cy.free(), cu.free()
        Y = eng.trace(table, y0_ref[None], u0_ref[None], clip=True, rot0=rot0, keep_last=True,
                      exact=exact, want=("y",))[0]
        y_ref = (y0_ref, u0_ref, Y[0, 0])
        m = int(resample*N**.5)
        pts = _points(eng, system, wl, rec, N, n, ref, y_ref, after, image, None, exact)
        if not pts[2]:
            pts[0].free(), pts[1].free()
            results.append(None)
            continue
        xs, _, o = regrid(eng, *pts, m, False, triangulation)
        try:
            count, lo, hi = eng.grid_range(o)
            r = dict(ptp=hi - lo, max_abs=max(abs(lo), abs(hi)), count=count)
            if download:
                r["opd"] = o.download()
        finally:
            o.free()
        radius = system[-1].distance
        pts = _points(eng, system, wl, rec, N, n, ref, y_ref, after, image, radius, exact)
        xs, _, o = regrid(eng, *pts, m, False, triangulation)
        pp, _, out, st = psf_of_grid(eng, xs, o, pad, wl/system.scale, radius)
        if download:
            try:
                r["psf"] = out.download()
            except Exception:
                out.free()
                raise
        r.update(psf_profiles(eng, pp, out, st))
        results.append(r)
    results.reverse()
    paraxial = system.paraxial
    mm, rm = scales(results)
    return dict(heights=list(heights), wavelength=wl, results=results,
                airy=paraxial.airy_radius[1]/paraxial.wavelength*wl, mm=mm, rm=rm)
