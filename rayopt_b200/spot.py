"""Through-focus spot images on the device: Analysis.spots
(rayopt/analysis.py:250-283) with the scatter plot of each defocus plane
replaced by an exact integer histogram (a geometric PSF) of every ray.

Each ray's point at plane k is ``q = (y_xy - c + z_k i_xy/i_z) - o_k`` (c the
chief ray's intercept), binned as ``np.histogram2d`` -- or its radius as
``np.histogram`` -- of the same points would bin it (include/rtx.h,
rtx_trace_spot).  Counts are integers, so they are the same in every call and
add exactly over chunks and wavelengths.
"""
import numpy as np

from .engine import default_engine, spot_spec, spot_shape

# half-width of the default range when the rays give none: no finite point,
# or every point on the centre (one ray in focus); in the system's length unit
DEFAULT_HALF_WIDTH = 1e-3


def _bins(bins, radial):
    b = [int(v) for v in np.atleast_1d(bins)]
    if radial:
        return (b[0],)
    return (b[0], b[0]) if len(b) == 1 else (b[0], b[1])


def default_range(extent, bins, radial=False):
    """The range that contains every finite point of the extents (K,3) a
    launch returned: ``[-h, h]`` on both axes with h the largest |q_x|, |q_y|
    over the planes (radial: ``[0, max r]``); ``DEFAULT_HALF_WIDTH`` when h is
    0, not finite or too small for a normal bin width"""
    ext = np.asarray(extent, np.float64)
    h = float(ext[:, 2].max() if radial else ext[:, :2].max()) if ext.size else 0.
    if not (np.isfinite(h) and 2*h/max(bins) >= np.finfo(np.float64).tiny):
        h = DEFAULT_HALF_WIDTH
    return ((0., h),) if radial else ((-h, h), (-h, h))


def spot_edges(range, bins, radial=False):
    """np.histogram2d's / np.histogram's bin edges: one np.linspace per axis"""
    return [np.linspace(lo, hi, n + 1) for (lo, hi), n in zip(range, _bins(bins, radial))]


def _range(range, radial):
    r = np.asarray(range, np.float64).reshape(-1, 2)
    return tuple((float(lo), float(hi)) for lo, hi in r[:1 if radial else 2])


def spot_images(eng, bundles, defocus=(0.,), bins=(256, 256), range=None, radial=False,
                offsets=None, download=True):
    """Bin several bundles at the planes `defocus` with one shared range.

    `bundles`: a list of (center, parts), `center` the bundle's chief
    intercept (2,) (NaN: nothing is counted) and `parts` callables
    ``part(spec, counts, extent) -> (tally, extent)`` that each bin one piece
    of the bundle's rays (Engine.trace_spot or Engine.spot_rows).  With
    ``range=None`` one extent-only pass over every part picks
    ``default_range``.  Returns a dict with z (K,), counts (B, K, nx, ny) or
    (B, K, nx) uint64 (a list of DeviceArrays when ``download=False``),
    edges, range and tally (B, K, 2): rays binned, rays with a non-finite
    point."""
    z = np.atleast_1d(np.asarray(defocus, np.float64))
    nb = _bins(bins, radial)
    if range is None:
        probe = ((-1., 1.),) if radial else ((-1., 1.), (-1., 1.))
        ext = np.zeros((len(z), 3))
        for c, parts in bundles:
            spec = spot_spec(z, nb, probe, c, radial, offsets)
            for part in parts:
                ext = np.maximum(ext, part(spec, None, True)[1])
        range = default_range(ext, nb, radial)
    range = _range(range, radial)
    counts, tally = [], np.zeros((len(bundles), len(z), 2), np.uint64)
    for b, (c, parts) in enumerate(bundles):
        spec = spot_spec(z, nb, range, c, radial, offsets)
        dev = eng.empty(spot_shape(spec), np.uint64)
        eng.memset(dev, 0)
        for part in parts:
            tally[b] += part(spec, dev, False)[0]
        if download:
            counts.append(dev.download())
            dev.free()
        else:
            counts.append(dev)
    if download:
        counts = np.stack(counts) if counts else np.zeros((0,) + spot_shape(spec), np.uint64)
    return dict(z=z, counts=counts, edges=spot_edges(range, nb, radial), range=range, tally=tally)


def spots(system, heights=(1., .707, 0.), wavelengths=None, nrays=150, distribution="hexapolar",
          defocus=5, bins=(256, 256), range=None, radial=False, chunk=2**26, engine=None,
          exact=False):
    """Analysis.spots (rayopt/analysis.py:250-283) on the device for a rayopt
    ``System``: for each height x wavelength the pupil is aimed on the host
    (``system.pupil``), the launch rays are generated in HBM in chunks of at
    most `chunk` rays (rtx_aim_rays) and each chunk is marched to the image
    with clipping and binned as it arrives (rtx_trace_spot) -- no trace is
    stored, so memory is bounded by `chunk`.  The planes are
    ``(arange(defocus) - defocus//2) * paraxial.rayleigh_range[1]`` and the
    centre is each bundle's chief ray, as in Analysis; one range serves every
    bundle, as Analysis shares its axes.

    Returns a dict: z (K,), counts (H, W, K, nx, ny) (radial: (H, W, K, nx))
    uint64, edges, range, airy (W,) the radii of Analysis's circles, tally
    (H, W, K, 2)."""
    from .rays import aim_record, grid_spec
    from .surface_table import pack_system
    eng = engine or default_engine()
    paraxial = system.paraxial
    wavelengths = list(system.wavelengths if wavelengths is None else wavelengths)
    heights = list(heights)
    z = (np.arange(defocus) - defocus//2)*paraxial.rayleigh_range[1]
    ref, grid = grid_spec(distribution, nrays)
    if grid is None:
        raise ValueError("distribution %r with %d rays is not generated on the device"
                         % (distribution, nrays))
    chunk = int(chunk)
    if chunk < 1:
        raise ValueError("chunk must be >= 1")
    plans = []
    for hi in heights:
        for wi in wavelengths:
            yo = (0, hi)
            zp, p = system.pupil(yo, l=wi)
            rec = aim_record(system.object, yo, zp, p, grid, False, system[0])
            table, _, rot0 = pack_system(system, wi, 1, None, n0=system.refractive_index(wi, 0))
            plans.append((rec, eng.aim_count(rec), table, rot0))
    cap = min(chunk, max([n for _, n, _, _ in plans] + [1]))
    y0, u0 = eng.empty((cap, 3)), eng.empty((cap, 3))
    try:
        def part(rec, table, rot0, first, count):
            def run(spec, counts, extent):
                eng.aim_rays_into(rec, y0, u0, count, first=first)
                return eng.trace_spot(table, y0, u0, spec, counts, N=count, clip=True, rot0=rot0,
                                      exact=exact, extent=extent)
            return run

        bundles = []
        for rec, n, table, rot0 in plans:
            cy, cu = eng.aim_rays(rec, first=ref, count=1)
            Y = eng.trace(table, cy.download(), cu.download(), clip=True, rot0=rot0,
                          keep_last=True, exact=exact, want=("y",))[0]
            cy.free(), cu.free()
            bundles.append((Y[0, 0, :2], [part(rec, table, rot0, int(f), int(min(chunk, n - f)))
                                          for f in np.arange(0, n, chunk)]))
        out = spot_images(eng, bundles, z, bins, range, radial)
    finally:
        y0.free(), u0.free()
    out["counts"] = out["counts"].reshape((len(heights), len(wavelengths)) + out["counts"].shape[1:])
    out["tally"] = out["tally"].reshape(len(heights), len(wavelengths), len(z), 2)
    out["airy"] = paraxial.airy_radius[1]/paraxial.wavelength*np.asarray(wavelengths, np.float64)
    return out
