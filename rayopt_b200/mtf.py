"""Geometric MTF through focus and across the field on the device.

The geometric OTF is the Fourier transform of the spot diagram:
``OTF(nu) = mean over the rays of exp(-2 pi i nu q)``, q a ray's point at a
defocus plane about a centre, along x (sagittal for fields along y) or y
(tangential).  Its only error is ray sampling, and the engine traces 1e7 -
1e8 rays in milliseconds, so the direct sum over every ray
(rtx_otf_rows, include/rtx.h) replaces a spot-diagram FFT.
"""
import numpy as np

from .engine import OTF_MAX_FREQS, default_engine, otf_spec


def _otf(S, count):
    """S / count per plane (NaN where nothing counted)"""
    with np.errstate(invalid="ignore", divide="ignore"):
        return S/np.asarray(count, np.float64)[..., None, None]


def default_dnu(system, nfreq):
    """The frequency step whose last frequency is 1/airy_radius of the
    primary wavelength: the MTF axis Analysis.opds draws"""
    return 1/system.paraxial.airy_radius[1]/max(int(nfreq) - 1, 1)


def geometric_mtf(system, heights=(0., .707, 1.), wavelengths=None, nrays=10**6,
                  distribution="hexapolar", defocus=(0.,), dnu=None, nfreq=64,
                  spectral_weights=None, chunk=2**24, engine=None, exact=False,
                  dtype=np.float64):
    """Geometric OTF and MTF of a rayopt ``System`` at each height x
    wavelength and defocus plane.

    For each height and wavelength the pupil is aimed on the host
    (``system.pupil``), the launch rays are generated in HBM in chunks of at
    most `chunk` rays (rtx_aim_rays), each chunk is marched to the image with
    clipping, keeping only the last surface (rtx_trace), and its OTF sums are
    taken on the device (rtx_otf_rows); the chunk sums are added on the host
    in chunk order.  Memory is bounded by `chunk`, and the chunking changes
    only the last bits, within the bound of include/rtx.h.

    The centre of every wavelength of a height is the chief ray of
    ``wavelengths[0]``, so the polychromatic OTF carries lateral colour; a
    vignetted chief ray counts nothing and gives NaN.  `defocus` are the
    plane distances from the image surface; Analysis's through-focus planes
    are ``(arange(n) - n//2)*system.paraxial.rayleigh_range[1]``.  The
    frequencies are ``arange(nfreq)*dnu`` in cycles per length unit;
    ``dnu=None`` ends them at 1/airy_radius of the primary wavelength, the
    MTF axis of Analysis.opds.

    Returns a dict: freq (F,), z (K,), otf complex (H, W, K, 2, F) (axis 0:
    x, 1: y), mtf = |otf|, count (H, W, K) int64, poly (H, K, 2, F) the
    `spectral_weights`-weighted mean (equal weights by default) of the OTFs
    of the wavelengths that count rays at that plane, heights,
    wavelengths."""
    from .rays import aim_record, grid_spec
    from .surface_table import pack_system
    eng = engine or default_engine()
    wavelengths = list(system.wavelengths if wavelengths is None else wavelengths)
    heights = list(heights)
    z = np.atleast_1d(np.asarray(defocus, np.float64))
    F = int(nfreq)
    dnu = default_dnu(system, F) if dnu is None else float(dnu)
    otf_spec(z, dnu, F, (0., 0.))                     # refuse a bad spec before any work
    weights = np.ones(len(wavelengths)) if spectral_weights is None else \
        np.asarray(spectral_weights, np.float64).reshape(len(wavelengths))
    ref, grid = grid_spec(distribution, nrays)
    if grid is None:
        raise ValueError("distribution %r with %d rays is not generated on the device"
                         % (distribution, nrays))
    chunk = int(chunk)
    if chunk < 1:
        raise ValueError("chunk must be >= 1")
    H, W, K = len(heights), len(wavelengths), len(z)
    plans = []
    for hi in heights:
        for wi in wavelengths:
            yo = (0, hi)
            zp, p = system.pupil(yo, l=wi)
            rec = aim_record(system.object, yo, zp, p, grid, False, system[0])
            table, _, rot0 = pack_system(system, wi, 1, None, n0=system.refractive_index(wi, 0))
            plans.append((rec, eng.aim_count(rec), table, rot0))
    cap = min(chunk, max([n for _, n, _, _ in plans] + [1]))
    ld = (cap + 63)//64*64
    S = np.zeros((H, W, K, 2, F), np.complex128)
    count = np.zeros((H, W, K), np.int64)
    bufs = [eng.empty((cap, 3), dtype), eng.empty((cap, 3), dtype),
            eng.empty((1, ld, 3), dtype), eng.empty((1, ld, 3), dtype)]
    y0, u0, Y, I = bufs
    try:
        for h in range(H):
            c = None
            for w in range(W):
                rec, n, table, rot0 = plans[h*W + w]
                if c is None:                          # the chief ray of wavelengths[0]
                    cy, cu = eng.aim_rays(rec, first=ref, count=1)
                    c = eng.trace(table, cy.download(), cu.download(), clip=True, rot0=rot0,
                                  keep_last=True, exact=exact, want=("y",))[0][0, 0, :2]
                    cy.free(), cu.free()
                    if not np.isfinite(c).all():
                        break
                    spec = otf_spec(z, dnu, F, c)
                for first in range(0, n, chunk):
                    m = min(chunk, n - first)
                    eng.aim_rays_into(rec, y0, u0, m, first=first)
                    eng.trace_device(table, y0, u0, Y, None, I, None, N=m, ld=ld, clip=True,
                                     keep_last=True, rot0=rot0, exact=exact)
                    s, k = eng.otf_rows(Y.rows(0), I.rows(0), spec, N=m)
                    S[h, w] += s
                    count[h, w] += k
    finally:
        for a in bufs:
            a.free()
    otf = _otf(S, count)
    return dict(freq=np.arange(F)*dnu, z=z, otf=otf, mtf=np.abs(otf), count=count,
                poly=poly_otf(otf, count, weights), heights=heights, wavelengths=wavelengths)


def poly_otf(otf, count, weights):
    """(H, K, 2, F): the weighted mean over the wavelengths (axis 1) of the
    OTFs (H, W, K, 2, F), each plane over the wavelengths with count > 0
    (NaN where none counts)"""
    wk = np.where(np.asarray(count) > 0, np.asarray(weights, np.float64)[:, None], 0.)
    num = np.einsum("hwk,hwkaf->hkaf", wk, np.where(wk[..., None, None] > 0, otf, 0))
    with np.errstate(invalid="ignore", divide="ignore"):
        return num/wk.sum(1)[..., None, None]


def _check_freqs(freqs):
    nu = np.ascontiguousarray(np.atleast_1d(np.asarray(freqs, np.float64)))
    if nu.ndim != 1 or not 1 <= len(nu) <= OTF_MAX_FREQS or not np.isfinite(nu).all():
        raise ValueError("need 1..%d finite frequencies, got %r" % (OTF_MAX_FREQS, freqs))
    return nu


def _spectral(spectral_weights, W):
    if spectral_weights is None:
        return np.ones(W)
    sw = np.asarray(spectral_weights, np.float64)
    if sw.size != W or not np.isfinite(sw).all():
        raise ValueError("spectral_weights must be %d finite values, got %r" % (W, spectral_weights))
    return sw.reshape(W)
