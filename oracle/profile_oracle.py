"""numpy statement of the encircled energy and MTF that Analysis.opds takes
from a PSF (rayopt/analysis.py:319-346), the yardstick of rtx_psf_profiles /
ResidentMixin.psf_profiles.

* ``polar_sum_azimuthal``: special_sums.polar_sum(m, center, "azimuthal")
  (rayopt/special_sums.py:240-263) with aspect 1 and binsize 1, restated so
  that it runs on NumPy 2: ``int`` for the removed ``np.int`` and
  ``minlength=0`` where the reference passes None.  Same operations, same
  order: bincount's weighted sums run over the pixels in row-major order.
* ``profiles``: Analysis.opds from (p, q, psf) of ``psf()`` on.
"""
import numpy as np

import psf_oracle


def polar_sum_azimuthal(m, center):
    """sum of m over the bins trunc(sqrt((j - c1)^2 + (i - c0)^2))"""
    m = np.atleast_2d(m)
    i, j = np.ogrid[:m.shape[0], :m.shape[1]]
    i, j = i - center[0], j - center[1]
    k = (j**2*1.**2 + i**2)**.5
    k = (k/1.).astype(int)
    return np.bincount(k.ravel(), m.ravel(), 0)


def line_sums(psf):
    """the column and row sums of the stored (FFT-order) PSF, as Analysis
    forms them: ifftshift(fftshift(psf).sum(i)), i = 0, 1"""
    s = np.fft.fftshift(psf)
    return np.fft.ifftshift(s.sum(0)), np.fft.ifftshift(s.sum(1))


def profiles(p, q, psf, x0=None, y0=None):
    """analysis.py:319-346 on the (p, q, psf) of ``psf()``: the centroid
    (x0, y0) (or the one given), dx of the fftshifted p axis after the
    centroid is subtracted, the radial bins about (nx/2 + x0/dx, ny/2 + y0/dx),
    their cumulative sum ee on the radii xe, and for i = 0, 1 the MTF
    |ifft(ifftshift(psf.sum(i)) size^.5)| on the first half of
    fftfreq(n, dx).  The PSF is taken square, as psf() makes it: one
    frequency axis ``of`` serves both curves."""
    stats = psf_oracle.stats(p, q, psf)
    x, y, psf = map(np.fft.fftshift, (p, q, psf))
    if x0 is None:
        x0 = (psf*x).sum()
    if y0 is None:
        y0 = (psf*y).sum()
    x, y = x - x0, y - y0
    dx = x[1, 0] - x[0, 0]
    center = (psf.shape[0]/2 + x0/dx, psf.shape[1]/2 + y0/dx)
    bins = polar_sum_azimuthal(psf, center)
    ee = np.cumsum(bins)
    xe = np.arange(ee.size)*dx
    mtf = []
    for i in range(2):
        ot = np.fft.ifft(np.fft.ifftshift(psf.sum(i))*psf.size**.5)
        of = np.fft.fftfreq(ot.size, dx)
        ot, of = ot[:ot.size//2], of[:of.size//2]
        mtf.append(np.absolute(ot))
        if i == 0:
            of0 = of
    return dict(stats=stats, x0=x0, y0=y0, dx=dx, center=center, bins=bins, xe=xe, ee=ee,
                of=of0, mtf=tuple(mtf))
