"""rtx_psf against the same PSF computed in extended precision: the pupil
function exp(-2 pi i o)/sqrt(#finite) and scipy.fft.fft2 in long double
(64-bit significand on x86-64), at the grid sizes the OPD path picks
(n = int(4 sqrt(nrays)): 282 = 6 47, 1264 = 16 79, 1788 = 12 149) and a prime
one, with zero padding 1 to 4 and an odd padded size.

Bounds, with eps = 2^-52 (DESIGN.md 3.8): measured on one H100 80GB HBM3 and
set a few times above the largest error seen, except Parseval's, which is
derived (every |z|^2 is 1/count, so sum psf = 1 up to the FFT's rounding,
O(eps log2 nx))."""
import math

import numpy as np
import pytest
import scipy.fft

from test_gpu_psf import pupil_opd

pytestmark = pytest.mark.gpu

PEAK_BOUND = 32       # max |psf - psf_ld| <= PEAK_BOUND eps max psf_ld
SUM_BOUND = 4         # |sum - fsum(psf_ld)| <= SUM_BOUND eps log2(nx) sum
MAX_BOUND = 32        # |max - max psf_ld| <= MAX_BOUND eps max psf_ld
MOMENT_BOUND = 4      # |sum psf k - fsum(psf_ld k)| <= MOMENT_BOUND eps log2(nx) sum max|k|
PARSEVAL_BOUND = 4    # |sum - 1| <= PARSEVAL_BOUND eps log2(nx)

EPS = np.finfo(np.float64).eps
PI = np.longdouble("3.14159265358979323846264338327950288")


@pytest.fixture(scope="module")
def eng():
    from rayopt_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def psf_long(o, pad):
    """|fft2(z)|^2/nx^2 of the zero-padded pupil function, in long double"""
    n = o.shape[0]
    nx = pad*n
    good = np.isfinite(o)
    a = -2*PI*o[good].astype(np.longdouble)
    z = np.zeros((nx, nx), np.clongdouble)
    z[:n, :n][good] = (np.cos(a) + 1j*np.sin(a))/np.sqrt(np.longdouble(good.sum()))
    f = scipy.fft.fft2(z, overwrite_x=True)
    del z
    return (f.real*f.real + f.imag*f.imag)/np.longdouble(nx*nx)


def fsum(a):
    return math.fsum(np.asarray(a, np.float64).ravel().tolist())


@pytest.mark.parametrize("n,pad", [(126, 4), (282, 1), (282, 3), (251, 3), (1264, 2),
                                   (1788, 1), (4099, 1)])
def test_psf_vs_long_double(eng, n, pad):
    if np.finfo(np.longdouble).nmant < 63:
        pytest.skip("long double is not extended precision here")
    _, o = pupil_opd(n, 100 + n + pad)
    od = eng.to_device(o)
    try:
        out, raw = eng.psf(od, pad)
    finally:
        od.free()
    psf = out.download()
    out.free()
    nx = n*pad
    want = psf_long(o, pad)
    peak = want.max()
    err = float(np.abs(psf - want).max()/peak)
    assert err <= PEAK_BOUND*EPS, err
    L = math.log2(nx)
    k = np.fft.fftfreq(nx, 1./nx)              # the signed frequency index
    s_ld = fsum(want)
    assert int(raw[0]) == np.isfinite(o).sum()
    d_sum = abs(raw[1] - s_ld)/s_ld
    d_max = abs(raw[2] - float(peak))/float(peak)
    d_mom = max(abs(raw[3] - fsum(want*k[:, None])), abs(raw[4] - fsum(want*k[None, :]))) \
        / (s_ld*np.fabs(k).max())
    parseval = abs(raw[1] - 1.)
    assert d_sum <= SUM_BOUND*EPS*L, d_sum
    assert d_max <= MAX_BOUND*EPS, d_max
    assert d_mom <= MOMENT_BOUND*EPS*L, d_mom
    assert parseval <= PARSEVAL_BOUND*EPS*L, parseval
    print("n=%d pad=%d nx=%d: max|dpsf|/peak %.2f eps, sum %.2f eps log2(nx), max %.2f eps, "
          "moments %.2f eps log2(nx), |sum - 1| %.2f eps log2(nx)"
          % (n, pad, nx, err/EPS, d_sum/(EPS*L), d_max/EPS, d_mom/(EPS*L), parseval/(EPS*L)))
