"""The extended-precision geometric OTF oracle (oracle/otf_oracle.py) and the
host checks of otf_spec.  No GPU.

The oracle is pinned to mpmath at 40 digits at phases up to 1e3 cycles, and
to the identities the definition implies: S(0) = n, the shift theorem,
conjugate symmetry and the count of finite points."""
import numpy as np
import pytest

import otf_oracle
from rayopt_b200.engine import otf_spec


def _rows(n, seed, spread=1.):
    rng = np.random.default_rng(seed)
    y = np.c_[rng.normal(0, spread, (n, 2)), np.zeros(n)]
    u = rng.normal(0, .05, (n, 2))
    return y, np.c_[u, np.sqrt(1 - np.square(u).sum(1))]


def _dyadic_rows(n, seed):
    """rows on a coarse dyadic grid with i_z = 1: every operation of the
    points is exact, so shifting c or flipping signs moves q exactly"""
    rng = np.random.default_rng(seed)
    y = np.c_[rng.integers(-2**10, 2**10, (n, 2))/2.**8, np.zeros(n)]
    inc = np.c_[rng.integers(-2**6, 2**6, (n, 2))/2.**8, np.ones(n)]
    return y, inc


def _S(re, im):
    return re.astype(np.float64) + 1j*im.astype(np.float64)


def _mp(mpmath, x):
    """a long double as an mpf, exactly (its 64-bit significand is two doubles)"""
    hi = np.float64(x)
    return mpmath.mpf(float(hi)) + mpmath.mpf(float(np.float64(x - hi)))


def test_against_mpmath():
    mpmath = pytest.importorskip("mpmath")
    mpmath.mp.dps = 40
    y, inc = _rows(300, 1, spread=1.)
    z, dnu, F = np.array([0., .3]), 1000/3./6, 7                # nu_6 |q| up to ~1e3 cycles
    c = (.1, -.2)
    re, im, n, phi = otf_oracle.otf(y, inc, c, z, dnu, F)
    assert phi.max() > 300 and phi.max() < 2000
    q = __import__("spot_oracle").points(y, inc, c, z)
    nu = otf_oracle.freqs(dnu, F)
    for k in range(len(z)):
        for a in range(2):
            for j in range(F):
                sr, si = mpmath.mpf(0), mpmath.mpf(0)
                for x in q[k, :, a]:
                    t = 2*mpmath.pi*mpmath.mpf(float(nu[j]))*mpmath.mpf(float(x))
                    sr += mpmath.cos(t)
                    si -= mpmath.sin(t)
                err = max(abs(float(sr - _mp(mpmath, re[k, a, j]))),
                          abs(float(si - _mp(mpmath, im[k, a, j]))))
                assert err <= 1e-15*n[k], (k, a, j, err/n[k])
                assert err <= otf_oracle.oracle_error(n, phi)[k]


def test_zero_frequency_is_the_count():
    y, inc = _rows(5000, 2)
    y[::7, 0] = np.nan
    re, im, n, _ = otf_oracle.otf(y, inc, (0., 0.), np.linspace(-.1, .1, 3), .37, 5)
    assert (n == 5000 - len(y[::7])).all()
    assert (re[..., 0] == n[:, None]).all() and (im[..., 0] == 0).all()


def test_shift_theorem():
    y, inc = _dyadic_rows(4000, 3)
    z, dnu, F, delta = np.array([0., .5, -1.]), 3.1, 33, np.array([.125, -.375])
    a = otf_oracle.otf(y, inc, (0., 0.), z, dnu, F)
    b = otf_oracle.otf(y, inc, delta, z, dnu, F)
    nu = otf_oracle.freqs(dnu, F)
    want = _S(a[0], a[1])*np.exp(2j*np.pi*nu[None, None, :]*delta[None, :, None])
    tol = otf_oracle.oracle_error(a[2], a[3]) + 4e-16*np.abs(nu*delta[:, None]).max()*a[2]
    assert np.abs(_S(b[0], b[1]) - want).max() <= tol.max()
    assert np.array_equal(a[2], b[2])


def test_negated_points_give_the_conjugate():
    y, inc = _dyadic_rows(3000, 4)
    z, o = np.array([0., .25]), np.array([[.5, -.25], [0., .125]])
    a = otf_oracle.otf(y, inc, (.25, .5), z, 2.7, 17, o)
    inc_n = inc.copy()
    inc_n[:, :2] *= -1
    b = otf_oracle.otf(-y, inc_n, (-.25, -.5), z, 2.7, 17, -o)
    tol = otf_oracle.oracle_error(a[2], a[3]).max()
    assert np.abs(_S(b[0], b[1]) - np.conj(_S(a[0], a[1]))).max() <= tol


def test_non_finite_points_are_not_counted():
    y, inc = _rows(2000, 5)
    bad_y = np.array([[np.nan, 0, 0], [np.inf, 0, 0], [0, -np.inf, 0], [0, 0, 0], [.1, .1, 0]])
    bad_i = np.array([[0, 0, 1]]*3 + [[0, 0, 0], [.1, .1, 0]])   # i_z = 0: 0/0 and .1/0
    z = np.array([0., .1])
    a = otf_oracle.otf(y, inc, (0., 0.), z, 1.3, 9)
    b = otf_oracle.otf(np.r_[bad_y[:2], y, bad_y[2:]], np.r_[bad_i[:2], inc, bad_i[2:]],
                       (0., 0.), z, 1.3, 9)
    # one non-finite component is enough; u = 0/0 or .1/0 gives NaN even at z = 0 (0*inf)
    q = __import__("spot_oracle").points(bad_y, bad_i, (0., 0.), z)
    assert np.isfinite(q).any() and not np.isfinite(q).all(2).any()
    assert np.array_equal(b[2], a[2]) and (a[2] == 2000).all()
    assert np.array_equal(b[0], a[0]) and np.array_equal(b[1], a[1])


@pytest.mark.parametrize("bad", [
    dict(z=()), dict(z=np.zeros(17)), dict(nfreq=0), dict(nfreq=257), dict(dnu=np.nan),
    dict(dnu=np.inf), dict(c=(np.nan, 0.)), dict(c=(0., -np.inf)), dict(z=(0., np.nan)),
    dict(offsets=((0., 0.), (np.inf, 0.)))])
def test_otf_spec_refuses(bad):
    ok = dict(z=(0., .1), dnu=.5, nfreq=64, c=(0., 0.))
    kw = dict(ok, **bad)
    if "offsets" in bad:
        kw["z"] = (0., .1)
    with pytest.raises(ValueError):
        otf_spec(**kw)


def test_otf_spec_record():
    rec = otf_spec((0., .1, -.2), .25, 256, (1., 2.), ((0., 1.), (2., 3.), (4., 5.)))
    s = rec[0]
    assert (s["planes"], s["nfreq"], s["dnu"]) == (3, 256, .25)
    assert np.array_equal(s["z"][:3], (0., .1, -.2)) and not s["z"][3:].any()
    assert np.array_equal(s["o"][:3], ((0., 1.), (2., 3.), (4., 5.))) and not s["o"][3:].any()
    otf_spec(np.zeros(16), 0., 1, (0., 0.))                 # the limits are accepted
