"""The spot-image oracle (oracle/spot_oracle.py) against numpy's own
histograms and the reference's own expressions, and the spot entry points'
argument checks.  CPU only."""
import ctypes as C
import warnings

import numpy as np
import pytest

import ref_shim
import spot_oracle
from rayopt_b200 import _lib, build
from rayopt_b200.engine import SPOT_DTYPE, spot_spec

RANGES = [(-0.3, 0.7, 7), (0.0, 1.0, 1), (-1e-3, 2e-3, 13), (-5.0, 5.0, 256), (0.1, 0.3, 3)]


def _adversarial(lo, hi, n, seed=0):
    """every edge, 1 ulp either side of it, the range ends, -0.0, NaN, +-inf
    and random points inside and just outside"""
    e = spot_oracle.edges(lo, hi, n)
    x = np.concatenate([e, np.nextafter(e, -np.inf), np.nextafter(e, np.inf),
                        [lo, hi, -0.0, 0.0, np.nan, np.inf, -np.inf],
                        np.random.default_rng(seed).uniform(lo - (hi - lo)*.1,
                                                            hi + (hi - lo)*.1, 200)])
    return x


@pytest.mark.parametrize("lo,hi,n", RANGES)
def test_bin_index_is_numpy_histogram_per_point(lo, hi, n):
    """each adversarial point alone: the oracle's bin is the one
    np.histogram puts it in (or none)"""
    for x in _adversarial(lo, hi, n):
        h, _ = np.histogram([x], bins=n, range=(lo, hi))
        want = int(np.flatnonzero(h)[0]) if h.any() else -1
        assert spot_oracle.bin_index(np.array([x]), lo, hi, n)[0] == want, (x, lo, hi, n)


@pytest.mark.parametrize("lo,hi,n", RANGES)
def test_histogram1d_equals_numpy(lo, hi, n):
    x = _adversarial(lo, hi, n, 1)
    want, edges = np.histogram(x, bins=n, range=(lo, hi))
    assert np.array_equal(spot_oracle.histogram1d(x, n, (lo, hi)), want)
    assert np.array_equal(spot_oracle.edges(lo, hi, n), edges)


@pytest.mark.parametrize("i,j", [(0, 1), (2, 0), (3, 4), (1, 1), (4, 2)])
def test_histogram2d_equals_numpy(i, j):
    """all pairs of two adversarial sets, nx != ny and n = 1 among them"""
    (xl, xh, nx), (yl, yh, ny) = RANGES[i], RANGES[j]
    xs, ys = np.meshgrid(_adversarial(xl, xh, nx, 2), _adversarial(yl, yh, ny, 3))
    xs, ys = xs.ravel(), ys.ravel()
    want, ex, ey = np.histogram2d(xs, ys, bins=(nx, ny), range=((xl, xh), (yl, yh)))
    got = spot_oracle.histogram(xs, ys, (nx, ny), ((xl, xh), (yl, yh)))
    assert got.dtype == np.uint64 and np.array_equal(got, want)
    assert np.array_equal(ex, spot_oracle.edges(xl, xh, nx))
    assert np.array_equal(ey, spot_oracle.edges(yl, yh, ny))


def test_spot_tallies_and_extent():
    """tallies count binned and non-finite points per plane; the extent is
    over the finite points only, 0 when there is none"""
    y = np.array([[0., 0., 0.], [1., 0., 0.], [np.nan, 0., 0.], [0., .5, 0.]])
    inc = np.array([[0., 0., 1.], [.1, 0., 1.], [0., 0., 1.], [.1, .1, 0.]])   # i_z = 0: inf
    counts, tally, ext = spot_oracle.spot(y, inc, (0., 0.), (0., 1.), (4, 4),
                                          ((-.5, .5), (-.5, .5)))
    assert counts.shape == (2, 4, 4) and counts.sum() == 2
    assert tally.tolist() == [[1, 2], [1, 2]]      # ray 1 outside the range; 0*inf is NaN too
    assert np.array_equal(ext, [[1., 0., 1.], [1.1, 0., 1.1]])
    _, tally, ext = spot_oracle.spot(y[2:3], inc[2:3], (0., 0.), (0.,), (4,), ((0., 1.),),
                                     radial=True)
    assert tally.tolist() == [[0, 1]] and not ext.any()


@pytest.mark.skipif(not ref_shim.available(), reason="reference tree not present")
@pytest.mark.parametrize("name", ["cooke", "double_gauss"])
def test_points_are_the_references_expressions(name):
    """analysis.py:266-280 restated on the reference's own GeometricTrace rows
    and rayopt.utils.tanarcsin (analysis.py itself imports matplotlib)"""
    import yaml
    import systems_yaml
    R = ref_shim.load()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        s = R.System(**yaml.safe_load(systems_yaml.SYSTEMS[name]))
        s.update()
        s.paraxial.refocus()
        z = (np.arange(5) - 5//2)*s.paraxial.rayleigh_range[1]
        for hi in (1., .707, 0.):
            t = R.GeometricTrace(s)
            t.rays_point((0, hi), s.wavelengths[0], nrays=150, distribution="hexapolar", clip=True)
            y = t.y[-1, :, :2] - t.y[-1, t.ref, :2]
            u = R.utils.tanarcsin(t.i[-1])
            want = np.stack([y + zi*u for zi in z])
            got = spot_oracle.points(t.y[-1], t.i[-1], t.y[-1, t.ref, :2], z)
            assert np.array_equal(got, want, equal_nan=True), (name, hi)


# ---- the C entry points' argument checks (no device needed)
@pytest.fixture(scope="module")
def lib():
    build.build()
    return _lib.load()


def test_spot_symbols_and_layout(lib):
    for name in ("rtx_sizeof_spot", "rtx_trace_spot", "rtx_spot_rows"):
        assert name in _lib.SYMBOLS and hasattr(lib, name)
    assert lib.rtx_sizeof_spot() == SPOT_DTYPE.itemsize == 456


def _bad_specs():
    ok = dict(z=(0., 1.), bins=(8, 4), range=((-1., 1.), (-2., 2.)), center=(0., 0.))
    yield "K = 0", dict(ok, z=())
    yield "K = 17", dict(ok, z=np.zeros(17))
    yield "nx = 0", dict(ok, bins=(0, 4))
    yield "ny = 0", dict(ok, bins=(8, 0))
    yield "radial ny = 2", dict(ok, bins=(8, 2), range=((0., 1.),), radial=True)
    yield "K nx ny = 2^31", dict(ok, z=np.zeros(2), bins=(2**15, 2**15))
    yield "nx = 2^31", dict(ok, z=(0.,), bins=(2**31, 1))
    yield "lo = nan", dict(ok, range=((np.nan, 1.), (-2., 2.)))
    yield "hi = inf", dict(ok, range=((-1., 1.), (-2., np.inf)))
    yield "lo = hi", dict(ok, range=((1., 1.), (-2., 2.)))
    yield "lo > hi", dict(ok, range=((-1., 1.), (2., -2.)))
    yield "subnormal step", dict(ok, range=((0., 1e-310), (-2., 2.)))
    yield "step overflows", dict(ok, range=((-1.7e308, 1.7e308), (-2., 2.)))
    yield "z = nan", dict(ok, z=(0., np.nan))
    yield "o = inf", dict(ok, offsets=((0., 0.), (np.inf, 0.)))


@pytest.mark.parametrize("what,kw", list(_bad_specs()))
def test_spot_refuses_bad_arguments_without_a_context(lib, what, kw):
    """every refusal of include/rtx.h comes before any device work: with
    ctx = NULL and a dummy counts pointer the checks still answer BADARG
    (and a good record is refused only for the NULL context)"""
    counts = C.c_void_p(0x1000)                      # never dereferenced
    rec = spot_spec(kw.pop("z"), kw.pop("bins"), kw.pop("range"), kw.pop("center"), **kw)
    p = rec.ctypes.data_as(C.c_void_p)
    assert lib.rtx_spot_rows(None, 0, 10, counts, counts, p, counts, None, None) == -1, what
    assert lib.rtx_trace_spot(None, None, 0, None, 0, 10, counts, counts, 0, p, counts, None,
                              None, 0) == -1, what


def test_spot_refuses_no_outputs_and_no_record(lib):
    rec = spot_spec((0.,), (4, 4), ((-1., 1.), (-1., 1.)), (0., 0.))
    p = rec.ctypes.data_as(C.c_void_p)
    d = C.c_void_p(0x1000)
    assert lib.rtx_spot_rows(None, 0, 10, d, d, p, None, None, None) == -1
    assert lib.rtx_spot_rows(None, 0, 10, d, d, None, d, None, None) == -1
    assert lib.rtx_trace_spot(None, None, 0, None, 0, 10, d, d, 0, p, None, None, None, 0) == -1
