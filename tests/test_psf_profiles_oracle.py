"""The encircled-energy / MTF oracle (oracle/profile_oracle.py) against the
reference's own polar_sum (rayopt/special_sums.py:240-263), where its tree is
present, and against known answers.  The reference's polar_sum uses the
removed np.int and bincount(minlength=None); it runs here under a test-scoped
patch that restores both."""
import importlib.util
import os

import numpy as np
import pytest

import profile_oracle
import psf_oracle
import ref_shim

needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="no reference tree staged")


@pytest.fixture
def ref_polar_sum(monkeypatch):
    path = os.path.join(ref_shim.REFERENCE_ROOT, "rayopt", "special_sums.py")
    spec = importlib.util.spec_from_file_location("_ref_special_sums", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    bincount = np.bincount
    monkeypatch.setattr(np, "int", int, raising=False)
    monkeypatch.setattr(np, "bincount", lambda x, weights=None, minlength=None:
                        bincount(x, weights, 0 if minlength is None else minlength))
    return lambda m, center: mod.polar_sum(m, center, "azimuthal")


def random_cases():
    rng = np.random.default_rng(3)
    for shape in [(1, 1), (3, 3), (7, 5), (64, 64), (127, 90), (256, 256)]:
        m = rng.random(shape)
        nx, ny = shape
        for center in [(nx/2 + .3712, ny/2 - 1.25),        # fractional, Analysis-like
                       (nx//2, ny//2), (1, 2),             # integer: Pythagorean boundaries
                       (nx/2 + .5, ny/2 - .5),             # half-integer
                       (-3.5, ny + 7.25), (nx + 20, -11)]: # outside the array
            yield m, center


@needs_ref
def test_restatement_bit_identical_to_reference(ref_polar_sum):
    count = 0
    for m, center in random_cases():
        want = ref_polar_sum(m, center)
        got = profile_oracle.polar_sum_azimuthal(m, center)
        assert got.dtype == want.dtype and np.array_equal(got, want), (m.shape, center)
        count += 1
    assert count == 36


def test_docstring_known_answers():
    m = np.arange(1., 10.).reshape((3, 3))
    assert np.array_equal(profile_oracle.polar_sum_azimuthal(m, (1, 1)), [5., 40.])
    assert np.array_equal(profile_oracle.polar_sum_azimuthal(m, (.5, .5)), [12., 24., 9.])


def test_integer_centre_boundaries_exact():
    """pixels on bin boundaries (3-4-5, 5-12-13, 8-15-17 triangles) bin exactly"""
    m = np.zeros((40, 40))
    c = (10, 10)
    for (di, dj), r in [((3, 4), 5), ((5, 12), 13), ((8, 15), 17), ((0, 7), 7)]:
        m[:] = 0
        m[c[0] + di, c[1] + dj] = 1.
        b = profile_oracle.polar_sum_azimuthal(m, c)
        assert b[r] == 1. and b.sum() == 1., (di, dj)


@pytest.mark.parametrize("n", [64, 65])
def test_profiles_of_a_delta(n):
    """a delta PSF (all energy at the zero frequency): EE = 1 from bin 0 (for
    odd n the centre sits half a pixel off the fftshift origin, Analysis's
    true division, still within bin 0); the MTF is 1 everywhere"""
    psf = np.zeros((n, n))
    psf[0, 0] = 1.
    f = np.fft.fftfreq(n, .01)
    p, q = np.broadcast_arrays(f[:, None], f)
    r = profile_oracle.profiles(p, q, psf)
    assert r["x0"] == 0 and r["y0"] == 0
    assert r["center"] == (n/2, n/2)
    assert np.all(r["ee"] == 1.)
    fs = np.fft.fftshift(f)
    assert r["dx"] == fs[1] - fs[0]
    for m in r["mtf"]:
        assert m.shape == (n//2,)
        np.testing.assert_allclose(m, 1., rtol=0, atol=1e-15)
    np.testing.assert_array_equal(r["of"], np.fft.fftfreq(n, r["dx"])[:n//2])
    np.testing.assert_array_equal(r["xe"], np.arange(r["ee"].size)*r["dx"])


def test_line_sums_are_the_stored_order_sums():
    rng = np.random.default_rng(5)
    psf = rng.random((9, 6))
    l0, l1 = profile_oracle.line_sums(psf)
    np.testing.assert_allclose(l0, psf.sum(0), rtol=1e-15)
    np.testing.assert_allclose(l1, psf.sum(1), rtol=1e-15)


@pytest.mark.parametrize("name", ["psf_cooke_f07", "psf_mirror"])
def test_profiles_of_stored_reference_psf(name):
    """the stored reference PSFs: EE rises to the PSF's sum, the MTF starts at
    the PSF's sum times sqrt(size)/n along each axis and never exceeds it"""
    from conftest import GOLDEN
    d = np.load(os.path.join(GOLDEN, "vs_reference", name + ".npz"))
    psf, f = d["psf"], d["f"]
    p, q = np.broadcast_arrays(f[:, None], f)
    r = profile_oracle.profiles(p, q, psf)
    s = psf.sum()
    assert abs(r["ee"][-1] - s) <= 1e-12*s
    assert np.all(np.diff(r["ee"]) >= 0)
    st = psf_oracle.stats(p, q, psf)
    assert r["stats"]["sum"] == st["sum"]
    for m in r["mtf"]:
        assert abs(m[0] - s) <= 1e-12*s
        assert m.max() <= m[0]*(1 + 1e-12)
