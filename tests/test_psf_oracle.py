"""The PSF oracle (oracle/psf_oracle.py) against scipy's griddata and the
reference's stored PSFs (tests/golden/vs_reference/psf_*.npz, made by
tests/golden/make_psf_golden.py); the library does not link cuFFT."""
import glob
import os
import subprocess

import numpy as np
import pytest
from scipy.interpolate import griddata

import psf_oracle
from conftest import GOLDEN, ROOT

CASES = sorted(os.path.basename(p)[:-4]
               for p in glob.glob(os.path.join(GOLDEN, "vs_reference", "psf_*.npz")))


def load(name):
    d = np.load(os.path.join(GOLDEN, "vs_reference", name + ".npz"))
    return {k: d[k] for k in d.files}


def test_fixtures_present_and_small():
    assert len(CASES) == 4, CASES
    for c in CASES:
        assert os.path.getsize(os.path.join(GOLDEN, "vs_reference", c + ".npz")) < 1 << 20


@pytest.mark.parametrize("m", [2000, 20000])
def test_regrid_bit_equal_to_griddata_random(m):
    rng = np.random.default_rng(m)
    x, y = rng.random((2, m))*2 - 1
    t = np.sin(3*x) + y*y
    n = int(4*m**.5)
    xs, ys, o = psf_oracle.regrid(x, y, t, n, np.fabs((x, y)).max())
    want = griddata((x, y), t, (xs, ys), method="linear", fill_value=np.nan)
    assert np.array_equal(o, want, equal_nan=True)


@pytest.mark.parametrize("name", CASES)
def test_regrid_bit_equal_on_exit_pupil_points(name):
    c = load(name)
    x, y, t = c["x"], c["y"], c["t"]
    xs, ys, o = psf_oracle.opd_grid(x, y, t, int(c["nrays"]))
    assert np.array_equal(xs[:, 0], c["gh"])
    ok = np.isfinite(x) & np.isfinite(y) & np.isfinite(t)
    want = griddata((x[ok], y[ok]), t[ok], (xs, ys), method="linear", fill_value=np.nan)
    assert np.array_equal(o, want, equal_nan=True)
    assert np.array_equal(o, c["o"], equal_nan=True)         # the reference's own opd()


@pytest.mark.parametrize("name", CASES)
def test_psf_matches_reference(name):
    c = load(name)
    xs, _, o = psf_oracle.opd_grid(c["x"], c["y"], c["t"], int(c["nrays"]))
    p, q, psf = psf_oracle.psf(xs, o, 4, float(c["wavelength"]), float(c["radius"]))
    assert np.array_equal(p[:, 0], c["f"]) and np.array_equal(q[0], c["f"])
    assert psf.shape == c["psf"].shape
    assert np.abs(psf - c["psf"]).max() <= 1e-12*c["psf"].max()


def test_library_does_not_link_cufft():
    from rayopt_b200 import build
    build.build()
    out = subprocess.run(["ldd", os.path.join(ROOT, "rayopt_b200", "librtx.so")],
                         capture_output=True, text=True, check=True).stdout
    assert "libcufft" not in out, out
