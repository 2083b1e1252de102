"""Pins the oracle AND the table packer against the reference (quartiq/rayopt).

The reference's packed tables, launch rays and traces are stored under
tests/golden/vs_reference/ (tests/golden/make_golden.py --vs-reference); the
oracle must reproduce them bit for bit.  When the reference tree itself is
available the stored tables are also checked against the packer run on the
reference's live System objects."""
import os
import warnings

import numpy as np
import pytest
import yaml

import np_oracle
import ref_shim
import systems_yaml
from conftest import GOLDEN
from rayopt_b200.surface_table import pack_system

CASES = [("cooke", 20000, False), ("double_gauss", 20000, True),
         ("zoom", 10000, True), ("cooke_asph", 400, True), ("mirror", 5000, False),
         ("singlet", 5000, True)]


def load(name):
    d = np.load(os.path.join(GOLDEN, "vs_reference", name + ".npz"))
    return {k: d[k] for k in d.files}


@pytest.mark.parametrize("name,n,clip", CASES)
def test_bitwise_vs_live_reference(name, n, clip):
    c = load(name)
    assert bool(c["clip"]) == clip and int(c["n_rays"]) == n
    for j in range(2):
        rot0 = c["rot0%d" % j] if c["rot0%d" % j].size else None
        Y, U, I, T = np_oracle.trace(c["table%d" % j], c["y0%d" % j], c["u0%d" % j], clip=clip,
                                     rot0=rot0)
        exact = name != "cooke_asph"   # Newton fprime uses np.dot (BLAS)
        for a, k in ((Y, "Y"), (U, "U"), (I, "I"), (T, "T")):
            b = c["%s%d" % (k, j)]
            if exact:
                assert np.array_equal(a, b, equal_nan=True), (name, j, k)
            else:
                assert np.array_equal(np.isnan(a), np.isnan(b))
                np.testing.assert_allclose(a, b, rtol=1e-13, atol=1e-13)


@pytest.mark.skipif(not ref_shim.available(), reason="reference tree not present")
@pytest.mark.parametrize("name", [c[0] for c in CASES])
def test_packer_vs_live_reference(name):
    """the stored tables are what pack_system makes of the reference's System"""
    R = ref_shim.load()
    c = load(name)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        s = R.System(**yaml.safe_load(systems_yaml.SYSTEMS[name]))
        s.update()
        s.paraxial.refocus()
        for j, l in enumerate(s.wavelengths[:2]):
            table, nn, rot0 = pack_system(s, l)
            assert table.tobytes() == c["table%d" % j].tobytes()
            assert np.array_equal(nn, c["n%d" % j])
            assert (rot0 is None) == (c["rot0%d" % j].size == 0)
