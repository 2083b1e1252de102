"""The helpers of tests/test_gpu_epilogue_rays.py, without a GPU: the seeded
lenses contain every feature the per-ray epilogue matrix is meant to cover,
and the per-ray rule (`ray_moments`, `check_rays`) is the exact oracle's
(epi_oracle.reduce_sums) for a bundle of one ray."""
from fractions import Fraction

import numpy as np
import pytest

import epi_oracle
import np_oracle
from test_gpu_config_invariance import random_rays
from test_gpu_epilogue_rays import (CONTRACTED, EPS, LAST_KINDS, LENSES, MANY_S, check_rays,
                                    features, lens, many_tables, random_lens, ray_moments)

FEATURES = {"asph 5..10", "alt", "mirror", "mu1"} | {"last " + k for k in LAST_KINDS}


def test_lenses_cover_the_matrix():
    """every feature, rot0 on and off, clip on and off, lenses whose
    exact-mode truth is np_oracle and lenses whose truth is the stored trace"""
    seen = set()
    for name in LENSES:
        table, rot0, clip, analytic = lens(name)
        seen |= features(table)
        seen.add(("rot0", rot0 is not None))
        seen.add(("clip", clip))
        seen.add(("oracle truth", analytic and rot0 is None))
        if analytic:
            assert (table["n_asph"] < 0).all() and not (table["flags"] & 1).any(), name
    want = FEATURES | {(k, v) for k in ("rot0", "clip", "oracle truth") for v in (False, True)}
    assert want <= seen, want - seen


@pytest.mark.parametrize("name", list(LENSES))
def test_each_lens_has_its_last_surface_and_rays(name):
    """the last surface is of the kind the lens is named for, and a fair share
    of the random launch rays reaches it finite (the per-ray checks are not
    about NaNs only)"""
    table, rot0, clip, _ = lens(name)
    last = LENSES[name][1]
    assert "last " + last in features(table), (name, features(table))
    y0, u0 = random_rays(np.random.default_rng(1), 4096)
    Y = np_oracle.trace(table, y0, u0, clip=clip, rot0=rot0)[0]
    fin = np.isfinite(Y[-1]).all(1).mean()
    assert fin >= .2, (name, fin)


def test_many_tables_differ_in_structure():
    """the 8 tables of the reduce_many test share S but not their kinds,
    tilts or coefficient counts"""
    tabs = many_tables()
    assert tabs.shape == (8, MANY_S)
    sig = {(tuple(t["n_asph"]), tuple(t["flags"]), tuple(t["c"] == 0), tuple(t["mu"] == -1))
           for t in tabs}
    assert len(sig) == len(tabs)
    assert len({int(t["n_asph"].max()) for t in tabs}) >= 3
    assert any((t["flags"] & 1).any() for t in tabs) and not all((t["flags"] & 1).any()
                                                                 for t in tabs)
    assert random_lens(900, LAST_KINDS[0], True, S=MANY_S).tobytes() == tabs[0].tobytes()


def _rows(n, seed):
    """random rows, rows with NaN, +-inf, +-0 and i_z = 0 components, centres
    and weights"""
    rng = np.random.default_rng(seed)
    y = np.c_[rng.normal(0, 2, (n, 2)), rng.normal(0, 1, n)]
    u = rng.normal(0, .1, (n, 2))
    inc = np.c_[u, np.sqrt(1 - np.square(u).sum(1))]
    special = [np.nan, np.inf, -np.inf, 0., -0.]
    for j, i in enumerate(range(0, n, 7)):
        a = y if j % 2 else inc
        a[i, j % 3] = special[j % len(special)]
    c = np.c_[rng.normal(0, 1, (n, 2)), rng.normal(0, .05, (n, 2))]
    c[3] = (y[3, 0], y[3, 1], inc[3, 0]/inc[3, 2], inc[3, 1]/inc[3, 2])   # dx = dy = ux = uy = 0
    w = rng.uniform(.5, 2., n)
    return y, inc, c, w


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_one_ray_rule_is_the_exact_oracle(dtype):
    """for N = 1, epi_oracle.reduce_sums is ray_moments column by column: the
    single-operation columns exactly, the contracted ones within the rule's
    bound; check_rays accepts the oracle's values"""
    y, inc, c, w = _rows(400, 3)
    y, inc = y.astype(dtype), inc.astype(dtype)
    for weighted in (False, True):
        wi = w.astype(dtype).astype(np.float64) if weighted else None
        want, ext, scale = ray_moments(y, inc, c, wi)
        got = np.array([epi_oracle.reduce_sums(y[i:i + 1], inc[i:i + 1],
                                               None if wi is None else wi[i:i + 1], c[i])[0]
                        for i in range(len(y))])
        cols = [k for k in range(20) if k not in CONTRACTED]
        assert np.array_equal(got[:, cols], want[:, cols], equal_nan=True)
        assert np.array_equal(got[:, CONTRACTED], want[:, CONTRACTED], equal_nan=True)
        check_rays(got, y, inc, c, wi, "oracle")
        assert np.isnan(want).any() and (want[:, 4] == 0).any() and (want[:, 8] == 0).any()


def _round(x):
    """a Fraction rounded to the nearest double (ties to even)"""
    return x.numerator/x.denominator


def test_contracted_bound_admits_every_fusion_and_no_more():
    """the extended-precision reference of m[3], m[18], m[19] is within
    2^-60 of the scale of the exact Fraction value; each order of evaluation
    the compiler may pick (plain, or either product fused into the sum) is
    accepted; a value 3 eps of the scale away is refused"""
    y, inc, c, w = _rows(300, 5)
    fin = np.isfinite(y).all(1) & np.isfinite(inc).all(1) & (inc[:, 2] != 0)
    y, inc, c, w = y[fin], inc[fin], c[fin], w[fin]
    want, ext, scale = ray_moments(y, inc, c, w)
    dx, dy = y[:, 0] - c[:, 0], y[:, 1] - c[:, 1]
    ux, uy = inc[:, 0]/inc[:, 2] - c[:, 2], inc[:, 1]/inc[:, 2] - c[:, 3]
    F = Fraction
    for i in range(len(y)):
        pairs = {3: ((dx[i], dx[i]), (dy[i], dy[i])), 18: ((dx[i], ux[i]), (dy[i], uy[i])),
                 19: ((ux[i], ux[i]), (uy[i], uy[i]))}
        for j, k in enumerate(CONTRACTED):
            (a, b), (p, q) = pairs[k]
            exact = F(w[i])*(F(a)*F(b) + F(p)*F(q))
            e = ext[i, j]
            assert abs(F(*e.as_integer_ratio()) - exact) <= \
                F(*scale[i, j].as_integer_ratio())/2**60, (i, k)
            s1, s2 = F(a)*F(b), F(p)*F(q)
            for s in (_round(F(_round(s1)) + F(_round(s2))),      # a*b + p*q
                      _round(s1 + F(_round(s2))),                 # fma(a, b, p*q)
                      _round(F(_round(s1)) + s2)):                # fma(p, q, a*b)
                m = want[i:i + 1].copy()
                m[0, k] = _round(F(w[i])*F(s))
                check_rays(m, y[i:i + 1], inc[i:i + 1], c[i], w[i:i + 1], "fusion")
            m = want[i:i + 1].copy()
            m[0, k] = float(e + 3*EPS*scale[i, j])
            if m[0, k] != want[i, k]:
                with pytest.raises(AssertionError):
                    check_rays(m, y[i:i + 1], inc[i:i + 1], c[i], w[i:i + 1], "off")
