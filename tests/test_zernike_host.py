"""The host side of rayopt_b200.zernike: Noll's table, the closed-form
basis, the fit from the Gram sums, and the argument refusals of
tolerance_zernike and zernike before any device work.  No GPU needed."""
import warnings

import numpy as np
import pytest

import ref_shim
from rayopt_b200.surface_table import pack_system
from rayopt_b200.zernike import (noll, nterms, tolerance_zernike, zernike, zernike_basis,
                                 zernike_fit, zernike_result)
from test_tolerance_driver_host import _NoEngine, _StubSystem

needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="no reference tree staged")


# ---- Noll's table and the closed-form basis ----------------------------------
def test_noll_table():
    t = noll(45)
    assert t.shape == (45, 2)
    anchors = {1: (0, 0), 2: (1, 1), 3: (1, -1), 4: (2, 0), 5: (2, -2), 6: (2, 2), 7: (3, -1),
               8: (3, 1), 9: (3, -3), 10: (3, 3), 11: (4, 0), 12: (4, 2), 13: (4, -2),
               14: (4, 4), 15: (4, -4), 16: (5, 1), 17: (5, -1), 22: (6, 0), 37: (8, 0),
               45: (8, -8)}
    for j, nm in anchors.items():
        assert tuple(t[j - 1]) == nm, j
    for j, (n, m) in enumerate(t, 1):
        assert n*(n + 1)//2 < j <= (n + 1)*(n + 2)//2                  # grouped by order
        assert (n - abs(m)) % 2 == 0 and abs(m) <= n
        assert m == 0 or (m > 0) == (j % 2 == 0)                      # even j: cosine
    assert len({tuple(r) for r in t}) == 45
    assert [nterms(k) for k in range(9)] == [1, 3, 6, 10, 15, 21, 28, 36, 45]


def test_basis_anchors():
    rng = np.random.default_rng(0)
    x, y = rng.uniform(-1, 1, (2, 200))
    r2, th = x*x + y*y, np.arctan2(y, x)
    r = np.sqrt(r2)
    Z = zernike_basis(45, x, y)
    want = {1: np.ones_like(x), 2: 2*x, 3: 2*y, 4: np.sqrt(3)*(2*r2 - 1),
            5: np.sqrt(6)*r2*np.sin(2*th), 6: np.sqrt(6)*r2*np.cos(2*th),
            7: np.sqrt(8)*(3*r**3 - 2*r)*np.sin(th), 8: np.sqrt(8)*(3*r**3 - 2*r)*np.cos(th),
            11: np.sqrt(5)*(6*r2**2 - 6*r2 + 1),
            22: np.sqrt(7)*(20*r**6 - 30*r**4 + 12*r2 - 1),
            37: 3*(70*r**8 - 140*r**6 + 90*r**4 - 20*r2 + 1)}
    for j, w in want.items():
        np.testing.assert_allclose(Z[..., j - 1], w, rtol=1e-12, atol=1e-13, err_msg=str(j))


def test_basis_orthonormal():
    """the mean of Z_j Z_k over the unit disc, on a Gauss-Legendre radial x
    uniform angular rule that integrates the degree-16 products exactly"""
    t, w = np.polynomial.legendre.leggauss(12)
    r, wr = (t + 1)/2, w/2                                     # on [0, 1]
    th = 2*np.pi*np.arange(40)/40
    R, TH = np.meshgrid(r, th, indexing="ij")
    Z = zernike_basis(45, R*np.cos(TH), R*np.sin(TH))           # (12, 40, 45)
    wt = (wr*r)[:, None]*np.full(40, 2*np.pi/40)/np.pi          # r dr dtheta / pi
    G = np.einsum("ab,abj,abk->jk", wt, Z, Z)
    assert np.abs(G - np.eye(45)).max() <= 1e-13


def test_basis_long_double():
    x = np.array([.3, -.7], np.longdouble)
    y = np.array([.1, .2], np.longdouble)
    Z = zernike_basis(28, x, y)
    assert Z.dtype == np.longdouble
    np.testing.assert_allclose(Z.astype(float), zernike_basis(28, x.astype(float),
                                                              y.astype(float)), atol=1e-14)


# ---- the fit from the sums ---------------------------------------------------
def hexapolar(rings):
    pts = [(0., 0.)]
    for i in range(1, rings + 1):
        a = 2*np.pi*np.arange(6*i)/(6*i)
        pts += list(zip(i/rings*np.cos(a), i/rings*np.sin(a)))
    return np.array(pts)


def gram_sums(a, x, y, rho, J):
    """rtx_trace_zernike_many's sums in long double: the upper triangle of
    the Gram of v = (a, Z_1 .. Z_J) at (x, y)/rho"""
    ld = np.longdouble
    Z = zernike_basis(J, np.asarray(x, ld)/ld(rho), np.asarray(y, ld)/ld(rho))
    v = np.concatenate([np.asarray(a, ld)[:, None], Z], 1)
    M = np.einsum("ij,ik->jk", v, v)
    return M[np.triu_indices(J + 1)].astype(np.float64)


@pytest.mark.parametrize("order", [0, 1, 4, 6, 8])
def test_fit_recovers_coefficients(order):
    """a = -lambda (Z c + noise) on a hexapolar grid of radius 3 (rho = 3):
    the fit returns c within the noise's own least-squares part, the
    residual and the piston-removed rms"""
    J = nterms(order)
    rng = np.random.default_rng(order)
    p = 3*hexapolar(12)
    x, y = p.T
    lam = 5.8756e-4
    c = rng.normal(0, .3, J)
    noise = rng.normal(0, 1e-3, len(x))
    Z = zernike_basis(J, x/3, y/3)
    t = Z @ c + noise                                          # waves
    a = -lam*t
    got = zernike_fit(gram_sums(a, x, y, 3., J)[None], J, lam)
    sol, *_ = np.linalg.lstsq(Z, t, rcond=None)
    r = t - Z @ sol
    np.testing.assert_allclose(got["coefficients"][0], sol, rtol=0, atol=1e-9)
    assert abs(got["coefficients"][0] - c).max() < 1e-3
    assert got["residual"][0] == pytest.approx(np.sqrt(np.mean(r*r)), rel=1e-6, abs=1e-10)
    assert got["rms"][0] == pytest.approx(np.std(t), rel=1e-12)
    assert got["rank"][0] == J


def test_fit_rank_deficient():
    """too few rays, and every ray on one line: the minimum-norm fit (as
    lstsq of the design matrix) and its rank"""
    lam = 5e-4
    J = nterms(4)
    rng = np.random.default_rng(3)
    for x, y, rank in ((rng.uniform(-1, 1, 7), rng.uniform(-1, 1, 7), 7),
                       (np.linspace(-1, 1, 41), np.zeros(41), 5)):
        Z = zernike_basis(J, x, y)
        t = rng.normal(0, .1, len(x))
        got = zernike_fit(gram_sums(-lam*t, x, y, 1., J)[None], J, lam)
        sol = np.linalg.lstsq(Z, t, rcond=1e-10)[0]
        assert got["rank"][0] == rank == np.linalg.matrix_rank(Z)
        np.testing.assert_allclose(got["coefficients"][0], sol, rtol=0, atol=1e-8)
        r = t - Z @ sol
        # sum a^2/n - c.b cancels: an exact fit (7 rays) leaves sqrt(eps mean t^2)
        floor = np.sqrt(1e3*2.0**-52*np.mean(t*t))
        assert got["residual"][0] == pytest.approx(np.sqrt(np.mean(r*r)), rel=1e-6, abs=floor)


def test_fit_empty_and_lost_chief():
    """n = 0 and a lost chief ray give NaN values and rank 0"""
    J = 3
    rng = np.random.default_rng(4)
    x, y = rng.uniform(-1, 1, (2, 50))
    s = gram_sums(rng.normal(0, 1e-4, 50), x, y, 1., J)
    sums = np.stack([s, np.zeros_like(s), s]).reshape(1, 1, 3, -1)
    out = zernike_result(sums, J, [5e-4]*3, np.full((1, 3), 50.),
                         chief=np.array([[[True, True, False]]]))
    assert np.isfinite(out["coefficients"][0, 0, 0]).all() and out["rank"][0, 0, 0] == J
    for w in (1, 2):
        assert np.isnan(out["coefficients"][0, 0, w]).all() and out["rank"][0, 0, w] == 0
        assert np.isnan(out["residual"][0, 0, w]) and np.isnan(out["rms"][0, 0, w])
    assert out["transmitted"][0, 0, 0] == 1 and out["transmitted"][0, 0, 1] == 0
    assert out["noll"].shape == (J, 2)


# ---- refusals before any device work -----------------------------------------
@pytest.mark.parametrize("kw, msg", [
    (dict(order=-1), "order"), (dict(order=9), "order"), (dict(order=2.5), "order"),
    (dict(order=True), "order"), (dict(order="6"), "order"),
    (dict(compensate="tilt"), "compensate"), (dict(chunk=0), "chunk"),
    (dict(heights=[]), "height"),
])
def test_refusals_before_device_work(kw, msg):
    args = dict(params=[(1, "curvature")], deltas=np.zeros((2, 1)))
    args.update(kw)
    with pytest.raises(ValueError, match=msg):
        tolerance_zernike(_StubSystem(), engine=_NoEngine(), **args)


@pytest.mark.parametrize("order", [-1, 9])
def test_zernike_refusals_before_device_work(order):
    with pytest.raises(ValueError, match="order"):
        zernike(_StubSystem(), order=order, engine=_NoEngine())


def _reference(name):
    import yaml
    import systems_yaml
    warnings.simplefilter("ignore")
    np.seterr(all="ignore")
    R = ref_shim.load()
    s = R.System(**yaml.safe_load(systems_yaml.SYSTEMS[name]))
    s.update()
    s.paraxial.refocus()
    return s


@needs_ref
@pytest.mark.parametrize("kw, msg", [
    (lambda S: dict(params=[(S + 1, "curvature")]), "not in"),
    (lambda S: dict(params=[(1, "bogus")]), "unknown tolerance kind"),
    (lambda S: dict(params=[(S, "curvature")]), "image surface"),
    (lambda S: dict(params=[(S, "tilt_x")]), "image surface"),
    (lambda S: dict(deltas=np.zeros((3, 2))), "deltas must be"),
])
def test_lens_refusals_before_device_work(kw, msg):
    s = _reference("cooke")
    args = dict(params=[(1, "curvature")], deltas=np.zeros((2, 1)))
    with np.errstate(all="ignore"):
        args.update(kw(len(pack_system(s, s.wavelengths[0], 1, None)[0])))
        with pytest.raises(ValueError, match=msg):
            tolerance_zernike(s, engine=_NoEngine(), **args)
