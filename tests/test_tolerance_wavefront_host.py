"""Host side of the wavefront tolerance analysis
(rayopt_b200.tolerance_wavefront): its refusals before any device work, the
result assembly from the 10 sums against a two-pass least-squares fit in
long double, and the per-variant reference sphere (wavefront_specs) against
lazy.opd_spec of a reference System with the same change made.  No GPU."""
import copy
import warnings

import numpy as np
import pytest

import ref_shim
from rayopt_b200.engine import OPD_DTYPE
from rayopt_b200.surface_table import pack_system
from rayopt_b200.tolerance import (perturbed_tables, tolerance_wavefront, wavefront_specs,
                                   wavefront_tolerance_result)
from test_tolerance_driver_host import _NoEngine, _StubSystem

needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="no reference tree staged")


@pytest.mark.parametrize("kw, msg", [
    (dict(targets=np.ones(5)), "targets"),
    (dict(targets=np.ones((2, 3))), "targets"),
    (dict(spectral_weights=[1., 2.]), "spectral_weights"),
    (dict(spectral_weights=[1., np.nan, 1.]), "spectral_weights"),
    (dict(compensate="tilt"), "compensate"),
    (dict(chunk=0), "chunk"),
])
def test_refusals_before_device_work(kw, msg):
    args = dict(params=[(1, "curvature")], deltas=np.zeros((2, 1)))
    args.update(kw)
    with pytest.raises(ValueError, match=msg):
        tolerance_wavefront(_StubSystem(), engine=_NoEngine(), **args)


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
    (lambda S: dict(params=[(S, "index")]), "is the last"),
    (lambda S: dict(params=[(S, "curvature")]), "image surface"),
    (lambda S: dict(params=[(S, "conic")]), "image surface"),
    (lambda S: dict(params=[(S, "asph1")]), "image surface"),
    (lambda S: dict(params=[(S, "tilt_x")]), "image surface"),
    (lambda S: dict(params=[(S, "tilt_y")]), "image surface"),
    (lambda S: dict(deltas=np.zeros((3, 2))), "deltas must be"),
    (lambda S: dict(deltas=np.zeros((2, 1, 1))), "deltas must be"),
])
def test_lens_refusals_before_device_work(kw, msg):
    """`kw` of the number of surfaces S"""
    s = _reference("cooke")
    args = dict(params=[(1, "curvature")], deltas=np.zeros((2, 1)))
    with np.errstate(all="ignore"):
        args.update(kw(len(pack_system(s, s.wavelengths[0], 1, None)[0])))
        with pytest.raises(ValueError, match=msg):
            tolerance_wavefront(s, engine=_NoEngine(), **args)


# ---- the result from the 10 sums ------------------------------------------
WL = np.array([5.8756e-4, 6.5627e-4, 4.8613e-4])


def _rays(rng, n, tilt):
    """n pupil points and their residuals: piston, a tilt `tilt` times the
    residual's scale, defocus-like and random parts"""
    x, y = rng.uniform(-1, 1, (2, n))*5
    a = 1e-4*(rng.normal() + tilt*(rng.normal()*x + rng.normal()*y)
              + .3*(x*x + y*y - 12) + rng.normal(0, 1, n))
    return a, x, y


def _sums_ld(a, x, y):
    a, x, y = (np.asarray(v, np.longdouble) for v in (a, x, y))
    return np.array([len(a), a.sum(), (a*a).sum(), x.sum(), y.sum(), (x*x).sum(), (x*y).sum(),
                     (y*y).sum(), (a*x).sum(), (a*y).sum()], np.longdouble)


def _fit_ld(a, x, y):
    """(piston-removed rms^2, tilt-removed rms^2) by two passes in long
    double: centre, then the 2x2 normal equations and the residuals"""
    a, x, y = (np.asarray(v, np.longdouble) for v in (a, x, y))
    ac, xc, yc = a - a.mean(), x - x.mean(), y - y.mean()
    Sxx, Sxy, Syy = (xc*xc).sum(), (xc*yc).sum(), (yc*yc).sum()
    Sax, Say = (ac*xc).sum(), (ac*yc).sum()
    det = Sxx*Syy - Sxy*Sxy
    b1, b2 = (Syy*Sax - Sxy*Say)/det, (Sxx*Say - Sxy*Sax)/det
    r = ac - b1*xc - b2*yc
    return (ac*ac).sum()/len(a), (r*r).sum()/len(a)


def _synthetic(seed, V=4, H=3, W=3):
    rng = np.random.default_rng(seed)
    N = rng.integers(50, 400, (H, W))
    sums = np.zeros((V, H, W, 10))
    want = np.full((V, H, W, 2), np.nan)
    chief = np.ones((V, H, W), bool)
    for v in range(V):
        for h in range(H):
            for w in range(W):
                n = int(rng.integers(10, N[h, w] + 1))
                if (v, h, w) == (1, 0, 2):
                    continue                              # nothing entered
                a, x, y = _rays(rng, n, (0., 3., 100.)[(v + h + w) % 3])
                a, x, y = a, x*1e-2, y*1e-2
                sums[v, h, w] = _sums_ld(a, x, y).astype(np.float64)
                r2, t2 = _fit_ld(a, x, y)
                want[v, h, w] = np.sqrt([float(r2), float(t2)])/WL[w]
    chief[2, 1, 1] = False                                # a lost chief ray
    sums[2, 1, 1] = 0.
    want[2, 1, 1] = np.nan
    return sums, N, chief, want


def test_result_against_long_double_fit():
    sums, N, chief, want = _synthetic(1)
    sw = np.array([1., 2., .5])
    res = wavefront_tolerance_result(sums, WL, N, sw, chief)
    nan = np.isnan(want[..., 0])
    for k, i in (("rms", 0), ("rms_tilt", 1)):
        assert np.array_equal(np.isnan(res[k]), nan), k
    rms = want[..., 0]
    assert np.all(np.abs(res["rms"][~nan] - rms[~nan]) <= 1e-12*rms[~nan])
    assert np.all(np.abs(res["rms_tilt"][~nan] - want[..., 1][~nan]) <= 1e-12*rms[~nan])
    assert np.all(res["rms_tilt"][~nan] <= res["rms"][~nan]*(1 + 1e-12))
    assert np.array_equal(res["strehl"], np.exp(-(2*np.pi*res["rms_tilt"])**2), equal_nan=True)
    assert np.allclose(res["strehl"][~nan], np.exp(-(2*np.pi*want[..., 1][~nan])**2),
                       rtol=1e-8, atol=0)
    with np.errstate(invalid="ignore"):
        tr = sums[..., 0]/N
    tr[~chief] = np.nan
    assert np.array_equal(res["transmitted"], tr, equal_nan=True)
    assert np.isnan(res["sums"][2, 1, 1]).all() and not res["chief"][2, 1, 1]
    for k, i in (("poly_rms", 0), ("poly_rms_tilt", 1)):
        p = np.sqrt((want[..., i]**2*sw).sum(-1)/sw.sum())
        assert np.array_equal(np.isnan(res[k]), np.isnan(p)), k
        f = np.isfinite(p)
        assert np.allclose(res[k][f], p[f], rtol=1e-12, atol=0), k
    assert np.isnan(res["poly_rms"][1, 0]) and np.isnan(res["poly_rms_tilt"][2, 1])


def test_result_against_lstsq():
    """the tilt fit against numpy's lstsq on 1, x, y (float64)"""
    rng = np.random.default_rng(5)
    a, x, y = _rays(rng, 300, 3.)
    s = _sums_ld(a, x, y).astype(np.float64)
    res = wavefront_tolerance_result(s.reshape(1, 1, 1, 10), [1.], [[300]], [1.])
    A = np.c_[np.ones_like(x), x, y]
    r = a - A @ np.linalg.lstsq(A, a, rcond=None)[0]
    assert np.isclose(res["rms_tilt"][0, 0, 0], np.sqrt((r*r).mean()), rtol=1e-10)


def test_degenerate_pupils():
    """one ray: both rms 0; rays on a line: the tilt along it is removed;
    a pure tilt leaves no residual (clamped at 0, never NaN)"""
    rows = []
    rows.append(_sums_ld([3e-4], [.1], [.2]))
    t = np.linspace(-1, 1, 7)
    rows.append(_sums_ld(2e-4*t + 1e-6*t*t, t, 2*t))
    x, y = np.meshgrid(np.linspace(-1, 1, 9), np.linspace(-1, 1, 9))
    rows.append(_sums_ld(1e-3*(.3*x - .7*y).ravel() + 4e-4, x.ravel(), y.ravel()))
    s = np.array(rows, np.float64).reshape(1, 1, 3, 10)
    res = wavefront_tolerance_result(s, [1., 1., 1.], [[1, 7, 81]], np.ones(3))
    assert res["rms"][0, 0, 0] == 0 and res["rms_tilt"][0, 0, 0] == 0
    r = 1e-6*(t*t - (t*t).mean())
    c = np.polyfit(t, r, 1)
    want = np.sqrt(((r - np.polyval(c, t))**2).mean())
    assert np.isclose(res["rms_tilt"][0, 0, 1], want, rtol=1e-6)
    # the residual of a pure tilt is rounding: of order sqrt(eps) of rms
    assert 0 <= res["rms_tilt"][0, 0, 2] <= 1e-7*res["rms"][0, 0, 2]


def test_targets_passed_and_yield():
    sums, N, chief, want = _synthetic(2)
    sw = np.ones(3)
    base = wavefront_tolerance_result(sums, WL, N, sw, chief)
    t = base["poly_rms_tilt"][3].copy()                   # variant 3 exactly on target
    res = wavefront_tolerance_result(sums, WL, N, sw, chief, t)
    with np.errstate(invalid="ignore"):
        ok = (base["poly_rms_tilt"] <= t).all(-1)
    assert np.array_equal(res["passed"], ok) and res["passed"][3]
    assert not res["passed"][1] and not res["passed"][2]   # NaN fails
    assert res["yield"] == ok.mean()
    scalar = wavefront_tolerance_result(sums, WL, N, sw, chief, 1e9)
    assert np.array_equal(scalar["passed"], ~np.isnan(base["poly_rms_tilt"]).any(-1))
    assert "passed" not in base


# ---- the per-variant reference sphere ----------------------------------------
CASES = {
    "cooke": lambda S: [(S - 1, "tilt_x", 1e-3), (S - 1, "tilt_y", -2e-3), (1, "index", 2e-3),
                        (S, "distance", .05), (S - 1, "curvature", 1e-3), (2, "distance", -.02),
                        (S - 2, "tilt_x", 5e-4)],
    "double_gauss": lambda S: [(S - 1, "tilt_y", 7e-4), (S - 1, "tilt_x", -1e-3),
                               (1, "index", 1e-3), (S, "distance", -.03),
                               (S - 1, "conic", -.1), (3, "distance", 1e-2)],
}


def _close(a, b, what):
    a, b = np.asarray(a, float), np.asarray(b, float)
    assert np.all(np.abs(a - b) <= 1e-15*max(np.abs(b).max(), 1e-300)), (what, a, b)


@needs_ref
@pytest.mark.parametrize("name", sorted(CASES))
def test_sphere_specs_match_opd_spec(name):
    """each variant's rtx_opd against lazy.opd_spec of a System with the
    same change, fed the reference's own chief image point: M, d and
    n_after within 1e-15 relative, the rest bit for bit"""
    from rayopt_b200.lazy import opd_spec
    from test_tolerance_host import apply
    R = ref_shim.load()
    s = _reference(name)
    L = len(s)
    W = len(s.wavelengths)
    nominal = np.stack([pack_system(s, l, 1, None, n0=s.refractive_index(l, 0))[0]
                        for l in s.wavelengths])
    S = nominal.shape[1]
    assert S == L - 1
    ei = s[L - 1]
    Ri = np.asarray(ei.rot_normal, float) if getattr(ei, "rotated", False) else np.eye(3)
    cases = CASES[name](S)
    for j, kind, d in cases:
        t = perturbed_tables(nominal, [(j, kind)], [[d]])[0]
        s2 = copy.deepcopy(s)
        apply(s2, j, kind, d)
        s2.update()
        for w, l in enumerate(s.wavelengths):
            tr = R.GeometricTrace(s2)
            tr.rays_point((0, .7), l, nrays=3, distribution="radau", clip=True)
            Y = np.asarray(tr.y[-1, tr.ref], float)
            y0, u0 = np.asarray(tr.y[0, tr.ref], float), np.asarray(tr.u[0, tr.ref], float)
            n_after = float(pack_system(s2, l, 1, None, n0=s2.refractive_index(l, 0))[0][S - 2]["n"])
            want = opd_spec(s2, s2.track, s2.origins, L - 2, L - 1, s2.refractive_index(l, 0),
                            n_after, y0, u0, Y)
            base = opd_spec(s, s.track, s.origins, L - 2, L - 1, s2.refractive_index(l, 0),
                            float(nominal[w, S - 2]["n"]), y0, u0, np.zeros(3))
            got = wavefront_specs(base, t[w][None], Y[None, :2], Ri, s[0].offset,
                                  nominal[w, S - 1])
            assert got.dtype == OPD_DTYPE and got.shape == (1,)
            g = got[0]
            what = (name, j, kind, w)
            _close(g["M"], np.reshape(want["M"], 9), what + ("M",))
            _close(g["d"], want["d"], what + ("d",))
            _close(g["n_after"], want["n_after"], what + ("n_after",))
            assert g["radius"] == base["radius"] and g["n0"] == want["n0"], what
            assert np.array_equal(g["y0_ref"], y0) and np.array_equal(g["u0_ref"], u0), what
            assert g["infinite"] == int(bool(want["infinite"])), what
        if kind in ("tilt_x", "tilt_y") and j == S - 1:
            assert not np.allclose(g["M"], np.eye(3).reshape(9))
