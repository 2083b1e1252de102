"""Host side of the MTF tolerance analysis (rayopt_b200.tolerance_mtf): its
refusals before any device work, the result assembly against direct numpy,
the variant chunk's byte budget, and the many-item OTF oracle
(tests/otf_many_oracle.py) against mpmath.  No GPU."""
import warnings

import numpy as np
import pytest

import otf_many_oracle as om
import ref_shim
from rayopt_b200.mtf import poly_otf
from rayopt_b200.tolerance import _variant_chunk, mtf_tolerance_result, tolerance_mtf
from test_tolerance_driver_host import _NoEngine, _StubSystem

needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="no reference tree staged")


@pytest.mark.parametrize("kw, msg", [
    (dict(freqs=[]), "frequencies"),
    (dict(freqs=[1., np.nan]), "frequencies"),
    (dict(freqs=np.arange(257.)), "frequencies"),
    (dict(defocus=[]), "defocus"),
    (dict(defocus=[0., np.inf]), "defocus"),
    (dict(defocus=np.zeros(17)), "defocus"),
    (dict(defocus=np.zeros((2, 2))), "defocus"),
    (dict(targets=np.ones(5)), "targets"),
    (dict(targets=np.ones((4, 2, 3))), "targets"),
    (dict(spectral_weights=[1., 2.]), "spectral_weights"),
    (dict(spectral_weights=[1., np.nan, 1.]), "spectral_weights"),
    (dict(compensate="tilt"), "compensate"),
    (dict(chunk=0), "chunk"),
])
def test_refusals_before_device_work(kw, msg):
    args = dict(params=[(1, "curvature")], deltas=np.zeros((2, 1)), freqs=[10., 20., 30.])
    args.update(kw)
    with pytest.raises(ValueError, match=msg):
        tolerance_mtf(_StubSystem(), engine=_NoEngine(), **args)


@needs_ref
@pytest.mark.parametrize("kw, msg", [
    (lambda S: dict(params=[(S + 1, "curvature")]), "not in"),
    (lambda S: dict(params=[(1, "bogus")]), "unknown tolerance kind"),
    (lambda S: dict(params=[(S, "index")]), "is the last"),
    (lambda S: dict(deltas=np.zeros((3, 2))), "deltas must be"),
    (lambda S: dict(deltas=np.zeros((2, 1, 1))), "deltas must be"),
])
def test_perturbed_tables_refusals_before_device_work(kw, msg):
    """`kw` of the number of surfaces S"""
    import yaml
    import systems_yaml
    from rayopt_b200.surface_table import pack_system
    warnings.simplefilter("ignore")
    R = ref_shim.load()
    s = R.System(**yaml.safe_load(systems_yaml.SYSTEMS["cooke"]))
    s.update()
    args = dict(params=[(1, "curvature")], deltas=np.zeros((2, 1)), freqs=[10.])
    with np.errstate(all="ignore"):
        args.update(kw(len(pack_system(s, s.wavelengths[0], 1, None)[0])))
        with pytest.raises(ValueError, match=msg):
            tolerance_mtf(s, engine=_NoEngine(), **args)


def _synthetic(seed, V=4, H=3, W=3, K=2, F=5):
    rng = np.random.default_rng(seed)
    count = rng.integers(0, 50, (V, H, W, K))
    count[0, 0, :, 0] = 0                       # no wavelength counts: NaN poly
    count[1, 2, 1, 1] = 0                       # one wavelength counts nothing
    phase = rng.uniform(-np.pi, np.pi, (V, H, W, K, 2, F))
    amp = rng.uniform(0, 1, (V, H, W, K, 2, F))*count[..., None, None]
    sums = np.where(count[..., None, None] > 0, amp*np.exp(1j*phase), 0)
    return sums, count


def test_result_assembly_against_numpy():
    sums, count = _synthetic(1)
    V, H, W, K, _, F = sums.shape
    sw = np.array([1., 2., .5])
    with np.errstate(all="ignore"):
        otf = sums/count[..., None, None]
    poly = np.array([poly_otf(otf[v], count[v], sw) for v in range(V)])
    # targets on the boundary of one variant's poly MTF pass
    t = np.abs(poly[2, :, 1]).copy()
    res = mtf_tolerance_result(sums, count, sw, t)
    assert np.array_equal(np.isnan(res["otf"]), np.isnan(otf))
    fin = np.isfinite(otf)
    assert np.array_equal(res["otf"][fin], otf[fin])
    assert np.array_equal(res["mtf"][fin], np.abs(otf[fin]))
    assert res["count"].dtype == np.int64 and np.array_equal(res["count"], count)
    assert np.array_equal(np.isnan(res["poly"]), np.isnan(poly))
    assert np.isnan(res["poly"][0, 0, 0]).all()
    fp = np.isfinite(poly)
    assert np.array_equal(res["poly"][fp], poly[fp])
    assert np.array_equal(res["poly_mtf"][fp], np.abs(poly[fp]))
    with np.errstate(invalid="ignore"):
        want = (np.abs(poly) >= t[:, None]).all(axis=(1, 3, 4))
    assert np.array_equal(res["passed"], want)
    assert res["passed"][2, 1]                   # exactly on target
    assert not res["passed"][0, 0]               # NaN fails
    assert np.array_equal(res["yield"], want.mean(0))
    assert "passed" not in mtf_tolerance_result(sums, count, sw)


def test_result_assembly_scalar_and_per_frequency_targets():
    sums, count = _synthetic(2)
    sw = np.ones(3)
    a = mtf_tolerance_result(sums, count, sw, .3)
    b = mtf_tolerance_result(sums, count, sw, np.full((3, 2, 5), .3))
    c = mtf_tolerance_result(sums, count, sw, np.full(5, .3))
    assert np.array_equal(a["passed"], b["passed"]) and np.array_equal(a["passed"], c["passed"])
    none = mtf_tolerance_result(sums, count, sw, 0.)
    # zero targets: every plane passes unless a poly MTF is NaN
    assert np.array_equal(none["passed"], ~np.isnan(none["poly_mtf"]).any(axis=(1, 3, 4)))


@pytest.mark.parametrize("K, F", [(1, 3), (5, 16), (16, 256)])
def test_variant_chunk_fits_the_budget(K, F):
    tables, tiles, items, budget = 3*10*512, 9*20, 9, 2**30
    row = 8*(4*K*F + K)
    n = _variant_chunk(tables, tiles, budget, row, items)
    per = tables + row*(tiles + items)
    assert n*per <= budget < (n + 1)*per + n + 1
    assert _variant_chunk(tables, tiles, budget) == _variant_chunk(tables, tiles, budget, 160, 0)
    assert _variant_chunk(tables, 10**9, 1000, row, items) == 1          # at least one


def _rays(seed, n):
    rng = np.random.default_rng(seed)
    y = np.c_[rng.normal(0, 2e-2, (n, 2)), np.zeros(n)]
    i = np.c_[rng.normal(0, .1, (n, 2)), np.ones(n)]
    i /= np.linalg.norm(i, axis=1)[:, None]
    y[1, 0] = np.nan                             # counts nowhere
    i[2, 2] = 0.                                 # i_z = 0: counts nowhere, even at z = 0
    i[3, :] = [0., 0., 0.]
    y[4, 1] = np.inf
    return y, i


def test_points_follow_the_kernel_rounding():
    y, i = _rays(3, 30)
    c = np.array([1e-3, -2e-3])
    z = np.array([0., 1e-2, -1e-2])
    q = om.points(y, i, c, z)
    for k, zk in enumerate(z):
        for r in range(30):
            with np.errstate(all="ignore"):
                d = np.float64(y[r, 0]) - np.float64(c[0])
                u = np.float64(i[r, 0])/np.float64(i[r, 2])
                want = d + np.float64(zk)*u
            assert np.array_equal(q[k, r, 0], want, equal_nan=True)
    _, _, count, _ = om.sums(y, i, c, z, [0., 10.])
    assert (count == 26).all()                   # rays 1..4 never count


def test_oracle_against_mpmath():
    mp = pytest.importorskip("mpmath")
    mp.mp.dps = 40
    y, i = _rays(4, 36)
    c = np.array([.003, -.01])
    z = np.array([0., 1e-2, -1e-2])
    nu = np.array([0., 10., 30., -52.5])
    re, im, count, phi = om.sums(y, i, c, z, nu)
    q = om.points(y, i, c, z)
    for k in range(len(z)):
        ok = np.isfinite(q[k]).all(1)
        assert count[k] == ok.sum() == 32
        tol = om.oracle_error(count[k:k + 1], phi[k:k + 1])[0]*count[k]
        for a in range(2):
            for j in range(len(nu)):
                S = mp.mpc(0)
                for x in q[k, ok, a]:
                    S += mp.exp(-2j*mp.pi*mp.mpf(nu[j])*mp.mpf(x))
                assert abs(float(S.real) - float(re[k, a, j])) <= tol
                assert abs(float(S.imag) - float(im[k, a, j])) <= tol
        assert np.array_equal(re[k, :, 0], np.full(2, count[k]))     # nu = 0: the count
