"""The drop-in wiring ON HARDWARE against the REAL reference.

The reference (staged under oracle/_ref by oracle/make_ref.py, or found
through $RAYOPT_REFERENCE) runs on the host; its own ``GeometricTrace`` / ``System``
classes are bound to the CUDA engine with ``rayopt_b200.bind`` /
``rayopt_b200.install`` and driven through the reference's own call patterns:

* ``rays_point`` / ``rays_clipping`` / ``rays_line`` / ``refocus`` / ``rms`` /
  ``opd``                      rayopt/geometric_trace.py:82-144,171-229
* ``System.aim_chief`` / ``aim_marginal`` / ``pupil``   rayopt/system.py:507-593
  (hundreds of 1-3 ray traces through the small-bundle CUDA path)
* the consumers of ``Analysis``  rayopt/analysis.py:231-245,269-280
  (``y[-1]``, ``i[-1]``, ``y[0]``, ``u[0]`` of tee / hexapolar bundles)
* the reference's own integration tests rayopt/test/test_raytrace.py:151-199

RTX_EXACT results must be BIT-IDENTICAL to the reference on the unrotated
analytic lenses; the default fast mode within 1e-10 (SURVEY 8d comparator).
"""
import warnings

import numpy as np
import pytest
import yaml

import ref_shim
import systems_yaml
from conftest import assert_parity

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not ref_shim.available(),
                                 reason="no reference tree (oracle/make_ref.py stages one "
                                        "from $RAYOPT_REFERENCE)")]


@pytest.fixture(scope="module")
def R():
    warnings.simplefilter("ignore")
    np.seterr(all="ignore")
    return ref_shim.load()


@pytest.fixture(scope="module")
def eng():
    from rayopt_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def build(R, name, cls=None, defocus=0.):
    s = (cls or R.System)(**yaml.safe_load(systems_yaml.SYSTEMS[name]))
    s.update()
    s.paraxial.refocus()
    if defocus:
        s[-1].distance += defocus
    return s


def same(got, ref, exact, what=""):
    for k in "yuit":
        a, b = np.asarray(getattr(got, k)), getattr(ref, k)
        if exact:
            assert np.array_equal(a, b, equal_nan=True), (what, k)
        else:
            assert_parity(a, b, 1e-10, "%s %s" % (what, k))
    assert np.array_equal(got.n, ref.n), what


CALLS = [
    ("rays_point", ((0, 1.),), dict(nrays=300, distribution="hexapolar", clip=True)),
    ("rays_point", ((0, .7),), dict(nrays=152, distribution="tee", clip=True)),
    ("rays_point", ((0, .5),), dict(nrays=9, distribution="meridional")),
    ("rays_point", ((0, 1.),), dict(nrays=13, distribution="radau", filter=False)),
    ("rays_clipping", ((0, 1.),), {}),
    ("rays_line", ((0, 1.),), dict(nrays=5)),
    ("rays_paraxial", (), {}),
]


@pytest.mark.parametrize("resident", [False, True])
@pytest.mark.parametrize("exact", [True, False])
@pytest.mark.parametrize("lens", ["cooke", "double_gauss"])
def test_bound_reference_trace_on_cuda(R, eng, lens, exact, resident):
    """bind(rayopt.GeometricTrace): the reference's own ray-launch helpers run
    on the CUDA engine (host arrays, or resident LazyRows) and reproduce the
    reference's trace of the same System"""
    from rayopt_b200 import bind
    s = build(R, lens)
    GT = bind(R.GeometricTrace, engine=eng, exact=exact, resident=resident)
    l0 = eng.launch_count()
    for fn, args, kw in CALLS:
        ref, got = R.GeometricTrace(s), GT(s)
        getattr(ref, fn)(*args, **kw)
        getattr(got, fn)(*args, **kw)
        same(got, ref, exact, "%s %s %s" % (lens, fn, kw.get("distribution", "")))
        assert got.ref == ref.ref and np.array_equal(got.w, ref.w)
        assert np.array_equal(got.path, ref.path) and np.array_equal(got.origins, ref.origins)
    assert eng.launch_count() - l0 >= len(CALLS)


@pytest.mark.parametrize("resident", [False, True])
def test_refocus_rms_opd_of_the_reference_class_on_cuda(R, eng, resident):
    """refocus (geometric_trace.py:82-99), rms (:171-183) and opd (:101-144) of
    the bound class against the reference on a defocused lens"""
    from rayopt_b200 import bind
    s1, s2 = build(R, "double_gauss", defocus=.3), build(R, "double_gauss", defocus=.3)
    GT = bind(R.GeometricTrace, engine=eng, exact=True, resident=resident)
    ref, got = R.GeometricTrace(s1), GT(s2)
    kw = dict(nrays=400, distribution="hexapolar", clip=True, filter=False)
    ref.rays_point((0, .7), **kw)
    got.rays_point((0, .7), **kw)
    same(got, ref, True, "before refocus")
    d0 = s1[-1].distance
    ref.refocus()
    got.refocus()
    assert abs(s1[-1].distance - d0) > 1e-3               # it had work to do
    assert abs((s1[-1].distance - d0) - (s2[-1].distance - d0)) < 1e-11
    assert_parity(np.asarray(got.y)[-1:], ref.y[-1:], 1e-10, "after refocus")
    # rms / opd need a bundle without vignetted rays
    ref.rays_point((0, 0.), nrays=200, distribution="hexapolar", clip=False)
    got.rays_point((0, 0.), nrays=200, distribution="hexapolar", clip=False)
    assert abs(got.rms() - ref.rms()) < 1e-13
    assert abs(got.rms(ref=0) - ref.rms(ref=0)) < 1e-13
    assert abs(got.rms(3) - ref.rms(3)) < 1e-12
    xr, yr, tr = ref.opd(resample=False)
    xg, yg, tg = got.opd(resample=False)       # resident: the device epilogue rtx_trace_opd
    np.testing.assert_allclose(tg, tr, rtol=0, atol=1e-9)  # waves
    np.testing.assert_allclose(xg, xr, rtol=0, atol=1e-12)
    np.testing.assert_allclose(yg, yr, rtol=0, atol=1e-12)
    xr, yr, tr = ref.opd()
    xg, yg, tg = got.opd()
    assert np.array_equal(np.isnan(tg), np.isnan(tr))
    np.testing.assert_allclose(np.nan_to_num(tg), np.nan_to_num(tr), rtol=0, atol=1e-8)
    if resident:
        # fused epilogues: one launch from row 0, nothing stored or read back
        assert abs(got.rms_fused() - ref.rms()) < 1e-13
        assert abs(got.rms_fused(3) - ref.rms(3)) < 1e-12
        for t in (ref, got):
            t.rays_point((0, .7), **kw)
        d1, d2 = s1[-1].distance, s2[-1].distance
        shift = got.refocus_fused(clip=True)
        ref.refocus()
        assert abs(shift - (s1[-1].distance - d1)) < 1e-11 and s2[-1].distance == d2 + shift
        got.free()


def test_fused_reduce_large_bundle(R, eng):
    """rtx_trace_reduce on a 3e5-ray aimed bundle: rms / centroid / vignetting
    count / focus shift from ONE launch equal the reference's numbers computed
    from its stored trace"""
    from rayopt_b200 import bind
    s = build(R, "double_gauss", defocus=.2)
    n = 300001
    rng = np.random.default_rng(11)
    r, phi = np.sqrt(rng.random(n)), 2*np.pi*rng.random(n)
    yp = np.c_[r*np.cos(phi), r*np.sin(phi)]
    yp[0] = 0
    w = rng.random(n)
    w /= w.sum()
    ref = R.GeometricTrace(s)
    got = bind(R.GeometricTrace, engine=eng, resident=True)(s)
    for t in (ref, got):
        t.rays((0, .7), yp, s.wavelengths[1], clip=True, filter=False, weight=w)
    m, c = got.reduce(clip=True)
    good = np.isfinite(ref.y[-1, :, 0])
    assert m[5] == n and m[4] == good.sum() and 0 < good.sum() < n
    y = ref.y[-1, good, :2]
    np.testing.assert_allclose(c[:2] + m[6:8]/m[4], y.mean(0), rtol=1e-13)
    np.testing.assert_allclose(m[0], w[good].sum(), rtol=1e-12)
    u = R.utils.tanarcsin(ref.i[-1])
    ok = np.all(np.isfinite(u), axis=1)
    yy, uu, ww = ref.y[-1, ok, :2], u[ok], w[ok]
    yy, uu = yy - yy.mean(0), uu - uu.mean(0)
    want = -np.dot((ww[:, None]*yy).ravel(), uu.ravel())/np.dot((ww[:, None]*uu).ravel(), uu.ravel())
    assert abs(eng.focus_shift_from_moments(m) - want) < 1e-10*abs(want)
    # rms needs an unvignetted bundle (the reference's rms is not NaN-masked)
    for t in (ref, got):
        t.rays((0, 0.), yp[:100000], s.wavelengths[0], clip=True, filter=False)
    assert abs(got.rms_fused(clip=True) - ref.rms()) < 1e-12*ref.rms() + 1e-15
    assert abs(got.rms_fused(5, clip=True) - ref.rms(5)) < 1e-12*ref.rms(5)
    got.free()


@pytest.mark.parametrize("resident", [False, True])
def test_text_and_resize_of_the_reference_class(R, eng, resident):
    """the reference's report / housekeeping methods run unchanged on the bound
    class: ``str(trace)`` (print_trace: cumsum of t, per-ray rows,
    geometric_trace.py:241-259) and ``resize`` (:231-234)"""
    from rayopt_b200 import bind
    s1, s2 = build(R, "cooke"), build(R, "cooke")
    ref = R.GeometricTrace(s1)
    got = bind(R.GeometricTrace, engine=eng, exact=True, resident=resident)(s2)
    for t in (ref, got):
        t.rays_point((0, .7), nrays=7, distribution="meridional")
    assert str(got) == str(ref) and len(str(ref)) > 500
    ref.resize(fn=lambda a, b: a)
    got.resize(fn=lambda a, b: a)
    assert [e.radius for e in s1[1:]] == [e.radius for e in s2[1:]]


def test_analysis_consumers_read_single_rows(R, eng):
    """what Analysis.transverse / spots read (analysis.py:231-245,269-280) from
    a resident bound trace: only the rows asked for cross PCIe"""
    from rayopt_b200 import bind
    s = build(R, "cooke")
    GT = bind(R.GeometricTrace, engine=eng, exact=True, resident=True)
    tanarcsin = R.utils.tanarcsin
    p = s.object.pupil.distance
    for hi, wi in ((1., s.wavelengths[0]), (.707, s.wavelengths[2])):
        ref, got = R.GeometricTrace(s), GT(s)
        for t in (ref, got):
            t.rays_point((0, hi), wi, nrays=152, distribution="tee", clip=True)
        y, yr = got.y[-1, :, :2] - got.y[-1, got.ref, :2], ref.y[-1, :, :2] - ref.y[-1, ref.ref, :2]
        assert np.array_equal(y, yr, equal_nan=True)
        py = got.y[0, :, :2] + p*tanarcsin(got.u[0])
        assert np.array_equal(py, ref.y[0, :, :2] + p*tanarcsin(ref.u[0]))
        rows = len(s)
        assert got.y.fetched_bytes == 2*got.nrays*24 and got.u.fetched_bytes == got.nrays*24
        assert got.t.fetched_bytes == 0 and rows > 3
        for t in (ref, got):
            t.rays_point((0, hi), wi, nrays=150, distribution="hexapolar", clip=True)
        assert np.array_equal(tanarcsin(got.i[-1]), tanarcsin(ref.i[-1]), equal_nan=True)
        assert np.array_equal(got.y[-1], ref.y[-1], equal_nan=True)
        got.free()


def test_installed_system_aims_through_the_cuda_path(R, eng):
    """install(System): aim_chief / aim_marginal (system.py:507-555) issue
    their 1-3 ray traces through rtx_trace_host's small-bundle path; the pupil
    solution equals the unpatched reference's, and the reference's own
    integration tests (test_raytrace.py:151-199) pass on the patched classes"""
    import rayopt_b200

    class System(R.System):          # patched copies: leave the shared classes alone
        pass

    class Trace(R.GeometricTrace):
        pass
    rayopt_b200.install(System, Trace, engine=eng, exact=True)
    s = build(R, "cooke", System)
    s.paraxial.update_conjugates()
    s0 = build(R, "cooke")
    s0.paraxial.update_conjugates()
    l0 = eng.launch_count()
    for yo in ((0, 1.), (0, .5), (.3, .6)):
        z1, p1 = s.pupil(yo)
        z0, p0 = s0.pupil(yo)
        np.testing.assert_allclose(z1, z0, rtol=1e-12)
        np.testing.assert_allclose(p1, p0, rtol=1e-12)
    z1, p1 = s.pupil((0, 1.), stop=-1)
    z0, p0 = s0.pupil((0, 1.), stop=-1)
    np.testing.assert_allclose(p1, p0, rtol=1e-12)
    assert eng.launch_count() - l0 > 50           # aiming really ran on the GPU
    g = Trace(s)
    # test_aim_point
    g.rays_point((0, 1.))
    g.rays_clipping((0, 1.))
    g.rays_line((0, 1.))
    # test_aim_point_more
    i = s.stop
    r = np.array([el.radius for el in s[1:-1]])
    g.rays_clipping((0, 1.))
    np.testing.assert_allclose(g.u[0, :, :], g.u[0, (0,)*g.u.shape[1], :])
    np.testing.assert_allclose(g.y[i, 0, 1], 0, atol=5e-3)
    np.testing.assert_allclose(min(g.y[1:-1, 1, 1] + r), 0, atol=1e-3)
    np.testing.assert_allclose(max(g.y[1:-1, 2, 1] - r), 0, atol=1e-3)
    g.rays_point((0, 1.), distribution="cross", nrays=5, filter=False)
    np.testing.assert_allclose(g.y[i, :3, 1]/s[i].radius, [-1, 0, 1], atol=1e-3, rtol=3e-2)
    np.testing.assert_allclose(g.y[i, :, 0]/s[i].radius, [0, 0, 0, -1, 0, 1], atol=1e-1)
    # test_quadrature: the known answer of the path
    g.rays_point((0, 1.), nrays=13, distribution="radau", filter=False)
    a = g.rms()
    np.testing.assert_allclose(a, .052, rtol=1e-2)
    g.rays_point((0, 1.), nrays=500, distribution="square", clip=False, filter=True)
    np.testing.assert_allclose(a, g.rms(), rtol=5e-2)
    # and the traces equal the unpatched reference's
    g0 = R.GeometricTrace(s0)
    g0.rays_point((0, 1.), nrays=13, distribution="radau", filter=False)
    g.rays_point((0, 1.), nrays=13, distribution="radau", filter=False)
    assert_parity(g.y, g0.y, 1e-10, "installed y")


@pytest.mark.parametrize("lens,n", [("cooke_asph", 2000), ("mirror", 3000), ("zoom", 20000)])
def test_bound_trace_other_lenses(R, eng, lens, n):
    """aspheres (Newton), the folded mirror (rotated frames: `i` is a real
    array) and the 20-surface zoom through the bound class, default fast mode"""
    from rayopt_b200 import bind
    s = build(R, lens)
    GT = bind(R.GeometricTrace, engine=eng)
    ref, got = R.GeometricTrace(s), GT(s)
    rng = np.random.default_rng(3)
    r, phi = np.sqrt(rng.random(n)), 2*np.pi*rng.random(n)
    yp = np.c_[r*np.cos(phi), r*np.sin(phi)]
    for t in (ref, got):
        t.rays((0, .7), yp, s.wavelengths[0], clip=lens != "mirror", filter=False)
    same(got, ref, False, lens)
    res = bind(R.GeometricTrace, engine=eng, resident=True)(s)
    res.rays((0, .7), yp, s.wavelengths[0], clip=lens != "mirror", filter=False)
    same(res, ref, False, lens + " resident")
    res.free()


def test_batched_host_front_end(R, eng):
    """rtx_trace_batch_host / propagate_many: Analysis' 3 fields x 3 wavelengths
    of 150-ray hexapolar bundles (analysis.py:266-280), plus ragged sizes and
    more than 8 bundles, in ONE call -- bit-identical (RTX_EXACT) to the
    reference's own rays_point loops"""
    import rayopt_b200
    s = build(R, "cooke")
    GT = rayopt_b200.bind(R.GeometricTrace, engine=eng, exact=True)
    refs, traces = [], []
    for k, hi in enumerate((1., .707, 0., .3)):
        for wi in s.wavelengths:
            n = 150 + 37*k
            ref_, yp, weight = R.utils.pupil_distribution("hexapolar", n)
            r = R.GeometricTrace(s)
            r.rays_point((0, hi), wi, nrays=n, distribution="hexapolar", clip=True)
            refs.append(r)
            t = GT(s)
            z, p = s.pupil((0, hi), l=wi)
            t.rays_given(*s.aim((0, hi), yp, z, p, filter=False), wi, weight, ref_)
            traces.append(t)
    assert len(traces) == 12
    l0 = eng.launch_count()
    rayopt_b200.propagate_many(traces, clip=True)
    assert eng.launch_count() - l0 == 2              # 8 + 4 bundles: two launches
    for r, t in zip(refs, traces):
        same(t, r, True, "batched")
    # the raw call: ragged bundles incl. a single ray and an empty one, keep-LAST
    from rayopt_b200.surface_table import pack_system
    table, _, _ = pack_system(s, s.wavelengths[0])
    ys = [refs[0].y[0], refs[3].y[0][:1], refs[6].y[0][:0], refs[9].y[0]]
    us = [refs[0].u[0], refs[3].u[0][:1], refs[6].u[0][:0], refs[9].u[0]]
    out = eng.trace_bundles([table]*4, ys, us, clip=True, keep_last=True, exact=True,
                            want=("y", "t"))
    for (Y, U, I, T), y0, u0 in zip(out, ys, us):
        want = eng.trace(table, y0, u0, clip=True, keep_last=True, exact=True) if len(y0) else None
        assert U is None and I is None and Y.shape == (1, len(y0), 3)
        if want is not None:
            assert np.array_equal(Y, want[0], equal_nan=True) and np.array_equal(T, want[3], equal_nan=True)
