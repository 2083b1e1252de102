"""The restatement of the trace epilogues (oracle/epi_oracle.py) pinned to the
live reference where its tree is present, and the engine's host-side operand
checks for the reductions and epilogues.  No GPU needed."""
import types
import warnings

import numpy as np
import pytest

import epi_oracle
import ref_shim
from conftest import load_golden

needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="no reference tree")


def _reference_trace(R, finite=False, n=400, field=(0, .7)):
    import yaml
    import systems_yaml
    d = yaml.safe_load(systems_yaml.SYSTEMS["cooke"])
    if finite:      # the object 200 mm in front of the first surface
        d["object"] = {"type": "finite", "radius": 20., "pupil": {"radius": 6.25, "aim": True}}
        d["elements"][1]["distance"] = 200.
    s = R.System(**d)
    s.update()
    s.paraxial.refocus()
    s[-1].distance += .2
    g = R.GeometricTrace(s)
    g.rays_point(field, nrays=n, distribution="hexapolar", clip=False)
    return s, g


@pytest.fixture(scope="module")
def R():
    warnings.simplefilter("ignore")
    np.seterr(all="ignore")
    return ref_shim.load()


def _rms(m, unit_weights):
    from rayopt_b200.engine import Engine
    return Engine.rms_from_moments(m, unit_weights=unit_weights)


@needs_ref
@pytest.mark.parametrize("finite", [False, True])
def test_moments_pin_rms_and_refocus(R, finite):
    """rms, rms(ref=...) and the refocus shift of the reference equal what the
    oracle's exact moments of its own stored rows give, to 1e-13"""
    from rayopt_b200.engine import Engine
    s, g = _reference_trace(R, finite)
    y, inc = g.y[-1], g.i[-1]
    c = np.r_[y[0, :2], inc[0, :2]/inc[0, 2]]
    m, _ = epi_oracle.exact_sum(epi_oracle.reduce_terms(y, inc, None, c))
    assert abs(_rms(m, True) - g.rms()) <= 1e-13*g.rms()
    mr, _ = epi_oracle.exact_sum(epi_oracle.moments_terms(y, None, y[3, :2]))
    assert abs(np.sqrt(mr[3]/mr[5]) - g.rms(ref=3)) <= 1e-13*g.rms(ref=3)
    w = np.linspace(1, 2, len(y))/len(y)
    g.w = w
    mw, _ = epi_oracle.exact_sum(epi_oracle.reduce_terms(y, inc, w, c))
    assert abs(_rms(mw, False) - g.rms()) <= 1e-13*g.rms()
    g.w = None
    # the stand-alone focus moments, about the means (refocus re-traces, so
    # they are taken first)
    f, _ = epi_oracle.exact_sum(epi_oracle.focus_terms(y, inc))
    f, _ = epi_oracle.exact_sum(epi_oracle.focus_terms(y, inc, None, f[2:6]/f[0]))
    d0 = s[-1].distance
    g.refocus()
    shift = s[-1].distance - d0
    assert abs(shift) > 1e-3
    assert abs(Engine.focus_shift_from_moments(m) - shift) <= 1e-13*abs(shift)
    assert abs(-f[6]/f[7] - shift) <= 1e-13*abs(shift)


def _spec_of(g, s, after=-2, image=-1, radius=None):
    """the rtx_opd record ResidentMixin.opd_rays builds, from the reference's
    stored rows"""
    after, image = range(len(s))[after], range(len(s))[image]
    if radius is None:
        radius = -s.image.pupil.distance
    ea, ei = s[after], s[image]
    Ra = np.asarray(ea.rot_normal, float) if ea.rotated else np.eye(3)
    Ri = np.asarray(ei.rot_normal, float) if ei.rotated else np.eye(3)
    return after, image, dict(
        y0_ref=g.y[0, g.ref], u0_ref=g.u[0, g.ref], n0=g.n[0], n_after=g.n[after], M=Ra @ Ri.T,
        d=(g.origins[after] - g.origins[image]) @ Ri.T - g.y[image, g.ref], radius=radius,
        infinite=not s.object.finite)


@needs_ref
@pytest.mark.parametrize("finite", [False, True])
def test_opd_pins_reference(R, finite):
    """opd(resample=False): the reference-order restatement is bit-identical
    to the reference; the device-order one (opd_epilogue, what rtx_trace_opd
    computes) is within 1e-9 waves.  The two orders round differently: the
    per-surface subtraction of t[ref] against one path sum, and the frame
    change folded into M and d.  Each rounds at about eps |A| with |A| the
    optical path (~70 mm here), which is eps |A| / l ~ 1e-10 waves after the
    division by the wavelength l (5.9e-4 mm); 1e-9 leaves a factor 10.  The
    finite object takes the branch without the tilted input plane."""
    s, g = _reference_trace(R, finite)
    assert bool(s.object.finite) == finite
    after, image, spec = _spec_of(g, s)
    xr, yr, tr = g.opd(resample=False)
    lam = g.l/s.scale
    x, y, t = epi_oracle.opd_reference_order(
        g.t[:after + 1], g.ref, g.y[0], g.u[0], g.n[0], g.n[after], g.y[after], g.u[after],
        None, None, g.origins[after], g.origins[image], g.y[image, g.ref], spec["radius"],
        spec["infinite"], lam)
    assert np.array_equal(t, tr, equal_nan=True)
    assert np.array_equal(x, xr, equal_nan=True) and np.array_equal(y, yr, equal_nan=True)
    ps = np.zeros(g.y.shape[1])
    for j in range(1, after + 1):            # the device's left-to-right path sum
        ps = ps + g.t[j]
    A, P = epi_oracle.opd_epilogue(g.y[0], g.y[after], g.u[after], ps, spec)
    td = -(A - A[g.ref])/lam
    P = P - P[g.ref]
    assert np.isfinite(td).all()
    assert np.abs(td - tr).max() <= 1e-9
    assert np.abs(P[:, 0] - xr).max() <= 1e-12 and np.abs(P[:, 1] - yr).max() <= 1e-12
    if finite:      # rays from one object point: the tilted plane would add 0
        return
    # the branch matters: the tilted plane changes the OPD by far more than 1e-9
    spec["infinite"] = 0
    A2, _ = epi_oracle.opd_epilogue(g.y[0], g.y[after], g.u[after], ps, spec)
    assert np.abs(-(A2 - A2[g.ref])/lam - tr).max() > 1e-6


def test_sums_equal_the_sharding_stand_in():
    """the oracle's 20 sums equal the numpy stand-in of rtx_trace_reduce in
    test_sharding_gloo.py (its `reducer`), on a vignetted bundle with weights.
    `want` below is a copy of that stand-in's expression: a change to the
    stand-in has to be carried over here."""
    import np_oracle
    c = load_golden("double_gauss_l1_clip")
    Y, U, I, T = np_oracle.trace(c["table"], c["y0"], c["u0"], clip=True)
    center = np.r_[Y[-1, 0, :2], I[-1, 0, :2]/I[-1, 0, 2]]
    w = np.linspace(1, 2, len(c["y0"]))
    cy, cu = center[:2], center[2:]
    d = Y[-1][:, :2] - cy
    s = I[-1][:, :2]/I[-1][:, 2:] - cu
    f, g = np.isfinite(d).all(1), np.isfinite(s).all(1)
    assert 0 < f.sum() < len(f)
    want = np.r_[w[f].sum(), (w[f, None]*d[f]).sum(0), (w[f]*(d[f]**2).sum(1)).sum(),
                 f.sum(), len(w), d[f].sum(0),
                 g.sum(), d[g].sum(0), s[g].sum(0), w[g].sum(), (w[g, None]*d[g]).sum(0),
                 (w[g, None]*s[g]).sum(0), (w[g]*(d[g]*s[g]).sum(1)).sum(),
                 (w[g]*(s[g]**2).sum(1)).sum()]
    got, a = epi_oracle.exact_sum(epi_oracle.reduce_terms(Y[-1], I[-1], w, center))
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-13*a.max())
    assert np.array_equal(got[[4, 5, 8]], want[[4, 5, 8]])


def test_exact_sum_large_n_matches_fsum():
    """the chunked extended-precision path agrees with math.fsum"""
    rng = np.random.default_rng(1)
    t = rng.standard_normal((epi_oracle.FSUM_MAX + 1001, 2))*10.0**rng.integers(-6, 6, (1, 2))
    t[::7] *= -1e3
    big, _ = epi_oracle.exact_sum(t)
    import math
    want = np.array([math.fsum(t[:, j]) for j in range(2)])
    np.testing.assert_allclose(big, want, rtol=1e-15)


class _NoLib:
    def __getattr__(self, name):
        raise AssertionError("%s called: the operands should have been refused first" % name)


def _dev(shape, dtype):
    dtype = np.dtype(dtype)
    return types.SimpleNamespace(shape=tuple(shape), dtype=dtype, ptr=0x1000,
                                 nbytes=int(np.prod(shape))*dtype.itemsize)


def test_engine_refuses_mismatched_operands():
    """Engine.trace_reduce, moments, refocus_shift and trace_opd take the
    element type from the rays: w, inc, A or P of another dtype, or too short
    for N rays, raise ValueError before the library is called"""
    from rayopt_b200.engine import Engine
    eng = object.__new__(Engine)
    eng.lib, eng.ctx = _NoLib(), None
    table = load_golden("cooke_f07_clip")["table"]
    spec = dict(y0_ref=np.zeros(3), u0_ref=np.zeros(3), n0=1., n_after=1., M=np.eye(3),
                d=np.zeros(3), radius=50., infinite=1)
    for dt, other in ((np.float32, np.float64), (np.float64, np.float32)):
        y = _dev((100, 3), dt)
        bad = [
            lambda: eng.trace_reduce(table, y, y, w=_dev((100,), other)),
            lambda: eng.trace_reduce(table, y, y, w=_dev((99,), dt)),
            lambda: eng.trace_reduce(table, y, _dev((100, 3), other)),
            lambda: eng.trace_reduce(table, y, y, N=101),
            lambda: eng.moments(y, _dev((100,), other)),
            lambda: eng.moments(y, _dev((50,), dt), N=100),
            lambda: eng.moments(_dev((1, 64, 3), dt), N=65),
            lambda: eng.refocus_shift(y, _dev((100, 3), other)),
            lambda: eng.refocus_shift(y, _dev((99, 3), dt)),
            lambda: eng.refocus_shift(y, y, w=_dev((100,), other)),
            lambda: eng.trace_opd(table, y, y, spec, _dev((100,), other), _dev((100, 3), dt)),
            lambda: eng.trace_opd(table, y, y, spec, _dev((100,), dt), _dev((100, 3), other)),
            lambda: eng.trace_opd(table, y, y, spec, _dev((99,), dt), _dev((100, 3), dt)),
            lambda: eng.trace_opd(table, y, y, spec, _dev((100,), dt), _dev((33, 3), dt)),
        ]
        for k, call in enumerate(bad):
            with pytest.raises(ValueError):
                call()


def test_aim_refuses_given_pupil_coordinates_not_fp64():
    """the ray generator reads given pupil coordinates as FP64 for FP64 and
    FP32 bundles alike: an array of another type raises ValueError before the
    library is called"""
    from rayopt_b200.engine import Engine
    from rayopt_b200.rays import infinite_record
    eng = object.__new__(Engine)
    eng.lib, eng.ctx = _NoLib(), None
    p = np.array(((-3., -2.5), (2., 2.8)))
    rec = infinite_record((0, .5), 30., p, .2)
    y = _dev((100, 3), np.float32)
    for dt in (np.float32, np.float16):
        yp = _dev((100, 2), dt)
        bad = [
            lambda: eng.aim_infinite_device((0, .5), 30., p, .2, yp=yp, dtype=np.float32),
            lambda: eng.aim_finite_device((0, .5), 30., p, 5., yp=yp),
            lambda: eng.aim_rays(rec, yp=yp),
            lambda: eng.aim_rays_into(rec, y, y, 100, yp=yp),
            lambda: eng.aim_count(rec, yp),
        ]
        for call in bad:
            with pytest.raises(ValueError):
                call()
    with pytest.raises(AssertionError, match="called"):
        eng.aim_count(rec, _dev((100, 2), np.float64))


def test_trace_device_refuses_mismatched_operands():
    """Engine.trace_device, trace_device_batch and trace_gather: an output or
    path sum of another dtype than the rays, an output smaller than rows x ld
    rays, a path sum shorter than N or a mask that is not ceil(N/32) 32-bit
    words raise ValueError before the library is called"""
    from rayopt_b200.engine import Engine
    eng = object.__new__(Engine)
    eng.lib, eng.ctx = _NoLib(), None
    table = load_golden("cooke_f07_clip")["table"]
    S = len(table)
    for dt, other in ((np.float32, np.float64), (np.float64, np.float32)):
        y = _dev((100, 3), dt)
        Y, T = _dev((S, 128, 3), dt), _dev((S, 128), dt)
        bad = [
            lambda: eng.trace_device(table, y, y, _dev((S, 128, 3), other), None, None, None),
            lambda: eng.trace_device(table, y, y, None, None, None, _dev((S, 128), other), ld=128),
            lambda: eng.trace_device(table, y, y, Y, _dev((S, 127, 3), dt), None, None, ld=128),
            lambda: eng.trace_device(table, y, y, None, None, None, _dev((S - 1, 128), dt), ld=128),
            lambda: eng.trace_device(table, y, y, _dev((1, 128, 3), dt), None, None, None),
            lambda: eng.trace_device(table, y, y, Y, None, None, T, ld=256),
            lambda: eng.trace_device(table, y, y, None, None, None, None, path_sum=_dev((100,), other)),
            lambda: eng.trace_device(table, y, y, None, None, None, None, path_sum=_dev((99,), dt)),
            lambda: eng.trace_device(table, y, y, None, None, None, None,
                                     mask=_dev((4,), np.uint64)),
            lambda: eng.trace_device(table, y, y, None, None, None, None,
                                     mask=_dev((3,), np.uint32)),
            lambda: eng.trace_device(table, y, _dev((100, 3), other), Y, None, None, None),
            lambda: eng.trace_device(table, y, y, Y, None, None, None, N=129),
            lambda: eng.trace_device_batch([table]*2, [y, y], [y, y], [Y, _dev((S, 128, 3), other)],
                                           None, None, None),
            lambda: eng.trace_device_batch([table]*2, [y, y], [y, y], [Y, _dev((S, 64, 3), dt)],
                                           None, None, None, ld=128),
            lambda: eng.trace_gather(table, y, y, [0x1000], 0, path_sum=_dev((100,), other)),
            lambda: eng.trace_gather(table, y, y, [0x1000], 0, mask=_dev((3,), np.uint32)),
        ]
        for k, call in enumerate(bad):
            with pytest.raises(ValueError):
                call()
        # operands that fit get through to the library
        with pytest.raises(AssertionError, match="called"):
            eng.trace_device(table, y, y, Y, None, None, T, mask=_dev((4,), np.uint32),
                             path_sum=_dev((100,), dt))
        with pytest.raises(AssertionError, match="called"):
            eng.trace_device(table, y, y, _dev((1, 128, 3), dt), None, None, None, keep_last=True)
