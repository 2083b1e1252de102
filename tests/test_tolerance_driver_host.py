"""Host side shared by the four tolerance analyses (tolerance,
tolerance_mtf, tolerance_wavefront, tolerance_zernike) through
tolerance.VariantMarch: the refusals every one makes before any device work,
and the device calls each makes, recorded by a stand-in engine: one launch
per chunk of variants, each on its chunk's perturbed (and refocused) tables
with height-major items, and nothing left on the device on any exit.  No
GPU."""
import copy
import warnings

import numpy as np
import pytest

import ref_shim
from rayopt_b200.tolerance import (_move_distance, _nominal, perturbed_tables, sensitivity_deltas,
                                   tolerance, tolerance_mtf, tolerance_wavefront)
from rayopt_b200.zernike import tolerance_zernike

needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="no reference tree staged")


class _NoEngine:
    def __getattr__(self, name):
        raise AssertionError("device work before the refusal: %s" % name)


class _StubSystem:
    """what the argument refusals read of a System: its wavelengths"""
    wavelengths = [5.8756e-07, 6.5627e-07, 4.8613e-07]


# analysis, its own required arguments, the launches it makes per chunk of
# variants (the last is the variant launch) and before the focus pass
ANALYSES = {
    "tolerance": (tolerance, {}, ["trace_reduce_many"], 0),
    "tolerance_mtf": (tolerance_mtf, dict(freqs=[10., 20.]), ["trace_otf_many"], 0),
    "tolerance_wavefront": (tolerance_wavefront, {},
                            ["trace_reduce_many", "trace_opd_many", "trace_opd_many"], 0),
    "tolerance_zernike": (tolerance_zernike, dict(order=2),
                          ["trace_reduce_many", "trace_opd_many", "trace_zernike_many"], 3),
}
WAVEFRONT = ("tolerance_wavefront", "tolerance_zernike")


def _run(name, system, engine, **kw):
    fn, args, _, _ = ANALYSES[name]
    args = dict(args, params=[(1, "curvature")], deltas=np.zeros((2, 1)))
    args.update(kw)
    return fn(system, engine=engine, **args)


@pytest.mark.parametrize("name", list(ANALYSES))
@pytest.mark.parametrize("kw, msg", [
    (dict(compensate="tilt"), "compensate"),
    (dict(chunk=0), "chunk"),
    (dict(chunk=-1), "chunk"),
    (dict(heights=[]), "height"),
    (dict(wavelengths=[]), "wavelength"),
])
def test_shared_refusals(name, kw, msg):
    with pytest.raises(ValueError, match=msg):
        _run(name, _StubSystem(), _NoEngine(), **kw)


def _cooke():
    import yaml
    import systems_yaml
    warnings.simplefilter("ignore")
    np.seterr(all="ignore")
    s = ref_shim.load().System(**yaml.safe_load(systems_yaml.SYSTEMS["cooke"]))
    s.update()
    s.paraxial.refocus()
    return s


@needs_ref
@pytest.mark.parametrize("name", list(ANALYSES))
@pytest.mark.parametrize("kw, msg", [
    (lambda S: dict(params=[(S + 1, "curvature")]), "not in"),
    (lambda S: dict(params=[(0, "curvature")]), "not in"),
    (lambda S: dict(params=[(1, "bogus")]), "unknown tolerance kind"),
    (lambda S: dict(deltas=np.zeros((3, 2))), "deltas must be"),
    (lambda S: dict(params=[(S, "curvature")]), "image surface"),
    (lambda S: dict(params=[(S, "tilt_y")]), "image surface"),
])
def test_lens_refusals(name, kw, msg):
    """`kw` of the number of surfaces S; a shape or tilt of the image surface
    is refused by the two wavefront analyses only"""
    s = _cooke()
    args = kw(_nominal(s, s.wavelengths)[0].shape[1])
    if msg == "image surface" and name not in WAVEFRONT:
        with pytest.raises(AssertionError, match="device work"):
            _run(name, s, _NoEngine(), **args)
    else:
        with pytest.raises(ValueError, match=msg):
            _run(name, s, _NoEngine(), **args)


# ---- the device calls, recorded ---------------------------------------------
class _Dev:
    """a device array stand-in"""

    def __init__(self, eng, shape, data, owner=True):
        self.eng, self.shape, self.data, self.dtype = eng, tuple(shape), data, np.dtype(np.float64)
        if owner:
            eng.live.add(self)

    def download(self):
        assert self in self.eng.live, "download of a freed array"
        return self.data.copy()

    def free(self):
        assert self in self.eng.live, "double free"
        self.eng.live.discard(self)

    def rows(self, r0, r1=None):
        d = self.data[r0:r1]
        return _Dev(self.eng, d.shape, d, owner=False)


class _Recorder:
    """an Engine stand-in that records every call and returns seeded values;
    it raises at the `fail`-th clipped *_many launch"""
    NRAYS = 600

    def __init__(self, fail=None):
        self.calls, self.live, self.fail, self.rng = [], set(), fail, np.random.default_rng(0)

    def _call(self, name, *args, **kw):
        for b in (args[1] if name.endswith("_many") else ()):
            assert b[0] in self.live and b[1] in self.live, "%s of a freed bundle" % name
        self.calls.append((name, args, kw))
        launches = [c for c in self.calls if c[0].endswith("_many") and c[2]["clip"]]
        if name.endswith("_many") and kw["clip"] and len(launches) - 1 == self.fail:
            raise RuntimeError("launch %d failed" % self.fail)
        return self.rng

    def aim_rays(self, rec, first=0, count=None, yp=None):
        rng = self._call("aim_rays", rec, first=first, count=count, yp=yp)
        n = count if count is not None else yp.shape[0] if yp is not None else self.NRAYS
        return tuple(_Dev(self, (n, 3), rng.uniform(-1, 1, (n, 3))) for _ in range(2))

    def to_device(self, a):
        self._call("to_device", a)
        return _Dev(self, np.shape(a), np.array(a))

    def trace(self, table, y0, u0, **kw):
        rng = self._call("trace", table, y0, u0, **kw)
        return tuple(rng.uniform(1, 2, (1, 1, 3)) for _ in range(3)) + (rng.uniform(1, 2, (1, 1)),)

    def trace_reduce_many(self, tables, bundles, items, centers=None, **kw):
        m = self._call("trace_reduce_many", tables, bundles, items, centers, **kw).uniform(
            1, 2, (len(items), 20))
        m[:, 4] = self.rng.integers(0, 2, len(items))         # chief rays lost and kept
        return m

    def trace_otf_many(self, tables, bundles, items, centers, z, freqs, **kw):
        rng = self._call("trace_otf_many", tables, bundles, items, centers, z, freqs, **kw)
        s = (len(items), len(z), 2, len(freqs))
        return rng.uniform(-1, 1, s) + 1j*rng.uniform(-1, 1, s), rng.integers(0, 9, s[:2])

    def trace_opd_many(self, tables, bundles, items, specs, a0=None, centers=None, **kw):
        s = self._call("trace_opd_many", tables, bundles, items, specs, a0, centers, **kw).uniform(
            1, 2, (len(items), 10))
        s[:, 0] = self.rng.integers(0, 2, len(items))
        return s

    def trace_zernike_many(self, tables, bundles, items, specs, rho, order, a0=None,
                           centers=None, **kw):
        rng = self._call("trace_zernike_many", tables, bundles, items, specs, rho, order, a0,
                         centers, **kw)
        J = (order + 1)*(order + 2)//2
        return rng.uniform(1, 2, (len(items), (J + 1)*(J + 2)//2)), rng.uniform(0, 1, len(items))


V = 5
PARAMS = [(1, "curvature"), (2, "distance"), (3, "conic")]
HEIGHTS = (0., .7)


@needs_ref
@pytest.mark.parametrize("compensate", [None, "focus"])
@pytest.mark.parametrize("chunk", [1, 2, V])
@pytest.mark.parametrize("name", list(ANALYSES))
def test_driver_launches(name, chunk, compensate):
    """one variant launch per chunk, on the chunk's perturbed tables moved
    by its focus shifts, with height-major items; the setup launches first,
    then the focus pass, then the chunks; nothing left on the device"""
    s = _cooke()
    deltas = sensitivity_deltas([1e-3, 2e-2, .05])[:V]
    eng = _Recorder()
    out = _run(name, copy.deepcopy(s), eng, params=PARAMS, deltas=deltas, heights=HEIGHTS,
               chunk=chunk, compensate=compensate)
    assert not eng.live
    _, _, per_chunk, setup = ANALYSES[name]
    nominal = _nominal(s, s.wavelengths)[0]
    H, W, S = len(HEIGHTS), len(nominal), nominal.shape[1]
    chunks = -(-V//chunk)
    many = [c for c in eng.calls if c[0].endswith("_many")]
    nfocus = chunks if compensate else 0
    assert [c[2]["clip"] for c in many] == [True]*setup + [False]*nfocus + [True]*(
        chunks*len(per_chunk))
    launches = many[setup + nfocus:]
    assert [c[0] for c in launches] == per_chunk*chunks
    for k in range(chunks):
        v0 = k*chunk
        n = min(chunk, V - v0)
        t = perturbed_tables(nominal, PARAMS, deltas[v0:v0 + n])
        if compensate:
            t["offset"][:, :, -1, 2] = _move_distance(t["offset"][:, :, -1, 2],
                                                      out["focus"][v0:v0 + n, None])
        v, h, w = (a.reshape(-1) for a in np.meshgrid(np.arange(n), np.arange(H), np.arange(W),
                                                      indexing="ij"))
        for _, (tables, bundles, items, *_), _ in launches[k*len(per_chunk):(k + 1)*len(per_chunk)]:
            want = t.reshape(n*W, S) if tables.shape[1] == S else t[:, :, :-1].reshape(n*W, S - 1)
            assert np.asarray(tables).tobytes() == want.tobytes()
            assert np.array_equal(items, np.stack([v*W + w, h*W + w], -1))
        assert [b[0].shape[0] for b in bundles] == [_Recorder.NRAYS]*(H*W)


@needs_ref
@pytest.mark.parametrize("compensate", [None, "focus"])
@pytest.mark.parametrize("name", list(ANALYSES))
def test_driver_frees_when_a_launch_fails(name, compensate):
    """the first chunk's variant launch raises: every stand-in array is freed"""
    _, _, per_chunk, setup = ANALYSES[name]
    eng = _Recorder(fail=setup + len(per_chunk) - 1)
    with pytest.raises(RuntimeError, match="failed"):
        _run(name, _cooke(), eng, params=PARAMS, deltas=sensitivity_deltas([1e-3, 2e-2, .05])[:V],
             heights=HEIGHTS, chunk=2, compensate=compensate)
    assert eng.calls[-1][0] == per_chunk[-1]
    assert not eng.live
