"""Through-focus spot images on the device (rtx_trace_spot, rtx_spot_rows,
rayopt_b200.spots) against the numpy statement of their contract
(oracle/spot_oracle.py).  Needs a GPU.

Counts, tallies and extents are integers or maxima of exact values, so every
comparison is exact: the fused epilogue sees the state rtx_trace stores
(tests/test_gpu_epilogues.py), bins it with separately rounded FP64
operations, and adds with integer atomics."""
import warnings

import numpy as np
import pytest

import ref_shim
import spot_oracle
from rayopt_b200._lib import RtxError
from rayopt_b200.engine import spot_spec, spot_shape
from rayopt_b200.spot import default_range
from test_gpu_epilogues import MODES, SYSTEMS, _system

pytestmark = pytest.mark.gpu

NS = [0, 1, 31, 32, 33, 511, 512, 513, 70001, 1000003]


@pytest.fixture(scope="module")
def eng():
    from rayopt_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def _counts(eng, spec):
    c = eng.empty(spot_shape(spec), np.uint64)
    eng.memset(c, 0)
    return c


def _oracle(y, inc, spec):
    s = spec[0]
    K, radial = int(s["planes"]), bool(s["radial"])
    rng = tuple(map(tuple, s["range"][:1 if radial else 2]))
    bins = (int(s["nx"]),) if radial else (int(s["nx"]), int(s["ny"]))
    return spot_oracle.spot(y, inc, s["c"], s["z"][:K], bins, rng, radial, s["o"][:K])


def _assert_same(got_counts, got_tally, got_ext, want, what):
    wc, wt, we = want
    assert np.array_equal(got_counts, wc), (what, np.argwhere(got_counts != wc)[:5])
    assert np.array_equal(got_tally, wt), (what, got_tally, wt)
    assert np.array_equal(got_ext, we), (what, got_ext, we)


def _edge_rows(spec, n_random, dtype, seed):
    """rows whose points at z = 0 land on every edge and 1 ulp either side
    (c = 0 and o = 0 leave y_xy unchanged there), plus NaN, inf and i_z = 0
    rows and random rays"""
    s = spec[0]
    rng = np.random.default_rng(seed)
    axes = []
    for a in range(1 if s["radial"] else 2):
        lo, hi = s["range"][a]
        e = np.linspace(lo, hi, int(s["nx"] if a == 0 else s["ny"]) + 1)
        axes.append(np.concatenate([e, np.nextafter(e, -np.inf), np.nextafter(e, np.inf)]))
    if s["radial"]:
        xs, ys = axes[0], np.zeros_like(axes[0])
    else:
        xs = np.concatenate([axes[0], rng.choice(axes[0], len(axes[1]))])
        ys = np.concatenate([rng.choice(axes[1], len(axes[0])), axes[1]])
    lo, hi = s["range"][0]
    span = hi - lo
    y = np.c_[np.r_[xs, rng.uniform(lo - span*.1, hi + span*.1, n_random)],
              np.r_[ys, rng.uniform(lo - span*.1, hi + span*.1, n_random)],
              np.zeros(len(xs) + n_random)]
    u = rng.normal(0, .05, (len(y), 2))
    inc = np.c_[u, np.sqrt(1 - np.square(u).sum(1))]
    bad = np.array([[np.nan, 0, 0], [np.inf, 0, 0], [0, -np.inf, 0], [0, 0, 0], [.1, .1, 0]])
    y = np.r_[y, bad[:3], [[0, 0, 0], [0, 0, 0]]]
    inc = np.r_[inc, [[0, 0, 1]]*3, bad[3:]]                   # i_z = 0: 0/0 and 0.1/0
    return y.astype(dtype), inc.astype(dtype)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("radial", [False, True])
@pytest.mark.parametrize("K", [1, 5, 16])
def test_rows_equal_oracle_exactly(eng, dtype, radial, K):
    """rtx_spot_rows on synthetic rows against the oracle, several bin
    shapes; a second call without zeroing doubles the counts"""
    for bins, rng_ in (((7, 7), ((-.3, .7), (-.3, .7))), ((13, 5), ((-1e-3, 2e-3), (-.5, .5))),
                       ((1, 256), ((0., 1.), (-4., 4.))), ((256, 3), ((.1, .3), (-.2, .2)))):
        if radial:
            bins, rng_ = bins[:1], ((0., rng_[0][1]),)
        z = np.zeros(K) if K == 1 else np.r_[0., np.linspace(-.02, .02, K - 1)]
        offsets = np.zeros((K, 2))
        offsets[1:] = np.random.default_rng(K).normal(0, .01, (K - 1, 2))
        spec = spot_spec(z, bins, rng_, (0., 0.), radial, offsets)
        y, inc = _edge_rows(spec, 5000, dtype, K)
        dy, di = eng.to_device(y, dtype), eng.to_device(inc, dtype)
        counts = _counts(eng, spec)
        tally, ext = eng.spot_rows(dy, di, spec, counts, extent=True)
        want = _oracle(y, inc, spec)
        what = (dtype.__name__, radial, K, bins)
        _assert_same(counts.download(), tally, ext, want, what)
        assert want[0][0].sum() > len(y)//4, what       # the edge points are in range
        tally2, _ = eng.spot_rows(dy, di, spec, counts)
        assert np.array_equal(counts.download(), 2*want[0]) and np.array_equal(tally2, tally)
        for a in (dy, di, counts):
            a.free()


def _rows(eng, table, dy0, du0, N, dtype, exact, clip, rot0):
    """rtx_trace keep-last: device rows y, i of the last surface"""
    ld = (max(N, 1) + 63)//64*64
    Y, I = eng.empty((1, ld, 3), dtype), eng.empty((1, ld, 3), dtype)
    eng.trace_device(table, dy0, du0, Y, None, I, None, N=N, ld=ld, clip=clip, keep_last=True,
                     rot0=rot0, exact=exact)
    eng.sync()
    return Y, I


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("name", SYSTEMS)
def test_fused_equals_rows_and_oracle(eng, systems, name, mode):
    """rtx_trace_spot = rtx_spot_rows on the rows rtx_trace stores for the
    same launch rays = the oracle on the downloaded rows, 2-D and radial,
    over N = 0 .. 1e6"""
    dtype, exact = MODES[mode]
    table, rot0, clip, rays = _system(name, systems)
    for k, N in enumerate(NS):
        y0, u0 = rays(max(N, 1), 300 + k)
        dy0, du0 = eng.to_device(y0, dtype), eng.to_device(u0, dtype)
        Y, I = _rows(eng, table, dy0, du0, N, dtype, exact, clip, rot0)
        y, inc = Y.download()[0, :N], I.download()[0, :N]
        c = np.nan_to_num(y[0, :2].astype(np.float64)) if N else np.zeros(2)
        radial = k % 2 == 1
        z = np.linspace(-.05, .05, 5)
        probe = spot_spec(z, (64,) if radial else (64, 48), ((-1., 1.),)*(1 if radial else 2), c,
                          radial)
        _, ext = eng.trace_spot(table, dy0, du0, probe, None, N=N, clip=clip, rot0=rot0,
                                exact=exact, extent=True)
        spec = spot_spec(z, (64,) if radial else (64, 48), default_range(ext, (64, 48), radial),
                         c, radial)
        cf, cr = _counts(eng, spec), _counts(eng, spec)
        tf, ef = eng.trace_spot(table, dy0, du0, spec, cf, N=N, clip=clip, rot0=rot0, exact=exact,
                                extent=True)
        tr, er = eng.spot_rows(Y.rows(0), I.rows(0), spec, cr, N=N, extent=True)
        what = (name, mode, N, radial)
        want = _oracle(y, inc, spec)
        _assert_same(cf.download(), tf, ef, want, what + ("fused",))
        _assert_same(cr.download(), tr, er, want, what + ("rows",))
        assert np.array_equal(ext, ef), what
        if N:
            assert (tf.sum(1) == N).all(), what          # the default range holds every finite point
        else:
            assert not tf.any() and not cf.download().any()
        for a in (dy0, du0, Y, I, cf, cr):
            a.free()


def test_deterministic_across_calls_contexts_and_chunks(eng, systems):
    """identical counts twice, in a second context, and when the bundle is
    split into uneven chunks (one of a single ray) that add into one buffer"""
    from rayopt_b200.engine import Engine
    table, rot0, clip, rays = _system("double_gauss", systems)
    N = 1000003
    y0, u0 = rays(N, 77)
    dy0, du0 = eng.to_device(y0), eng.to_device(u0)
    z = np.linspace(-.05, .05, 5)
    _, ext = eng.trace_spot(table, dy0, du0, spot_spec(z, (1, 1), ((-1., 1.),)*2, (0., 0.)),
                            None, clip=clip, extent=True)
    spec = spot_spec(z, (128, 128), default_range(ext, (128, 128)), (0., 0.))

    def run(e, a, b, cuts):
        c = _counts(e, spec)
        tally = np.zeros((5, 2), np.uint64)
        for f, t in zip(cuts[:-1], cuts[1:]):
            tally += e.trace_spot(table, a.rows(f, t), b.rows(f, t), spec, c, N=t - f,
                                  clip=clip)[0]
        out = c.download()
        c.free()
        return out, tally
    one = run(eng, dy0, du0, [0, N])
    assert one[0].sum() == one[1][:, 0].sum() and (one[1].sum(1) == N).all()
    for cuts in ([0, N], [0, 1, 2, 70001, 500000, 999999, N], [0, 333333, 333334, N]):
        got = run(eng, dy0, du0, cuts)
        assert np.array_equal(got[0], one[0]) and np.array_equal(got[1], one[1]), cuts
    e2 = Engine(0)
    try:
        a, b = e2.to_device(y0), e2.to_device(u0)
        got = run(e2, a, b, [0, N])
        a.free(), b.free()
    finally:
        e2.close()
    assert np.array_equal(got[0], one[0]) and np.array_equal(got[1], one[1])
    dy0.free(), du0.free()


def _ref_system(R, name):
    import yaml
    import systems_yaml
    s = R.System(**yaml.safe_load(systems_yaml.SYSTEMS[name]))
    s.update()
    s.paraxial.refocus()
    return s


@pytest.mark.skipif(not ref_shim.available(), reason="reference tree not present")
@pytest.mark.parametrize("nrays", [150, 100000])
@pytest.mark.parametrize("name", ["cooke", "double_gauss"])
def test_spots_end_to_end_against_reference(eng, name, nrays):
    """rayopt_b200.spots against the oracle histogram of the reference's own
    GeometricTrace points (Analysis.spots' rays_point with clip=True) with
    the returned range: bit for bit in exact mode; in fast mode only points
    within 1e-9 h of an edge may change bins"""
    from rayopt_b200 import spots
    R = ref_shim.load()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        s = _ref_system(R, name)
        heights = (0., .707, 1.)
        out = {ex: spots(s, heights, nrays=nrays, bins=(96, 80), engine=eng, exact=ex)
               for ex in (True, False)}
        z = out[True]["z"]
        assert np.array_equal(z, (np.arange(5) - 2)*s.paraxial.rayleigh_range[1])
        for a, hi in enumerate(heights):
            for b, wi in enumerate(s.wavelengths):
                t = R.GeometricTrace(s)
                t.rays_point((0, hi), wi, nrays=nrays, distribution="hexapolar", clip=True)
                for ex, o in out.items():
                    h = o["range"][0][1]
                    assert o["counts"].shape == (3, len(s.wavelengths), 5, 96, 80)
                    want, wt, _ = spot_oracle.spot(t.y[-1], t.i[-1], t.y[-1, t.ref, :2], z,
                                                   (96, 80), o["range"])
                    got = o["counts"][a, b]
                    if ex:
                        assert np.array_equal(got, want), (name, hi, wi)
                        assert np.array_equal(o["tally"][a, b], wt)
                        continue
                    q = spot_oracle.points(t.y[-1], t.i[-1], t.y[-1, t.ref, :2], z)
                    near = 0
                    for ax, n in ((0, 96), (1, 80)):
                        e = np.linspace(*o["range"][ax], n + 1)
                        with np.errstate(invalid="ignore"):
                            d = np.abs(q[..., ax, None] - e).min(-1)
                        near += np.count_nonzero(d <= 1e-9*h)
                    moved = np.abs(got.astype(np.int64) - want.astype(np.int64)).sum()
                    assert moved <= 2*near, (name, hi, wi, moved, near)
        assert np.array_equal(out[True]["airy"],
                              s.paraxial.airy_radius[1]/s.paraxial.wavelength
                              * np.asarray(s.wavelengths))


@pytest.mark.skipif(not ref_shim.available(), reason="reference tree not present")
def test_spots_large_chunked(eng):
    """1e8 rays in chunks of 2^24 equal one unchunked launch per bundle;
    with the default range every ray is binned or non-finite"""
    from rayopt_b200 import spots
    R = ref_shim.load()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        s = _ref_system(R, "double_gauss")
        kw = dict(heights=(.7,), wavelengths=s.wavelengths[:1], nrays=10**8, bins=(512, 512),
                  engine=eng)
        a = spots(s, chunk=2**24, **kw)
        b = spots(s, chunk=2**27, **kw)
    n = int(a["tally"][0, 0, 0].sum())
    assert n > 9*10**7 and (a["tally"][0, 0].sum(1) == n).all()
    assert a["range"] == b["range"]
    assert np.array_equal(a["counts"], b["counts"]) and np.array_equal(a["tally"], b["tally"])


def test_write_contract_and_refusals(eng, systems):
    """nothing outside the (K, nx, ny) block is written; the launch rays and
    stored rows are unchanged; the Engine methods raise RtxError for every
    refusal of include/rtx.h"""
    table, rot0, clip, rays = _system("cooke_asph", systems)
    N = 70001
    y0, u0 = rays(N, 5)
    dy0, du0 = eng.to_device(y0), eng.to_device(u0)
    Y, I = _rows(eng, table, dy0, du0, N, np.float64, False, clip, rot0)
    before = [a.download() for a in (dy0, du0, Y, I)]
    spec = spot_spec(np.linspace(-.1, .1, 3), (40, 24), ((-.2, .2), (-.1, .1)), (0., 0.))
    M, pad = int(np.prod(spot_shape(spec))), 4099
    buf = eng.empty((M + 2*pad,), np.uint64)
    eng.memset(buf, 0xA5)
    inner = buf.rows(pad, pad + M)
    eng.memset(inner, 0)
    eng.trace_spot(table, dy0, du0, spec, inner, N=N, clip=clip)
    eng.spot_rows(Y.rows(0), I.rows(0), spec, inner, N=N)
    got = buf.download()
    guard = np.frombuffer(b"\xa5"*8, np.uint64)[0]
    assert (got[:pad] == guard).all() and (got[pad + M:] == guard).all()
    want = _oracle(Y.download()[0, :N], I.download()[0, :N], spec)[0]
    assert np.array_equal(got[pad:pad + M].reshape(want.shape), 2*want)
    for a, b in zip(before, (dy0, du0, Y, I)):
        assert np.array_equal(a, b.download(), equal_nan=True)
    ok = dict(z=(0., .1), bins=(8, 4), range=((-1., 1.), (-1., 1.)), center=(0., 0.))
    bad = [dict(ok, z=()), dict(ok, z=np.zeros(17)), dict(ok, bins=(0, 4)), dict(ok, bins=(8, 0)),
           dict(ok, bins=(8, 2), range=((0., 1.),), radial=True),
           dict(ok, bins=(2**15, 2**15)), dict(ok, range=((np.nan, 1.), (-1., 1.))),
           dict(ok, range=((-1., 1.), (-1., np.inf))), dict(ok, range=((1., 1.), (-1., 1.))),
           dict(ok, range=((0., 1e-310), (-1., 1.))), dict(ok, z=(0., np.nan)),
           dict(ok, offsets=((0., 0.), (np.inf, 0.)))]
    n0 = eng.launch_count()
    for kw in bad:
        kw = dict(kw)
        rec = spot_spec(kw.pop("z"), kw.pop("bins"), kw.pop("range"), kw.pop("center"), **kw)
        with pytest.raises(RtxError):
            eng.trace_spot(table, dy0, du0, rec, None, N=N, clip=clip, extent=True)
        with pytest.raises(RtxError):
            eng.spot_rows(Y.rows(0), I.rows(0), rec, None, N=N, extent=True)
    rec = spot_spec(**ok)
    with pytest.raises(RtxError):                        # neither counts nor extent
        eng.trace_spot(table, dy0, du0, rec, None, N=N, clip=clip)
    with pytest.raises(RtxError):
        eng.spot_rows(Y.rows(0), I.rows(0), rec, None, N=N)
    assert eng.launch_count() == n0
    tally, ext = eng.spot_rows(Y.rows(0), I.rows(0), rec, None, N=0, extent=True)
    assert not tally.any() and not ext.any() and eng.launch_count() == n0
    for a in (dy0, du0, Y, I, buf):
        a.free()


def test_resident_spot_image_fused_equals_rows(eng, systems):
    """ResidentTrace.spot_image (stored rows) and spot_image_fused (re-march)
    give the same counts, range and tallies, and equal the oracle"""
    from rayopt_b200.lazy import ResidentTrace
    R = ref_shim.load() if ref_shim.available() else None
    if R is None:
        pytest.skip("reference tree not present")
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        s = _ref_system(R, "cooke")
        t = ResidentTrace(s, engine=eng)
        t.rays_point((0, .7), nrays=20000, distribution="hexapolar", clip=True)
        z = np.linspace(-.05, .05, 3)
        for radial in (False, True):
            a = t.spot_image(z, bins=(50, 40), radial=radial)
            b = t.spot_image_fused(z, bins=(50, 40), radial=radial, clip=True)
            assert a["range"] == b["range"]
            assert np.array_equal(a["counts"], b["counts"]) and np.array_equal(a["tally"], b["tally"])
            y, inc = np.asarray(t.y[-1]), np.asarray(t.i[-1])
            want = spot_oracle.spot(y, inc, y[t.ref, :2], z, (50,) if radial else (50, 40),
                                    a["range"], radial)
            assert np.array_equal(a["counts"], want[0]) and np.array_equal(a["tally"], want[1])
            assert (a["tally"].sum(1) == t.nrays).all()
        t.free()
