"""Geometric OTF sums on the device (rtx_otf_rows, Engine.otf_rows,
rayopt_b200.geometric_mtf, ResidentMixin.geometric_mtf) against the
long-double oracle (oracle/otf_oracle.py), within the error bound of
include/rtx.h -- a bound that is itself asserted to be <= 1e-11 in OTF units
in every oracle comparison, so that a loose bound cannot pass.  Needs a GPU."""
import ctypes as C
import warnings

import numpy as np
import pytest

import otf_oracle
import ref_shim
from rayopt_b200._lib import RtxError, check
from rayopt_b200.engine import OTF_DTYPE, OTF_SLOT, otf_bound, otf_spec, spot_spec
from test_gpu_epilogues import MODES, SYSTEMS, _system
from test_gpu_spot import _ref_system, _rows

pytestmark = pytest.mark.gpu

EPS = 2.**-52


@pytest.fixture(scope="module")
def eng():
    from rayopt_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def _assert_oracle(eng, dy, di, N, spec, y, inc, what):
    """otf_rows on the device rows against the oracle of the host rows;
    returns (S, count)"""
    s = spec[0]
    K, F = int(s["planes"]), int(s["nfreq"])
    S, count = eng.otf_rows(dy, di, spec, N=N)
    re, im, n, phi = otf_oracle.otf(y[:N], inc[:N], s["c"], s["z"][:K], s["dnu"], F, s["o"][:K])
    assert S.shape == (K, 2, F) and count.shape == (K,), what
    assert np.array_equal(count, n), (what, count, n)
    bound = otf_bound(spec, N, n, phi)
    assert (bound <= 1e-11*np.maximum(n, 1)).all(), (what, bound/np.maximum(n, 1))
    tol = (bound + otf_oracle.oracle_error(n, phi))[:, None, None]
    err = np.maximum(np.abs(S.real - re.astype(np.float64)), np.abs(S.imag - im.astype(np.float64)))
    assert (err <= tol).all(), (what, (err/tol).max())
    assert np.array_equal(S[..., 0].real, n[:, None].repeat(2, 1).astype(np.float64)), what
    return S, count


def _synthetic(N, dtype, seed):
    """random rows with NaN, +-inf and i_z = 0 rows among them"""
    rng = np.random.default_rng(seed)
    y = np.c_[rng.normal(0, .05, (N, 2)), np.zeros(N)]
    u = rng.normal(0, .05, (N, 2))
    inc = np.c_[u, np.sqrt(1 - np.square(u).sum(1))]
    if N >= 40:
        at = rng.choice(N, 10, replace=False)
        y[at[0], 0], y[at[1], 1], y[at[2], 0] = np.nan, np.inf, -np.inf
        inc[at[3], 2], inc[at[4]] = 0., (0., 0., 0.)
        inc[at[5], 0] = np.nan
    return y.astype(dtype), inc.astype(dtype)


def _spec(K, F, phi_target, q_scale, seed):
    rng = np.random.default_rng(seed)
    z = np.zeros(K) if K == 1 else np.r_[0., np.linspace(-.5, .5, K - 1)]
    o = np.zeros((K, 2))
    o[1:] = rng.normal(0, .01, (K - 1, 2))
    return otf_spec(z, phi_target/q_scale/max(F - 1, 1), F, rng.normal(0, .01, 2), o)


# (N, K, F): every K x F at small N, the N sweep at small K*F (the oracle's cost)
CASES = ([(33, K, F) for K in (1, 5, 16) for F in (1, 64, 256)]
         + [(N, 1, 64) for N in (0, 1, 31, 32, 33, OTF_SLOT - 1, OTF_SLOT, OTF_SLOT + 1,
                                 100003)]
         + [(OTF_SLOT + 1, 5, 64), (3000, 16, 256)])


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_synthetic_rows_against_oracle(eng, dtype):
    for i, (N, K, F) in enumerate(CASES):
        y, inc = _synthetic(max(N, 1), dtype, i)
        dy, di = eng.to_device(y, dtype), eng.to_device(inc, dtype)
        spec = _spec(K, F, 300., .3, i)
        _assert_oracle(eng, dy, di, N, spec, y, inc, (dtype.__name__, N, K, F))
        dy.free(), di.free()


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("name", SYSTEMS)
def test_traced_rows_against_oracle_and_spot_tally(eng, systems, name, mode):
    """the rows rtx_trace stores for each system: the oracle within the
    bound, and count = N minus rtx_spot_rows' non-finite tally"""
    dtype, exact = MODES[mode]
    table, rot0, clip, rays = _system(name, systems)
    N = 20011
    y0, u0 = rays(N, 11)
    dy0, du0 = eng.to_device(y0, dtype), eng.to_device(u0, dtype)
    Y, I = _rows(eng, table, dy0, du0, N, dtype, exact, clip, rot0)
    y, inc = Y.download()[0, :N], I.download()[0, :N]
    c = np.nan_to_num(y[0, :2].astype(np.float64))
    z = np.linspace(-.05, .05, 5)
    import spot_oracle
    q = spot_oracle.points(y, inc, c, z)
    fin = np.isfinite(q).all(2)
    h = max(float(np.abs(q[fin]).max()) if fin.any() else 1., 1e-300)
    spec = otf_spec(z, 200./h/63, 64, c)
    _, count = _assert_oracle(eng, Y.rows(0), I.rows(0), N, spec, y, inc, (name, mode))
    tally, _ = eng.spot_rows(Y.rows(0), I.rows(0), spot_spec(z, (1, 1), ((-1., 1.),)*2, c),
                             None, N=N, extent=True)
    assert np.array_equal(count, N - tally[:, 1].astype(np.int64)), (name, mode)
    for a in (dy0, du0, Y, I):
        a.free()


def test_identical_bits_across_calls_and_contexts(eng):
    from rayopt_b200.engine import Engine
    N = 3*OTF_SLOT + 77
    y, inc = _synthetic(N, np.float64, 9)
    spec = _spec(5, 256, 500., .3, 9)
    dy, di = eng.to_device(y), eng.to_device(inc)
    a = eng.otf_rows(dy, di, spec)
    b = eng.otf_rows(dy, di, spec)
    e2 = Engine(0)
    try:
        d2y, d2i = e2.to_device(y), e2.to_device(inc)
        c = e2.otf_rows(d2y, d2i, spec)
        d2y.free(), d2i.free()
    finally:
        e2.close()
    for other in (b, c):
        assert a[0].tobytes() == other[0].tobytes() and np.array_equal(a[1], other[1])
    dy.free(), di.free()


def test_write_contract_and_refusals(eng):
    """exactly K*2*F*2 doubles and K counts are written (guards around both
    host buffers stay); every refusal of include/rtx.h launches and allocates
    nothing; the record layout matches"""
    from rayopt_b200 import _lib
    from rayopt_b200.engine import Engine
    assert eng.lib.rtx_sizeof_otf() == OTF_DTYPE.itemsize
    N = 5000
    y, inc = _synthetic(N, np.float64, 3)
    dy, di = eng.to_device(y), eng.to_device(inc)
    spec = _spec(3, 40, 100., .3, 3)
    M, pad = 3*2*40*2, 17
    sums = np.full(M + 2*pad, -7.25)
    cnt = np.full(3 + 2*pad, -5, np.int64)
    p = lambda a, off: C.c_void_p(a.ctypes.data + off*a.itemsize)  # noqa: E731
    check(eng.lib.rtx_otf_rows(eng.ctx, 0, N, dy.ptr, di.ptr, _lib.ptr(spec), p(sums, pad),
                               p(cnt, pad)))
    assert (sums[:pad] == -7.25).all() and (sums[pad + M:] == -7.25).all()
    assert (cnt[:pad] == -5).all() and (cnt[pad + 3:] == -5).all()
    S, count = eng.otf_rows(dy, di, spec)
    got = sums[pad:pad + M].reshape(3, 2, 40, 2)
    assert np.array_equal(got[..., 0] + 1j*got[..., 1], S)
    assert np.array_equal(cnt[pad:pad + 3], count)
    check(eng.lib.rtx_otf_rows(eng.ctx, 0, 0, None, None, _lib.ptr(spec), p(sums, pad),
                               p(cnt, pad)))                       # N = 0: zeros, NULL rows
    assert not sums[pad:pad + M].any() and not cnt[pad:pad + 3].any()
    assert (sums[pad + M:] == -7.25).all() and (cnt[pad + 3:] == -5).all()

    def rec(**kw):
        r = spec.copy()
        for k, v in kw.items():
            if k in ("z", "o"):
                r[k][0, 1] = v
            else:
                r[k][0] = v
        return r
    bad_specs = [rec(planes=0), rec(planes=17), rec(nfreq=0), rec(nfreq=257), rec(dnu=np.nan),
                 rec(dnu=np.inf), rec(c=(np.nan, 0.)), rec(z=np.inf), rec(o=(0., np.nan))]
    e2 = Engine(0)                          # a fresh context keeps no OTF workspace yet
    try:
        a, b = e2.to_device(y), e2.to_device(inc)
        free0, n0 = e2.free_bytes(), e2.launch_count()
        big = 10**9                         # would need gigabytes of slot sums
        s = np.zeros(16*2*256*2)
        k = np.zeros(16, np.int64)
        calls = [(e2.ctx, 0, big, a.ptr, b.ptr, _lib.ptr(r), _lib.ptr(s), _lib.ptr(k))
                 for r in bad_specs]
        good = _lib.ptr(spec)
        calls += [(None, 0, N, a.ptr, b.ptr, good, _lib.ptr(s), _lib.ptr(k)),
                  (e2.ctx, 0, N, a.ptr, b.ptr, None, _lib.ptr(s), _lib.ptr(k)),
                  (e2.ctx, 0, N, a.ptr, b.ptr, good, None, _lib.ptr(k)),
                  (e2.ctx, 0, N, a.ptr, b.ptr, good, _lib.ptr(s), None),
                  (e2.ctx, 0, N, None, b.ptr, good, _lib.ptr(s), _lib.ptr(k)),
                  (e2.ctx, 0, N, a.ptr, None, good, _lib.ptr(s), _lib.ptr(k)),
                  (e2.ctx, 0, -1, a.ptr, b.ptr, good, _lib.ptr(s), _lib.ptr(k)),
                  (e2.ctx, 2, big, a.ptr, b.ptr, good, _lib.ptr(s), _lib.ptr(k))]
        for args in calls:
            assert eng.lib.rtx_otf_rows(*args) == -1, args
        assert not s.any() and not k.any()
        assert e2.launch_count() == n0
        assert free0 - e2.free_bytes() < 2**30          # no slot sums were allocated
        for r in bad_specs[:2]:
            with pytest.raises(RtxError):
                e2.otf_rows(a, b, r, N=N)
        a.free(), b.free()
    finally:
        e2.close()
    dy.free(), di.free()


@pytest.mark.skipif(not ref_shim.available(), reason="reference tree not present")
def test_geometric_mtf_large_chunked(eng):
    """1e8 rays: several chunk sizes against one unchunked call.  Every ray's
    terms are the same bits in each (the rays, the trace and the phasors do
    not depend on the chunking), so only the summation order differs: the
    difference is within the sum of the two summation-depth terms."""
    from rayopt_b200 import geometric_mtf
    R = ref_shim.load()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        s = _ref_system(R, "double_gauss")
        kw = dict(heights=(.7,), wavelengths=s.wavelengths[:1], nrays=10**8, nfreq=64,
                  defocus=(np.arange(3) - 1)*s.paraxial.rayleigh_range[1], engine=eng)
        one = geometric_mtf(s, chunk=2**27, **kw)
        n = one["count"][0, 0]
        assert (n > 9*10**7).all()
        S1 = one["otf"][0, 0]*n[:, None, None]
        N = 11*10**7                        # at least the bundle's rays

        def depth(chunk):                   # one call's depth + the host's chunk adds
            return OTF_SLOT//8 + 8 + -(-min(chunk, N)//OTF_SLOT) + -(-N//chunk)
        for chunk in (2**24, 3*10**7 + 1, 10**7 - 3):
            got = geometric_mtf(s, chunk=chunk, **kw)
            assert np.array_equal(got["count"], one["count"]), chunk
            # + 4: the division by n and the multiplication back, in each
            tol = (depth(chunk) + depth(2**27) + 4)*EPS*n[:, None, None]
            S = got["otf"][0, 0]*n[:, None, None]
            err = np.maximum(np.abs(S.real - S1.real), np.abs(S.imag - S1.imag))
            assert (err <= tol).all(), (chunk, (err/tol).max())
        assert np.array_equal(one["freq"], np.arange(64)*one["freq"][1])
        assert np.isclose(one["freq"][-1], 1/s.paraxial.airy_radius[1], rtol=1e-15, atol=0)


@pytest.mark.skipif(not ref_shim.available(), reason="reference tree not present")
@pytest.mark.parametrize("name", ["cooke", "double_gauss"])
def test_geometric_mtf_end_to_end_against_reference(eng, name):
    """geometric_mtf(exact=True) against the oracle OTF of the reference's own
    GeometricTrace.rays_point(..., clip=True) rows about the chief ray of the
    first wavelength; poly against the documented weighted mean"""
    from rayopt_b200 import geometric_mtf
    R = ref_shim.load()
    nrays, heights, F = 20000, (0., .707, 1.), 32
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        s = _ref_system(R, name)
        z = (np.arange(3) - 1)*s.paraxial.rayleigh_range[1]
        wts = np.arange(1., len(s.wavelengths) + 1)
        out = geometric_mtf(s, heights, nrays=nrays, defocus=z, nfreq=F, spectral_weights=wts,
                            engine=eng, exact=True)
        dnu = out["freq"][1]
        H, W = len(heights), len(s.wavelengths)
        assert out["otf"].shape == (H, W, 3, 2, F) and out["poly"].shape == (H, 3, 2, F)
        want = np.zeros((H, W, 3, 2, F), np.complex128)
        for a, hi in enumerate(heights):
            c = None
            for b, wi in enumerate(s.wavelengths):
                t = R.GeometricTrace(s)
                t.rays_point((0, hi), wi, nrays=nrays, distribution="hexapolar", clip=True)
                if c is None:
                    c = t.y[-1, t.ref, :2]
                re, im, n, phi = otf_oracle.otf(t.y[-1], t.i[-1], c, z, dnu, F)
                assert np.array_equal(out["count"][a, b], n), (name, hi, wi)
                N = len(t.y[-1])
                bound = otf_bound(otf_spec(z, dnu, F, c), N, n, phi)
                assert (bound <= 1e-11*n).all(), (name, hi, wi, bound/n)
                tol = ((bound + otf_oracle.oracle_error(n, phi))/n)[:, None, None]
                w = (re.astype(np.float64) + 1j*im.astype(np.float64))/n[:, None, None]
                got = out["otf"][a, b]
                err = np.maximum(np.abs(got.real - w.real), np.abs(got.imag - w.imag))
                assert (err <= tol + 2*EPS).all(), (name, hi, wi, (err/tol).max())
                want[a, b] = w
        assert np.allclose(np.abs(out["otf"]), out["mtf"], rtol=0, atol=0)
        poly = np.einsum("w,hwkaf->hkaf", wts, want)/wts.sum()
        assert np.abs(out["poly"] - poly).max() <= 1e-11


@pytest.mark.skipif(not ref_shim.available(), reason="reference tree not present")
def test_resident_geometric_mtf_equals_otf_rows(eng):
    """ResidentTrace.geometric_mtf = otf_rows on the trace's downloaded and
    re-uploaded rows, bit for bit"""
    from rayopt_b200.lazy import ResidentTrace
    R = ref_shim.load()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        s = _ref_system(R, "cooke")
        t = ResidentTrace(s, engine=eng)
        t.rays_point((0, .7), nrays=50000, distribution="hexapolar", clip=True)
        z = np.linspace(-.05, .05, 3)
        got = t.geometric_mtf(z, nfreq=48)
        y, inc = np.asarray(t.y[-1]), np.asarray(t.i[-1])
        dy, di = eng.to_device(y), eng.to_device(inc)
        S, count = eng.otf_rows(dy, di, otf_spec(z, got["freq"][1], 48, y[t.ref, :2]))
        with np.errstate(invalid="ignore"):
            want = S/count[:, None, None]
        assert got["otf"].tobytes() == want.tobytes() and np.array_equal(got["count"], count)
        assert (count > 0).all()
        dy.free(), di.free()
        t.free()
