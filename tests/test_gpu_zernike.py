"""rtx_trace_zernike_many and rayopt_b200.tolerance_zernike / zernike on
the device.  Needs a GPU.

Each item's rays are traced with rtx_trace_opd through the item's table with
the item's sphere; the oracle (tests/zernike_oracle.py) forms their (a, x,
y) and the exact Zernike Gram sums in long double: counts and r2max
exactly, every sum within include/rtx.h's bound (a) + (b).  Then bit-for-bit
determinism, agreement with tolerance_wavefront's rms and rms_tilt, the
reference's own opd() of perturbed lenses, the symmetries of a centred
lens, focus compensation, a 4096-variant run in chunks, and the C
refusals."""
import copy
import ctypes as C
import warnings

import numpy as np
import pytest

import ref_shim
from test_gpu_tolerance import case, variants
from test_gpu_tolerance_wavefront import (device_bundles, free, item_specs, opd_rows, spec_for,
                                          tol_case)
from zernike_oracle import oracle

pytestmark = pytest.mark.gpu

MODES = {"f64_exact": True, "f64_fast": False}
NZ = [0, 1, 511, 513, 4099]          # N = 0, and N not a multiple of 512


@pytest.fixture(scope="module")
def eng():
    from rayopt_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def zrn_items(eng, name, systems, seed):
    table, rot0, _, rays = case(name, systems)
    march = table[:-1]
    tabs = variants(march, 6, seed)
    bundles, host = device_bundles(eng, rays, NZ)
    rng = np.random.default_rng(seed)
    items = np.c_[rng.integers(0, 6, 12), rng.integers(0, len(NZ), 12)]
    items[:len(NZ), 1] = np.arange(len(NZ))
    specs, a0, cen = item_specs(march, host, items, seed + 1)
    return tabs, rot0, bundles, host, items, specs, a0, cen


@pytest.mark.parametrize("clip", [True, False], ids=["clip", "noclip"])
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("order", [0, 1, 4, 8])
def test_sums_match_oracle(eng, systems, order, mode, clip):
    exact = MODES[mode]
    tabs, rot0, bundles, host, items, specs, a0, cen = zrn_items(eng, "double_gauss", systems, 3)
    try:
        # rho about each item's own pupil radius, from its r2max (order 0)
        _, r2 = eng.trace_zernike_many(tabs, bundles, items, specs, np.ones(len(items)), 0, a0,
                                       cen, clip=clip, rot0=rot0, exact=exact)
        rng = np.random.default_rng(order)
        rho = np.where(r2 > 0, np.sqrt(r2), 1.)*rng.uniform(.7, 1.3, len(items))
        s, r2b = eng.trace_zernike_many(tabs, bundles, items, specs, rho, order, a0, cen,
                                        clip=clip, rot0=rot0, exact=exact)
        J = (order + 1)*(order + 2)//2
        assert s.shape == (len(items), (J + 1)*(J + 2)//2)
        assert r2b.tobytes() == r2.tobytes()
        for i, (t, b) in enumerate(items):
            N = bundles[b][2]
            if N == 0:
                assert (s[i] == 0).all() and r2[i] == 0
                continue
            A, P = opd_rows(eng, tabs[t], bundles[b][0], bundles[b][1], N, specs[i], exact,
                            clip, rot0)
            want, bound, n, r2max = oracle(A, P, a0[i], cen[i], rho[i], order)
            assert s[i, J + 1] == n, (i, s[i, J + 1], n)
            assert r2[i] == r2max, (i, r2[i], r2max)
            err = np.abs(s[i] - want.astype(float))
            assert np.all(err <= bound), (i, np.max(err/np.maximum(bound, 1e-300)))
    finally:
        free(bundles)


@pytest.mark.parametrize("mode", list(MODES))
def test_deterministic(eng, systems, mode):
    """the same bits in two calls, alone, under a permutation and in halves"""
    exact = MODES[mode]
    tabs, rot0, bundles, host, items, specs, a0, cen = zrn_items(eng, "double_gauss", systems, 8)
    from rayopt_b200.engine import OPD_DTYPE, _opd_record
    recs = np.concatenate([_opd_record(s) for s in specs]).astype(OPD_DTYPE)
    rho = np.random.default_rng(1).uniform(1, 5, len(items))

    def run(sel):
        return eng.trace_zernike_many(tabs, bundles, items[sel], recs[sel], rho[sel], 6, a0[sel],
                                      cen[sel], clip=True, rot0=rot0, exact=exact)
    try:
        every = np.arange(len(items))
        a, ra = run(every)
        b, rb = run(every)
        assert a.tobytes() == b.tobytes() and ra.tobytes() == rb.tobytes()
        assert run(every[3:4])[0].tobytes() == a[3:4].tobytes()
        p = np.random.default_rng(2).permutation(len(items))
        assert run(p)[0].tobytes() == a[p].tobytes()
        h = np.concatenate([run(every[:5])[0], run(every[5:])[0]])
        assert h.tobytes() == a.tobytes()
    finally:
        free(bundles)


def test_refusals_launch_and_allocate_nothing(eng, systems):
    """each refusal returns its code with no launch and no allocation; the
    outputs have host guard bands that stay untouched"""
    from rayopt_b200 import _lib
    from rayopt_b200.engine import OPD_DTYPE, _opd_record
    table, _, clip, rays = case("double_gauss", systems)
    march = np.ascontiguousarray(variants(table[:-1], 2, 1))
    y, u = rays(1000, 1)
    dy, du = eng.to_device(y), eng.to_device(u)
    S = march.shape[1]
    good = _opd_record(spec_for(march[0], y, u, 1)).astype(OPD_DTYPE)
    eng.trace_zernike_many(march, [(dy, du, None)], [[0, 0]], good, [1.], 4)      # warm

    def call(nt=2, tables=march, S=S, dtype=0, N=(1000,), y0=(dy.ptr,), u0=(du.ptr,), it=(0,),
             specs=good, order=4, rho=(1.,), sums=True, r2=True, flags=0):
        Na = np.ascontiguousarray(N, np.int64)
        ya = (C.c_void_p*1)(*y0)
        ua = (C.c_void_p*1)(*u0)
        ita, iba = np.ascontiguousarray(it, np.int32), np.zeros(1, np.int32)
        sa = None if specs is None else np.ascontiguousarray(specs, OPD_DTYPE)
        ra = None if rho is None else np.ascontiguousarray(rho, np.float64)
        out = np.full(1081 + 64, 7.25)
        r2o = np.full(64, 7.25)
        rc = eng.lib.rtx_trace_zernike_many(
            eng.ctx, nt, _lib.ptr(tables), S, None, dtype, 1, _lib.ptr(Na), ya, ua, 1,
            _lib.ptr(ita), _lib.ptr(iba), _lib.ptr(sa), None, None, 1, order, _lib.ptr(ra),
            _lib.ptr(out) if sums else None, _lib.ptr(r2o) if r2 else None, flags)
        return rc, out, r2o

    E_BAD, E_UNS = -1, -2
    y32, u32 = eng.to_device(y.astype(np.float32)), eng.to_device(u.astype(np.float32))
    bad = good.copy()
    bad["radius"] = 0.
    cases = [(dict(sums=False), E_BAD), (dict(r2=False), E_BAD), (dict(rho=None), E_BAD),
             (dict(specs=None), E_BAD), (dict(nt=0), E_BAD), (dict(it=(2,)), E_BAD),
             (dict(N=(-1,)), E_BAD), (dict(specs=bad), E_BAD),
             (dict(order=-1), E_BAD), (dict(order=9), E_BAD),
             (dict(rho=(0.,)), E_BAD), (dict(rho=(-1.,)), E_BAD), (dict(rho=(np.nan,)), E_BAD),
             (dict(rho=(np.inf,)), E_BAD),
             (dict(dtype=1, y0=(y32.ptr,), u0=(u32.ptr,)), E_UNS),
             (dict(dtype=1, y0=(y32.ptr,), u0=(u32.ptr,), flags=1), E_UNS)]
    try:
        for kw, want in cases:
            eng.sync()
            fb, launches = eng.free_bytes(), eng.launch_count()
            rc, out, r2o = call(**kw)
            assert rc == want, (kw, rc)
            assert eng.launch_count() == launches and eng.free_bytes() == fb, kw
            assert (out == 7.25).all() and (r2o == 7.25).all(), kw
        rc, out, r2o = call()                                         # guard bands
        E = 16*17//2
        assert rc == 0 and (out[E:] == 7.25).all() and (r2o[1:] == 7.25).all()
        assert 0 < out[16] <= 1000 and r2o[0] > 0
        rc, out, r2o = call(N=(0,), y0=(None,), u0=(None,))           # N = 0: zeros
        assert rc == 0 and (out[:E] == 0).all() and r2o[0] == 0
        fb = eng.free_bytes()
        rc, _, _ = call(N=(2**52,))                                   # 2^43 tile rows
        assert rc == _lib.RTX_E_NOMEM and eng.free_bytes() == fb
    finally:
        for a in (dy, du, y32, u32):
            a.free()


# ---- rayopt_b200.tolerance_zernike end to end --------------------------------
needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="no reference tree staged")


@pytest.fixture(scope="module")
def R():
    warnings.simplefilter("ignore")
    np.seterr(all="ignore")
    return ref_shim.load()


def build(R, name):
    import yaml
    import systems_yaml
    s = R.System(**yaml.safe_load(systems_yaml.SYSTEMS[name]))
    s.update()
    s.paraxial.refocus()
    return s


def lens_case(R, name):
    from rayopt_b200.surface_table import pack_system
    sys_ = build(R, name)
    S = len(pack_system(sys_, sys_.wavelengths[0], 1, None)[0])
    tol = tol_case(name, S)
    return sys_, [(j, k) for j, k, _ in tol], [abs(t) for _, _, t in tol]


@needs_ref
@pytest.mark.parametrize("name", ["cooke", "double_gauss"])
def test_agrees_with_tolerance_wavefront(eng, R, name):
    """64 Monte Carlo variants: the residual at order 0 is
    tolerance_wavefront's rms and at order 1 its rms_tilt (the same
    least-squares subspaces, 1 and 1, x, y), within 1e-7 relative or 1e-9
    waves; the counts and the chief flags are the same"""
    import rayopt_b200
    sys_, params, tol = lens_case(R, name)
    deltas = rayopt_b200.monte_carlo_deltas(tol, 64, seed=5)
    w = rayopt_b200.tolerance_wavefront(copy.deepcopy(sys_), params, deltas, nrays=500,
                                        engine=eng)
    worst = 0.
    for order, key in ((0, "rms"), (1, "rms_tilt")):
        z = rayopt_b200.tolerance_zernike(copy.deepcopy(sys_), params, deltas, nrays=500,
                                          order=order, engine=eng)
        assert np.array_equal(z["chief"], w["chief"])
        assert np.array_equal(z["sums"][..., (order + 1)*(order + 2)//2 + 1], w["sums"][..., 0])
        for got, want in ((z["residual"], w[key]), (z["rms"], w["rms"])):
            err = np.abs(got - want)
            worst = max(worst, np.nanmax(err/want))
            assert np.all(err <= np.maximum(1e-7*want, 1e-9)), (order, np.nanmax(err))
    print("%s: largest relative difference %.2e" % (name, worst))


@needs_ref
@pytest.mark.parametrize("name", ["cooke", "double_gauss"])
def test_against_reference_opd(eng, R, name):
    """RTX_EXACT, a few perturbed lenses: the reference's own opd() points
    of each perturbed System, fitted in long double with the same rho.  The
    reference forms each ray's t in its own operation order, within
    ~1e-10 waves of the device's (test_gpu_tolerance_wavefront); a per-ray
    difference d moves the fit by at most |G+| sqrt(sum_j mean|Z_j|^2) d"""
    import rayopt_b200
    from rayopt_b200.lazy import opd_spec
    from rayopt_b200.rays import grid_spec
    from rayopt_b200.tolerance import launch_bundles
    from rayopt_b200.zernike import zernike_basis
    from test_tolerance_host import apply
    sys_, params, tol = lens_case(R, name)
    deltas = rayopt_b200.sensitivity_deltas(tol)[:4]
    heights, nrays, order = (0., .7), 300, 4
    out = rayopt_b200.tolerance_zernike(copy.deepcopy(sys_), params, deltas, heights,
                                        nrays=nrays, order=order, engine=eng, exact=True)
    J = out["coefficients"].shape[-1]
    nom = copy.deepcopy(sys_)
    bundles, _ = launch_bundles(nom, heights, nom.wavelengths, nrays, "hexapolar", eng)
    radius = opd_spec(nom, nom.track, nom.origins, len(nom) - 2, len(nom) - 1, 1., 1.,
                      np.zeros(3), np.zeros(3), np.zeros(3))["radius"]
    launch = [(y.download(), u.download()) for y, u in bundles]
    for y, u in bundles:
        y.free(), u.free()
    ref_i = grid_spec("hexapolar", nrays)[0]
    W = len(sys_.wavelengths)
    worst = 0.
    ld = np.longdouble
    for v, row in enumerate(deltas):
        ref = copy.deepcopy(sys_)
        for (j, kind), dv in zip(params, row):
            if dv:
                apply(ref, j, kind, dv)
        for h in range(len(heights)):
            for w, l in enumerate(sys_.wavelengths):
                g = R.GeometricTrace(ref)
                g.rays_given(*launch[h*W + w], l, ref=ref_i)
                g.propagate(clip=True)
                x, y, t = g.opd(radius=radius, resample=0)
                ok = np.isfinite(x) & np.isfinite(y) & np.isfinite(t)
                x, y, t = x[ok], y[ok], t[ok]
                rho = out["radius"][h, w]
                Z = zernike_basis(J, np.asarray(x, ld)/ld(rho), np.asarray(y, ld)/ld(rho))
                G = (Z.T @ Z)/len(t)
                c = np.linalg.solve(G.astype(float), ((Z.T @ np.asarray(t, ld))/len(t)).astype(float))
                got = out["coefficients"][v, h, w]
                Zf = np.abs(Z.astype(float))
                tol_c = (np.linalg.norm(np.linalg.inv(G.astype(float)), 2)
                         * np.sqrt(((Zf.mean(0))**2).sum())*1e-9 + 1e-12)
                err = np.abs(got - c).max()
                worst = max(worst, err)
                assert err <= tol_c, ((v, h, w), err, tol_c)
    print("%s: largest coefficient difference from the reference's opd() %.2e waves"
          % (name, worst))


@needs_ref
def test_symmetry_and_defocus(eng, R):
    """order 4 on the Cooke triplet, hexapolar rays: on axis every m != 0
    coefficient vanishes; at fields along y the lens is symmetric under
    x -> -x, so every term odd in x vanishes (cos m theta with m odd, sin m
    theta with m even: Z2, Z5, Z8, Z10, Z13, Z15); a pure image-distance
    change moves Z4 with the sign of the defocus, and zernike() is the
    undisturbed variant"""
    import rayopt_b200
    from rayopt_b200.surface_table import pack_system
    sys_ = build(R, "cooke")
    S = len(pack_system(sys_, sys_.wavelengths[0], 1, None)[0])
    d = np.array([[0.], [.05], [-.05]])
    out = rayopt_b200.tolerance_zernike(copy.deepcopy(sys_), [(S, "distance")], d,
                                        heights=(0., .7, 1.), nrays=1000, order=4, engine=eng)
    c = out["coefficients"]
    m = out["noll"][:, 1]
    big = np.abs(c).max(-1, keepdims=True)
    assert np.all(np.abs(c[:, 0][..., m != 0]) <= 1e-9*big[:, 0])
    odd_x = ((m > 0) & (m % 2 == 1)) | ((m < 0) & (m % 2 == 0))
    assert list(np.flatnonzero(odd_x) + 1) == [2, 5, 8, 10, 13, 15]
    assert np.all(np.abs(c[:, 1:][..., odd_x]) <= 1e-9*big[:, 1:])
    assert np.abs(c[:, 1:][..., ~odd_x & (m != 0)]).max() > 1e-6     # not all vanish
    z4 = c[..., 3]
    assert np.all((z4[1] - z4[0])*(z4[2] - z4[0]) < 0)                # opposite signs
    s1 = np.sign(z4[1] - z4[0])
    assert np.all(s1 == s1.flat[0])                                   # one sign everywhere
    nom = rayopt_b200.zernike(copy.deepcopy(sys_), heights=(0., .7, 1.), nrays=1000, order=4,
                              engine=eng)
    assert nom["coefficients"].tobytes() == c[0].tobytes()
    assert nom["radius"].tobytes() == out["radius"].tobytes()


@needs_ref
def test_focus_compensation(eng, R):
    """compensate="focus" gives tolerance()'s focus shifts bit for bit"""
    import rayopt_b200
    sys_, params, tol = lens_case(R, "cooke")
    deltas = rayopt_b200.monte_carlo_deltas(tol, 8, seed=2)
    z = rayopt_b200.tolerance_zernike(copy.deepcopy(sys_), params, deltas, nrays=300,
                                      compensate="focus", engine=eng)
    t = rayopt_b200.tolerance(copy.deepcopy(sys_), params, deltas, nrays=300,
                              compensate="focus", engine=eng)
    assert z["focus"].tobytes() == t["focus"].tobytes()
    assert np.isfinite(z["coefficients"]).all()


@needs_ref
def test_scale_and_chunking(eng, R):
    """4096 Monte Carlo variants x 9 bundles of the Cooke triplet at order 6:
    chunks of 1000 variants give the same bits as one launch"""
    import rayopt_b200
    sys_, params, tol = lens_case(R, "cooke")
    deltas = rayopt_b200.monte_carlo_deltas(tol, 4096, seed=9)
    a = rayopt_b200.tolerance_zernike(copy.deepcopy(sys_), params, deltas, nrays=1000,
                                      order=6, engine=eng, chunk=4096)
    b = rayopt_b200.tolerance_zernike(copy.deepcopy(sys_), params, deltas, nrays=1000,
                                      order=6, engine=eng, chunk=1000)
    assert a["sums"].tobytes() == b["sums"].tobytes()
    assert a["coefficients"].tobytes() == b["coefficients"].tobytes()
    assert (a["transmitted"] > 0).all()
