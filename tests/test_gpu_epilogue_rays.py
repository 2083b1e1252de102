"""The fused epilogues ray by ray: rtx_trace_reduce, rtx_trace_reduce_many,
rtx_trace_opd and rtx_trace_spot on seeded random lenses, the decision-boundary
bundles and launch rays with non-finite components.  Needs a GPU.

epi_kernel is a second copy of the march, compiled once per epilogue and mode,
each copy with its own inlining and FMA contraction.  Its promise is that the
epilogue sees, for every ray, the bits rtx_trace stores at the last surface.
Sums hide a ray that is a few ulps off, so each epilogue is observed per ray:

  OPD     A and P of every ray, bit for bit, against epi_oracle.opd_epilogue
          of the ray's row and path sum;
  many    one launch with one item per ray, each item its own one-ray bundle
          and a random centre: the warp, tile and item sums then add only
          zeros, so every column is one IEEE operation on the ray (`ray_moments`)
          and is compared exactly (+0 == -0), the counts pin the finite / good
          gating, and only the contractable m[3], m[18], m[19] are compared
          within 2 eps of their scale (extended precision);
  reduce  rtx_trace_reduce of one ray (atomics into zeros are exact) for a
          subsample: every boundary ray and SUB random rays per lens, half of
          them weighted; the same columns;
  spot    rtx_trace_spot of one ray on the same subsample, 5 offset planes:
          per plane |q_x|, |q_y|, r and the tallies of the ray, the counts of
          the subsample added up; and each whole bundle once, counts, tallies
          and extents against spot_oracle.spot.

Each whole bundle also goes through rtx_trace_reduce, its sums against the
exact sums within (L + 64) eps sum|term| (tests/test_gpu_epilogues.py).

The truth is np_oracle's rows in exact FP64 on unrotated analytic lenses and on
every edge bundle (whose launch rays are finite), and elsewhere the rows of
rtx_trace (keep-last) in the same dtype and mode, which
tests/test_gpu_config_invariance.py pins across kernel configurations.

rtx_trace_reduce_many is also run with 8 independently drawn tables of the
same length (different surface kinds, rotations and coefficient counts): one-ray
items that cycle through the tables, so that every tile restages the table,
ragged items, items without rays, and total tile counts around the grid size
(one and two CTAs per SM), which covers the edges of the contiguous-run split.
"""
import numpy as np
import pytest

import edge_bundles as eb
import epi_oracle
import np_oracle
import spot_oracle
from rayopt_b200.engine import spot_spec, spot_shape
from rayopt_b200.surface_table import SURFACE_DTYPE
from test_gpu_config_invariance import euler, random_rays
from test_gpu_domain_edges import CASES as EDGE
from test_gpu_epilogues import MODES, _L_epi, _spec, _stored, _within

pytestmark = pytest.mark.gpu

EPS = 2.0**-52
NS = [1, 31, 33, 511, 512, 513, 70001]
SUB = 256                       # random rays per lens through the one-ray launches
CONTRACTED = (3, 18, 19)        # sums of products the compiler may fuse
ROT0 = euler(.01, -.02, .015)


# ---- seeded random lenses ---------------------------------------------------
LAST_KINDS = ("sphere", "conic", "plane", "newton", "mirror", "alt", "tilted")


def random_lens(seed, last, analytic=False, inner=(), S=None):
    """a random table in the manner of test_gpu_config_invariance.random_table,
    with controls: `last` the kind of the last surface (LAST_KINDS),
    `analytic` no Newton surface and no tilt (else surface 0 is an asphere of
    5..10 coefficients and surface 2 is tilted), `inner` features forced onto
    distinct inner surfaces ("alt", "mirror", "mu1"); S drawn from 4..8
    unless given"""
    rng = np.random.default_rng(seed)
    S = int(rng.integers(4, 9)) if S is None else S
    force = dict(zip(rng.permutation(np.arange(1, S - 1))[:len(inner)].tolist(), inner))
    force[S - 1] = last
    kinds = ["sphere", "conic", "plane"] + ([] if analytic else ["asph"])
    t = np.zeros(S, SURFACE_DTYPE)
    n0 = 1.0
    for j in range(S):
        f = force.get(j)
        r = t[j]
        r["offset"] = (0, 0, rng.uniform(.5, 6.))
        r["rot"] = np.eye(3).reshape(9)
        flags = 0
        if f == "tilted" or (not analytic and f is None and (j == 2 or rng.random() < .3)):
            r["offset"][:2] = rng.normal(0, .05, 2)
            r["rot"] = euler(*rng.normal(0, .03, 3)).reshape(9)
            flags |= 1
        if f in ("sphere", "conic", "plane"):
            kind = f
        elif f == "newton" or (j == 0 and not analytic):
            kind = "asph"
        elif f == "alt":                          # the flag only matters to the quadric roots
            kind = str(rng.choice(["sphere", "conic"]))
        else:
            kind = str(rng.choice(kinds))
        c = 0. if kind == "plane" else rng.choice([-1, 1])/rng.uniform(8., 200.)
        k = 0.
        if kind == "conic" or (kind == "asph" and rng.random() < .7):
            k = rng.uniform(-1.5, .8)
        r["c"], r["k"] = c, k
        r["kc2"] = (1 + k)*c**2
        radius = rng.uniform(3., 6.)
        r["radius2"] = radius**2 if rng.random() < .8 else np.inf
        u = rng.random()
        if f == "mirror" or (f is None and u < .08):
            n, mu = n0, -1.
        elif f == "mu1" or (f is None and u < .16):
            n, mu = n0, 1.
        else:
            n = rng.choice([1.0, rng.uniform(1.4, 1.9)]) if n0 > 1 else rng.uniform(1.4, 1.9)
            mu = n0/n
        r["mu"], r["muf"], r["sgn"], r["mu2m1"] = mu, abs(mu), np.sign(mu), mu**2 - 1
        r["n0"], r["n"] = n0, n
        n0 = n
        r["n_asph"] = -1
        if kind == "asph":
            na = int(rng.integers(5, 11)) if j == 0 or f == "newton" else int(rng.integers(1, 11))
            a = rng.normal(0, 1, na)*10.0**(-3 - 2*np.arange(na))
            r["n_asph"] = na
            r["asph"][:na] = a
            r["dasph"][:na] = [2*(i + 1)*a[i] for i in range(na)]
        if f == "alt" or (kind != "plane" and rng.random() < .05):
            flags |= 2
        r["flags"] = flags
    return t


# name: (seed, last surface, clip, rot0, analytic, forced inner surfaces)
LENSES = {
    "a_sphere": (101, "sphere", True, False, True, ()),
    "a_conic": (102, "conic", False, False, True, ("alt", "mirror")),
    "a_plane": (122, "plane", True, False, True, ("mu1",)),
    "a_mirror": (104, "mirror", False, False, True, ()),
    "a_alt": (105, "alt", True, False, True, ("mu1",)),
    "newton_rot0": (106, "newton", True, True, False, ()),
    "newton_alt": (107, "newton", False, False, False, ("alt",)),
    "mirror_rot0": (108, "mirror", True, True, False, ()),
    "alt": (109, "alt", False, False, False, ("mirror",)),
    "tilted": (110, "tilted", True, False, False, ()),
    "tilted_rot0_mu1": (111, "tilted", False, True, False, ("mu1",)),
    "sphere_rot0": (112, "sphere", False, True, False, ()),
    "conic_mirror": (113, "conic", True, False, False, ("mirror",)),
    "plane_rot0": (114, "plane", False, True, False, ("alt",)),
    "newton_mirror_alt": (115, "newton", True, False, False, ("mirror", "alt")),
    "tilted_rot0": (116, "tilted", True, True, False, ()),
}


def lens(name):
    """(table, rot0 or None, clip, np_oracle is the exact-mode truth)"""
    seed, last, clip, rot0, analytic, inner = LENSES[name]
    return random_lens(seed, last, analytic, inner), ROT0 if rot0 else None, clip, analytic


def features(table):
    """the features of one table that the lens matrix must contain"""
    na, flags, mu = table["n_asph"], table["flags"], table["mu"]
    quadric = (na < 0) & (table["c"] != 0)
    out = set()
    if ((na >= 5) & (na <= 10)).any():
        out.add("asph 5..10")
    if ((flags & 2) != 0)[quadric].any():
        out.add("alt")
    if (mu == -1).any():
        out.add("mirror")
    if (mu == 1).any():
        out.add("mu1")
    last = table[-1]
    if last["flags"] & 1:
        out.add("last tilted")
    if last["n_asph"] > 4:
        out.add("last newton")
    if last["mu"] == -1:
        out.add("last mirror")
    if last["n_asph"] < 0:
        if last["c"] == 0:
            out.add("last plane")
        elif last["flags"] & 2:
            out.add("last alt")
        else:
            out.add("last sphere" if last["k"] == 0 else "last conic")
    return out


# 8 independently drawn tables of the same length for rtx_trace_reduce_many
MANY_S = 6
MANY_TABLES = [(900 + i, LAST_KINDS[i % len(LAST_KINDS)], i in (0, 4)) for i in range(8)]


def many_tables():
    return np.stack([random_lens(s, last, analytic, S=MANY_S) for s, last, analytic in MANY_TABLES])


# ---- the per-ray rule -------------------------------------------------------
def ray_moments(y, inc, center, w=None):
    """What rtx_trace_reduce and rtx_trace_reduce_many return for a bundle of
    one ray, for each row of y, inc (N, 3) with the centres (N, 4) (or one
    (4,)) and weights w (N,) or None (= 1).  Returns

      want   (N, 20) float64: every column as the single IEEE double operation
             the kernel applies to the ray (dx = y_x - c_x, ux = i_x/i_z - c_u,
             w dx, ...), gated as in include/rtx.h; m[3], m[18], m[19] as
             numpy evaluates them (their reference where they are not finite);
      ext    (N, 3) long double: m[3], m[18], m[19] in extended precision;
      scale  (N, 3) long double: the magnitudes their bound is relative to,
             w (dx^2 + dy^2), w (|dx ux| + |dy uy|), w (ux^2 + uy^2).

    Evaluated in float64 also for float32 rows (the kernels widen them)."""
    y, i = np.asarray(y, np.float64), np.asarray(inc, np.float64)
    N = len(y)
    c = np.broadcast_to(np.asarray(center, np.float64).reshape(-1, 4), (N, 4))
    w = np.ones(N) if w is None else np.asarray(w, np.float64)
    want = np.zeros((N, 20))
    L = np.longdouble
    ext, scale = np.zeros((N, 3), L), np.zeros((N, 3), L)
    with np.errstate(all="ignore"):
        dx, dy = y[:, 0] - c[:, 0], y[:, 1] - c[:, 1]
        ux, uy = i[:, 0]/i[:, 2] - c[:, 2], i[:, 1]/i[:, 2] - c[:, 3]
        f = np.isfinite(dx) & np.isfinite(dy)
        g = np.isfinite(ux) & np.isfinite(uy)
        want[:, 5] = 1.
        for k, v in ((0, w), (1, w*dx), (2, w*dy), (3, w*(dx*dx + dy*dy)), (4, 1.), (6, dx),
                     (7, dy)):
            want[f, k] = np.broadcast_to(v, (N,))[f]
        for k, v in ((8, 1.), (9, dx), (10, dy), (11, ux), (12, uy), (13, w), (14, w*dx),
                     (15, w*dy), (16, w*ux), (17, w*uy), (18, w*(dx*ux + dy*uy)),
                     (19, w*(ux*ux + uy*uy))):
            want[g, k] = np.broadcast_to(v, (N,))[g]
        lw, ldx, ldy, lux, luy = (np.asarray(a, L) for a in (w, dx, dy, ux, uy))
        e3 = lw*(ldx*ldx + ldy*ldy)
        e18 = lw*(ldx*lux + ldy*luy)
        e19 = lw*(lux*lux + luy*luy)
        ext[f, 0], scale[f, 0] = e3[f], np.abs(e3[f])
        ext[g, 1], scale[g, 1] = e18[g], (np.abs(lw)*(np.abs(ldx*lux) + np.abs(ldy*luy)))[g]
        ext[g, 2], scale[g, 2] = e19[g], np.abs(e19[g])
    return want, ext, scale


def check_rays(got, y, inc, center, w, what):
    """got (N, 20) of N one-ray bundles against ray_moments: the counts and
    the single-operation columns exactly (NaN == NaN, +0 == -0), m[3], m[18],
    m[19] within 2 eps of their scale where numpy's value is finite and equal
    to it elsewhere.  Returns the worst ratio of a contracted column to its
    bound."""
    got = np.asarray(got, np.float64)
    want, ext, scale = ray_moments(y, inc, center, w)
    same = (got == want) | (np.isnan(got) & np.isnan(want))
    cols = [k for k in range(20) if k not in CONTRACTED]
    bad = ~same[:, cols]
    if bad.any():
        r, k = np.argwhere(bad)[0]
        raise AssertionError("%s: %d rays differ, first ray %d m[%d]: got %r, want %r (y %r, i %r)"
                             % (what, bad.any(1).sum(), r, cols[k], got[r, cols[k]],
                                want[r, cols[k]], np.asarray(y)[r], np.asarray(inc)[r]))
    gc, wc = got[:, CONTRACTED], want[:, CONTRACTED]
    fin = np.isfinite(wc)
    assert (same[:, CONTRACTED] | fin).all(), (what, np.argwhere(~same[:, CONTRACTED] & ~fin)[:4])
    with np.errstate(invalid="ignore"):
        err = np.abs(np.asarray(gc, np.longdouble) - ext)
    tol = 2*EPS*scale
    over = fin & ~(err <= tol)
    if over.any():
        r, k = np.argwhere(over)[0]
        raise AssertionError("%s: %d contracted sums off, first ray %d m[%d]: got %r, extended %r, "
                             "scale %r" % (what, over.sum(), r, CONTRACTED[k], gc[r, k],
                                           float(ext[r, k]), float(scale[r, k])))
    with np.errstate(all="ignore"):
        ratio = np.where(fin & (tol > 0), err/np.where(tol > 0, tol, 1), 0)
    return float(ratio.max(initial=0))


# ---- one bundle through every epilogue ---------------------------------------
@pytest.fixture(scope="module")
def eng():
    from rayopt_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def _truth(eng, table, rot0, clip, y0, u0, dy0, du0, dtype, exact, oracle):
    """rows y, u, i at the last surface (host, dtype) and the path sum of the
    launch rays: np_oracle's (`oracle`) or rtx_trace's (keep-last)"""
    N = len(y0)
    if oracle:
        Y, U, I, T = np_oracle.trace(table, y0, u0, clip=clip, rot0=rot0)
        ps = np.zeros(N)
        for t in T:
            ps = ps + t
        return Y[-1], U[-1], I[-1], ps
    Y, U, I, ps = _stored(eng, table, dy0, du0, N, dtype, exact, clip, rot0, path_sum=True)
    return Y[0], U[0], I[0], ps


def _spot_spec(y, inc, rng, radial):
    """5 planes with offsets about a random centre near the rows, the range
    over the middle of their points (so that rays fall inside, outside and
    on the edges)"""
    fin = np.isfinite(y[:, :2]).all(1)
    c = (y[np.argmax(fin), :2].astype(np.float64) if fin.any() else np.zeros(2)) \
        + rng.normal(0, .01, 2)
    z = np.linspace(-.2, .2, 5)
    o = rng.normal(0, .01, (5, 2))
    q = spot_oracle.points(y, inc, c, z, o)
    if radial:
        v = spot_oracle.radii(q)
        v = v[np.isfinite(v)]
        hi = float(np.percentile(v, 90)) if len(v) else 1.
        rng_ = ((0., hi if hi > 1e-9 else 1.),)
        bins = (16,)
    else:
        rng_ = []
        for a in range(2):
            v = q[..., a][np.isfinite(q[..., a])]
            lo, hi = (np.percentile(v, (5, 95)) if len(v) else (-1., 1.))
            if not hi - lo > 1e-9:
                lo, hi = lo - 1., hi + 1.
            rng_.append((float(lo), float(hi)))
        bins = (16, 12)
    return spot_spec(z, bins, rng_, c, radial, o), c, z, o, bins, rng_


def _spot_rays(eng, table, rot0, clip, exact, dy0, du0, idx, y, inc, spec, what):
    """rtx_trace_spot of each ray of `idx` alone, the counts added up: per
    ray the tallies and extents of spot_oracle's points, the counts of all
    of them together"""
    s = spec[0]
    K, radial = int(s["planes"]), bool(s["radial"])
    c, z, o = s["c"], s["z"][:K], s["o"][:K]
    bins = (int(s["nx"]),) if radial else (int(s["nx"]), int(s["ny"]))
    rng_ = tuple(map(tuple, s["range"][:1 if radial else 2]))
    counts = eng.empty(spot_shape(spec), np.uint64)
    eng.memset(counts, 0)
    q = spot_oracle.points(y[idx], inc[idx], c, z, o)                  # (K, n, 2)
    r = spot_oracle.radii(q)
    fin = np.isfinite(q[..., 0]) & np.isfinite(q[..., 1])
    if radial:
        binned = spot_oracle.bin_index(r.ravel(), *rng_[0], bins[0]).reshape(r.shape) >= 0
    else:
        jx = spot_oracle.bin_index(q[..., 0].ravel(), *rng_[0], bins[0]).reshape(r.shape)
        jy = spot_oracle.bin_index(q[..., 1].ravel(), *rng_[1], bins[1]).reshape(r.shape)
        binned = (jx >= 0) & (jy >= 0)
    with np.errstate(invalid="ignore"):
        ext = np.where(fin[..., None], np.stack([np.abs(q[..., 0]), np.abs(q[..., 1]), r], -1), 0.)
    for j, i in enumerate(np.asarray(idx).tolist()):
        tally, e = eng.trace_spot(table, dy0.rows(i), du0.rows(i), spec, counts, N=1, clip=clip,
                                  rot0=rot0, exact=exact, extent=True)
        want_t = np.stack([binned[:, j], ~fin[:, j]], -1).astype(np.uint64)
        assert np.array_equal(tally, want_t), (what, "spot tally of ray", i, tally, want_t)
        assert np.array_equal(e, ext[:, j]), (what, "spot extent of ray", i, e, ext[:, j])
    want = spot_oracle.spot(y[idx], inc[idx], c, z, bins, rng_, radial, o)[0]
    got = counts.download()
    counts.free()
    assert np.array_equal(got, want), (what, "spot counts of the one-ray launches")


def run_bundle(eng, table, rot0, clip, y0, u0, mode, oracle, sub, seed, what):
    """every epilogue on one bundle (y0, u0 float64 host) against the truth;
    `sub` the rays also launched one by one.  Returns the worst ratios of the
    contracted columns and of the whole-bundle sums to their bounds."""
    dtype, exact = MODES[mode]
    N = len(y0)
    rng = np.random.default_rng(seed)
    dy0, du0 = eng.to_device(y0, dtype), eng.to_device(u0, dtype)
    y, u, inc, ps = _truth(eng, table, rot0, clip, y0, u0, dy0, du0, dtype, exact, oracle)
    worst = [0., 0.]
    # OPD: A and P of every ray
    k = int(rng.integers(6))
    spec = _spec(y0, u0, y, 1.0, float(table["n"][-1]) or 1.0, k % 2 == 0, .02*(k % 3))
    A, P = eng.empty((N,), dtype), eng.empty((N, 3), dtype)
    eng.trace_opd(table, dy0, du0, spec, A, P, N=N, clip=clip, rot0=rot0, exact=exact)
    eng.sync()
    a, p = A.download(), P.download()
    A.free(), P.free()
    wa, wp = epi_oracle.opd_epilogue(y0.astype(dtype), y, u, ps, spec)
    assert a.dtype == wa.dtype
    bad = ~((a == wa) | (np.isnan(a) & np.isnan(wa))) | \
        ~((p == wp) | (np.isnan(p) & np.isnan(wp))).all(1)
    assert not bad.any(), (what, "OPD", np.flatnonzero(bad)[:8])
    # many: one item per ray
    centers = np.c_[rng.normal(0, 1, (N, 2)), rng.normal(0, .05, (N, 2))]
    bundles = [(dy0.rows(i), du0.rows(i), 1) for i in range(N)]
    m = eng.trace_reduce_many(table[None], bundles, np.c_[np.zeros(N, int), np.arange(N)],
                              centers, clip=clip, rot0=rot0, exact=exact)
    worst[0] = check_rays(m, y, inc, centers, None, "%s many" % what)
    # reduce: the whole bundle within the bound
    dw = eng.to_device(rng.uniform(.5, 2., N), dtype)
    wh = dw.download().astype(np.float64)
    center = centers[0]
    m = eng.trace_reduce(table, dy0, du0, N=N, clip=clip, rot0=rot0, exact=exact, w=dw,
                         center=center)
    s, sa = epi_oracle.reduce_sums(y, inc, wh, center)
    for j in (4, 5, 8):
        assert m[j] == s[j], (what, j, m[j], s[j])
    worst[1] = _within(m, s, sa, _L_epi(eng, N), "%s reduce" % what)
    # reduce: one ray at a time, every other one weighted
    for j, i in enumerate(np.asarray(sub).tolist()):
        wi = dw.rows(i) if j % 2 else None
        m = eng.trace_reduce(table, dy0.rows(i), du0.rows(i), N=1, clip=clip, rot0=rot0,
                             exact=exact, w=wi, center=centers[i])
        r = check_rays(m[None], y[i:i + 1], inc[i:i + 1], centers[i], wh[i:i + 1] if j % 2 else
                       None, "%s reduce ray %d" % (what, i))
        worst[0] = max(worst[0], r)
    dw.free()
    # spot: the whole bundle, then one ray at a time
    sspec, c, z, o, bins, rng_ = _spot_spec(y, inc, rng, radial=k % 2 == 1)
    counts = eng.empty(spot_shape(sspec), np.uint64)
    eng.memset(counts, 0)
    tally, ext = eng.trace_spot(table, dy0, du0, sspec, counts, N=N, clip=clip, rot0=rot0,
                                exact=exact, extent=True)
    wc, wt, we = spot_oracle.spot(y, inc, c, z, bins, rng_, k % 2 == 1, o)
    got = counts.download()
    counts.free()
    assert np.array_equal(got, wc), (what, "spot counts", np.argwhere(got != wc)[:5])
    assert np.array_equal(tally, wt) and np.array_equal(ext, we), (what, tally, wt, ext, we)
    _spot_rays(eng, table, rot0, clip, exact, dy0, du0, sub, y, inc, sspec, what)
    dy0.free(), du0.free()
    return worst


# ---- the tests ----------------------------------------------------------------
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("name", list(LENSES))
def test_lens(eng, name, mode):
    """random bundles of N = 1 .. 70001 and one with non-finite and signed-zero
    launch components through a seeded random lens; the subsample is SUB
    rays of the largest bundle and every special ray of the mixed one"""
    table, rot0, clip, analytic = lens(name)
    oracle = analytic and mode == "f64_exact" and rot0 is None
    seed = LENSES[name][0]
    worst = [0., 0.]
    for k, N in enumerate(NS + [513]):
        y0, u0 = random_rays(np.random.default_rng(10*seed + k), N)
        sub = np.arange(0)
        if N == NS[-1]:
            sub = np.random.default_rng(seed).choice(N, SUB, replace=False)
        if k == len(NS):
            # launch rays with a NaN, +-inf or +-0 component in warps of
            # ordinary ones: outside the oracle's promise, so against rtx_trace
            y0, u0, _ = eb.mixed_bundle(y0, u0, seed)
            special = np.zeros(N, bool)
            special[1::4] = True
            sub = np.flatnonzero(special)
        w = run_bundle(eng, table, rot0, clip, y0, u0, mode, oracle and k < len(NS), sub,
                       seed + k, "%s %s N=%d" % (name, mode, N))
        worst = [max(a, b) for a, b in zip(worst, w)]
    print("%s %s: worst contracted / bound %.3g, sums / bound %.3g" % (name, mode, *worst))


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("name", list(EDGE))
def test_edge_bundle(eng, name, mode):
    """every decision-boundary bundle of oracle/edge_bundles.py, every ray
    also alone; exact FP64 against np_oracle's rows"""
    c = EDGE[name]
    run_bundle(eng, c.table, None, c.clip, c.y0, c.u0, mode, mode == "f64_exact",
               np.arange(len(c.y0)), 7, "%s %s" % (name, mode))


TILES = {"sm-1": (1, -1), "sm": (1, 0), "sm+1": (1, 1), "2sm-1": (2, -1), "2sm": (2, 0),
         "2sm+1": (2, 1)}
RAGGED = [1, 511, 512, 513, 4097]


@pytest.mark.parametrize("tiles", list(TILES))
@pytest.mark.parametrize("mode", list(MODES))
def test_many_tables_that_differ(eng, mode, tiles):
    """rtx_trace_reduce_many over 8 unrelated tables: one-ray items cycling
    through them (a restage on every tile), ragged items and items without
    rays, the total tile count around one and two CTAs per SM.  One-ray items
    per ray against the rows of their own table, ragged items within the
    bound, empty items zero."""
    dtype, exact = MODES[mode]
    mult, off = TILES[tiles]
    total = mult*eng.sm_count + off
    clip, rot0 = off != 0, ROT0 if mult == 2 else None
    tabs = many_tables()
    nt = len(tabs)
    rng = np.random.default_rng(17 + total)
    n_one = total - sum(-(-n//512) for n in RAGGED)
    y1, u1 = random_rays(rng, n_one)
    y1, u1, _ = eb.mixed_bundle(y1, u1, total)
    d1, e1 = eng.to_device(y1, dtype), eng.to_device(u1, dtype)
    bundles = [(d1.rows(i), e1.rows(i), 1) for i in range(n_one)]
    host = {}
    for n in RAGGED:
        y, u = random_rays(rng, n)
        host[len(bundles)] = (y, u)
        bundles.append((eng.to_device(y, dtype), eng.to_device(u, dtype), n))
    bundles.append((d1, e1, 0))
    empty = len(bundles) - 1
    items = [(i % nt, i) for i in range(n_one)]
    for b in sorted(host):                                    # ragged items among the one-ray ones
        items.insert(int(rng.integers(0, len(items) + 1)), (int(rng.integers(nt)), b))
    items.insert(len(items)//3, (0, empty))
    items.append((nt - 1, empty))
    items = np.array(items)
    centers = np.c_[rng.normal(0, 1, (len(items), 2)), rng.normal(0, .05, (len(items), 2))]
    m = eng.trace_reduce_many(tabs, bundles, items, centers, clip=clip, rot0=rot0, exact=exact)
    assert sum(-(-bundles[b][2]//512) for _, b in items) == total
    one = items[:, 1] < n_one
    for t in range(nt):
        sel = np.flatnonzero(one & (items[:, 0] == t))
        rays = items[sel, 1]
        dy, du = eng.to_device(y1[rays], dtype), eng.to_device(u1[rays], dtype)
        Y, _, I, _ = _stored(eng, tabs[t], dy, du, len(rays), dtype, exact, clip, rot0)
        dy.free(), du.free()
        check_rays(m[sel], Y[0], I[0], centers[sel], None, "%s %s table %d" % (mode, tiles, t))
    for i in np.flatnonzero(~one):
        t, b = items[i]
        if b == empty:
            assert np.array_equal(m[i], np.zeros(20)), (i, m[i])
            continue
        y, u = host[b]
        dy, du = bundles[b][0], bundles[b][1]
        Y, _, I, _ = _stored(eng, tabs[t], dy, du, len(y), dtype, exact, clip, rot0)
        s, a = epi_oracle.reduce_sums(Y[0], I[0], None, centers[i])
        for j in (4, 5, 8):
            assert m[i, j] == s[j], (i, j, m[i, j], s[j])
        _within(m[i], s, a, -(-len(y)//512), "%s %s item %d" % (mode, tiles, i))
    for b in host:
        bundles[b][0].free(), bundles[b][1].free()
    d1.free(), e1.free()
