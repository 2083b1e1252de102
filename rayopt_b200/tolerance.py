"""Tolerance analysis on the device: trace many perturbed copies of a lens in
one launch (rtx_trace_reduce_many) and reduce each to its spot moments.

A perturbation is a list of parameters ``(j, kind)`` (j the index of a
surface in the ``System``, >= 1) and a (V, P) array of deltas, one row per
variant of the lens.  ``perturbed_tables`` applies them to the packed surface
tables with ``pack_system``'s own expressions, so that a variant's records
are the records of the ``System`` with the same change made.

``tolerance`` aims every field and wavelength of the NOMINAL lens once
(``system.pupil`` on the host, the launch rays generated in HBM) and marches
that one object-space bundle through every variant: variants are not
re-aimed, so a perturbation that moves the stop shows up as vignetting, and
the stop and apertures of the perturbed lens decide which rays pass.
"""
import copy
import math

import numpy as np

from .engine import Engine, default_engine
from .surface_table import F_ROTATED, RTX_MAX_ASPH, SURFACE_DTYPE, pack_system

KINDS = ("curvature", "conic", "distance", "tilt_x", "tilt_y", "index") + tuple(
    "asph%d" % i for i in range(RTX_MAX_ASPH))

# rayopt's TransformMixin.update treats angles within np.allclose's default
# absolute tolerance of 0 as no rotation at all
_ANGLE_ATOL = 1e-8


def _rot_rxyz(a):
    """``rot_normal`` of a straight element with Euler angles `a` (rayopt's
    TransformMixin.update, elements.py:120-154): the rotating-frame x-y-z
    Euler matrix (axes "rxyz"), composed onto the identity as the reference
    composes it"""
    # rotating x-y-z: the angle sequence enters reversed and negated
    si, sj, sk = math.sin(-a[2]), math.sin(-a[1]), math.sin(-a[0])
    ci, cj, ck = math.cos(-a[2]), math.cos(-a[1]), math.cos(-a[0])
    cc, cs = ci*ck, ci*sk
    sc, ss = si*ck, si*sk
    M = np.identity(3)
    M[2, 2] = cj*ck
    M[2, 1] = sj*sc - cs
    M[2, 0] = sj*cc + ss
    M[1, 2] = cj*sk
    M[1, 1] = sj*ss + cc
    M[1, 0] = sj*cs - sc
    M[0, 2] = -sj
    M[0, 1] = cj*si
    M[0, 0] = cj*ci
    return np.dot(np.eye(3), M)


def _parse(params, S):
    out = []
    for j, kind in params:
        if kind not in KINDS:
            raise ValueError("unknown tolerance kind %r" % (kind,))
        if int(j) != j or not 1 <= j <= S:
            raise ValueError("surface %r is not in 1..%d" % (j, S))
        out.append((int(j), kind))
    return out


def _checked(tables, params):
    """(tables as (W, S) records, params parsed) after every refusal
    perturbed_tables and record_tangents share (ValueError)"""
    tables = np.asarray(tables, SURFACE_DTYPE)
    if tables.ndim == 1:
        tables = tables[None]
    S = tables.shape[1]
    params = _parse(params, S)
    for j, kind in params:
        r = tables[:, j - 1]
        if kind == "distance" and np.any(r["offset"][:, :2] != 0):
            raise ValueError("surface %d is not on the axis of its predecessor" % j)
        if kind in ("tilt_x", "tilt_y") and np.any(r["flags"] & F_ROTATED):
            raise ValueError("surface %d is already rotated" % j)
        if kind == "index":
            if j == S:
                raise ValueError("surface %d is the last: no medium follows it" % j)
            for rr in (r, tables[:, j]):
                if np.any(rr["mu"] == -1):
                    raise ValueError("index of surface %d: a mirror bounds the medium" % j)
                if np.any((rr["mu"] == 1) & (rr["n"] == rr["n0"])):
                    raise ValueError("index of surface %d: the medium after it is not "
                                     "bounded by two materials" % j)
    return tables, params


def _move_distance(off_z, d):
    """rayopt's ``distance += d`` on the offset's z (the element's length
    along its direction, +z or, for a negative distance, -z)"""
    return np.where(np.signbit(off_z), off_z - d, off_z + d)


def perturbed_tables(tables, params, deltas):
    """The (V, W, S) tables of V perturbed lenses from the nominal (W, S)
    tables (one per wavelength, ``pack_system(system, l)``), the parameters
    `params` [(j, kind)] and `deltas` (V, P).

    kind       what changes in record j-1
    curvature  c, then kc2
    conic      k, then kc2
    asph<i>    aspheric coefficient i and its derivative; a non-zero delta on
               a surface without aspherics (or with fewer than i+1) makes it a
               Newton surface of i+1 coefficients
    distance   offset[2] (the element's distance); refused for an offset with
               x or y != 0
    tilt_x/_y  the Euler angles of an unrotated element (a tilt about the
               surface vertex); refused for a rotated record
    index      the index of the medium after surface j at every wavelength: n
               and mu of record j-1, n0 and mu of record j; refused for the
               last surface, a mirror, or a surface that does not bound a
               medium (mu = 1 and n = n0) on either side

    Raises ValueError before building anything."""
    tables, params = _checked(tables, params)
    deltas = np.asarray(deltas, np.float64)
    if deltas.ndim != 2 or deltas.shape[1] != len(params):
        raise ValueError("deltas must be (V, %d), got %s" % (len(params), deltas.shape))
    V = deltas.shape[0]
    out = np.repeat(tables[None], V, axis=0)
    kc2_rows, mu_rows, angles = set(), set(), {}
    for p, (j, kind) in enumerate(params):
        r, d = j - 1, deltas[:, p, None]                       # (V, 1) over W
        if kind == "curvature":
            out["c"][:, :, r] += d
            kc2_rows.add(r)
        elif kind == "conic":
            out["k"][:, :, r] += d
            kc2_rows.add(r)
        elif kind.startswith("asph"):
            i = int(kind[4:])
            out["asph"][:, :, r, i] += d
            out["dasph"][:, :, r, i] = 2*(i + 1)*out["asph"][:, :, r, i]    # elements.py:472
            na = out["n_asph"][:, :, r]
            out["n_asph"][:, :, r] = np.where(d != 0, np.maximum(na, i + 1), na)
        elif kind == "distance":
            out["offset"][:, :, r, 2] = _move_distance(out["offset"][:, :, r, 2], d)
        elif kind in ("tilt_x", "tilt_y"):
            angles.setdefault(r, np.zeros((V, 3)))[:, int(kind == "tilt_y")] += deltas[:, p]
        else:                                                  # index
            out["n"][:, :, r] += d
            out["n0"][:, :, r + 1] += d
            mu_rows.update((r, r + 1))
    for r in kc2_rows:
        out["kc2"][:, :, r] = (1 + out["k"][:, :, r])*out["c"][:, :, r]**2   # elements.py:448,467
    for r in mu_rows:                                          # Interface.get_n_mu, elements.py:283-289
        mu = out["n0"][:, :, r]/out["n"][:, :, r]
        out["mu"][:, :, r] = mu
        out["muf"][:, :, r] = np.abs(mu)
        out["sgn"][:, :, r] = np.sign(mu)
        out["mu2m1"][:, :, r] = mu**2 - 1
    for r, a in angles.items():
        for v in range(V):
            if np.all(np.abs(a[v]) <= _ANGLE_ATOL):
                continue
            out["rot"][v, :, r] = _rot_rxyz([float(x) for x in a[v]]).reshape(9)
            out["flags"][v, :, r] |= F_ROTATED
    return out


# d rot_normal / d angle of _rot_rxyz at zero angles, for the angles tilt_x
# (a[0]) and tilt_y (a[1]) move
_ROT_GENERATOR = {"tilt_x": np.array([[0., 0., 0.], [0., 0., -1.], [0., 1., 0.]]),
                  "tilt_y": np.array([[0., 0., 1.], [0., 0., 0.], [-1., 0., 0.]])}


def record_tangents(tables, params):
    """The derivative of perturbed_tables(tables, params, deltas) with
    respect to each delta at deltas = 0, with the same refusals: a list of P
    parameters, each a list of moves (row, records), `records` the (W,)
    derivatives of tables[:, row] (SURFACE_DTYPE; a single record for a 1-D
    table).  Only the fields perturbed_tables moves are non-zero:

    kind       fields of row j-1 (index: and of row j)
    curvature  c = 1, kc2 = (1 + k) 2c
    conic      k = 1, kc2 = c^2
    distance   offset z = +-1, the sign of _move_distance
    asph<i>    asph[i] = 1, dasph[i] = 2(i + 1)
    tilt_x/_y  rot = the generator of _rot_rxyz at zero angles
    index      row j-1: n = 1, mu = -mu/n, muf = sgn dmu, mu2m1 = 2 mu dmu;
               row j: n0 = 1, mu = 1/n, muf = sgn dmu, mu2m1 = 2 mu dmu

    Moves are the unit the device Jacobian takes (Engine.trace_jacobian), so
    a caller may build its own: [(j, d_dist_j), (j + 1, -d_dist_{j+1})]
    shifts a group of surfaces."""
    one = np.asarray(tables).ndim == 1
    tables, params = _checked(tables, params)
    out = []
    for j, kind in params:
        r = j - 1
        t = tables[:, r]
        rec = np.zeros(t.shape, SURFACE_DTYPE)
        moves = [(r, rec)]
        if kind == "curvature":
            rec["c"] = 1
            rec["kc2"] = (1 + t["k"])*2*t["c"]
        elif kind == "conic":
            rec["k"] = 1
            rec["kc2"] = t["c"]**2
        elif kind.startswith("asph"):
            i = int(kind[4:])
            rec["asph"][:, i] = 1
            rec["dasph"][:, i] = 2*(i + 1)
        elif kind == "distance":
            rec["offset"][:, 2] = np.where(np.signbit(t["offset"][:, 2]), -1., 1.)
        elif kind in ("tilt_x", "tilt_y"):
            rec["rot"] = _ROT_GENERATOR[kind].reshape(9)
        else:                                                  # index
            rec2 = np.zeros(t.shape, SURFACE_DTYPE)
            moves.append((r + 1, rec2))
            for x, row, dn, dn0 in ((rec, t, 1., 0.), (rec2, tables[:, r + 1], 0., 1.)):
                mu, n = row["mu"], row["n"]
                dmu = (dn0 - mu*dn)/n                          # d(n0/n)
                x["n"], x["n0"], x["mu"] = dn, dn0, dmu
                x["muf"] = np.sign(mu)*dmu
                x["mu2m1"] = 2*mu*dmu
        out.append([(row, x[0] if one else x) for row, x in moves])
    return out


def sensitivity_deltas(tol):
    """(1 + 2P, P) deltas: row 0 the nominal lens, then +tol_p e_p and
    -tol_p e_p for each parameter p in turn"""
    tol = np.asarray(tol, np.float64).reshape(-1)
    P = len(tol)
    d = np.zeros((1 + 2*P, P))
    d[1 + 2*np.arange(P), np.arange(P)] = tol
    d[2 + 2*np.arange(P), np.arange(P)] = -tol
    return d


def monte_carlo_deltas(tol, trials, seed=None):
    """(trials, P) deltas uniform in [-tol, tol] from np.random.default_rng(seed)"""
    tol = np.asarray(tol, np.float64).reshape(-1)
    return np.random.default_rng(seed).uniform(-tol, tol, (int(trials), len(tol)))


def _nominal(system, wavelengths):
    """the nominal lens's (W, S) tables, one per wavelength, and its rot0"""
    packs = [pack_system(system, l, 1, None, n0=system.refractive_index(l, 0)) for l in wavelengths]
    return np.stack([t for t, _, _ in packs]), packs[0][2]


def _centers(eng, nominal, rot0, chiefs, exact):
    """(bundles, 4) (y_x, y_y, u_x, u_y) of each bundle's chief ray (the
    launch rays `chiefs` of launch_bundles) at the last surface of
    nominal[b % W], zeros where it does not get there"""
    out = np.zeros((len(chiefs), 4))
    for b, (y0, u0) in enumerate(chiefs):
        Y, _, I, _ = eng.trace(nominal[b % len(nominal)], y0, u0, clip=True, rot0=rot0,
                               keep_last=True, exact=exact, want=("y", "i"))
        with np.errstate(all="ignore"):
            c = np.r_[Y[0, 0, :2], I[0, 0, :2]/I[0, 0, 2]].astype(np.float64)
        if np.all(np.isfinite(c)):
            out[b] = c
    return out


def launch_bundles(system, heights, wavelengths, nrays, distribution, engine):
    """The nominal lens's launch rays of each (height, wavelength), generated
    in HBM: a list of (y0, u0) DeviceArrays in height-major order and the
    launch rays (2, 3) of each bundle's chief ray on the host"""
    from .rays import aim_record, grid_spec
    ref, grid = grid_spec(distribution, nrays)
    if grid is None:
        raise ValueError("distribution %r with %d rays is not generated on the device"
                         % (distribution, nrays))
    bundles, chiefs = [], []
    for h in heights:
        for l in wavelengths:
            yo = (0, h)
            z, p = system.pupil(yo, l=l)
            rec = aim_record(system.object, yo, z, p, grid, False, system[0])
            bundles.append(engine.aim_rays(rec))
            cy, cu = engine.aim_rays(rec, first=ref, count=1)
            chiefs.append((cy.download(), cu.download()))
            cy.free(), cu.free()
    return bundles, chiefs


def _focus_bundles(system, l, engine):
    """GeometricTrace.refocus's bundle in Analysis.run (analysis.py:84-88):
    13 Radau rays on axis at `l`, unclipped, as given pupil coordinates.  The
    reference weights them, and rtx_trace_reduce_many does not, so the rays
    are split into one bundle per weight: [(weight, y0, u0)]"""
    from rayopt.utils import pupil_distribution           # the reference's own helper
    from .rays import aim_record
    _, yp, weight = pupil_distribution("radau", 13)
    yp = np.asarray(yp, np.float64)
    w = np.ones(len(yp)) if weight is None else np.asarray(weight, np.float64)
    z, p = system.pupil((0, 0.), l=l)
    rec = aim_record(system.object, (0, 0.), z, p, None, False, system[0])
    out = []
    for wv in np.unique(w):
        dyp = engine.to_device(yp[w == wv])
        y0, u0 = engine.aim_rays(rec, yp=dyp)
        dyp.free()
        out.append((float(wv), y0, u0))
    return out


def focus_shifts(m, weights):
    """GeometricTrace.refocus's shift from the unweighted moments m (..., G,
    20) of G groups of rays that carry the weights `weights` (G,): the
    weighted sums are sum_g w_g m_g"""
    m = np.asarray(m, np.float64)
    w = np.asarray(weights, np.float64)
    tot = m.sum(-2)
    tot[..., 13:20] = (m[..., 13:20]*w[:, None]).sum(-2)
    return np.array([Engine.focus_shift_from_moments(t) for t in tot.reshape(-1, 20)]
                    ).reshape(tot.shape[:-1])


def _variant_chunk(tables_bytes_per_variant, tiles_per_variant, budget, row_bytes=160,
                   items_per_variant=0):
    """variants per launch whose device tables, tile rows and item rows
    (`row_bytes` each: 20 moments, or an OTF row) fit in `budget` bytes"""
    per = tables_bytes_per_variant + row_bytes*(tiles_per_variant + items_per_variant) + 1
    return max(1, int(budget//per))


def _focus(eng, fsys, nominal, params, deltas, l, rot0, step, exact):
    """(V,) GeometricTrace.refocus's shift of every variant: 13 Radau rays
    on axis at `l`, unclipped, aimed on `fsys` (the NOMINAL lens), marched
    through each variant's table at `l` (nominal[0]), `step` variants per
    launch"""
    fb = _focus_bundles(fsys, l, eng)
    try:
        G, V = len(fb), len(deltas)
        focus = np.empty(V)
        for v0 in range(0, V, step):
            t = perturbed_tables(nominal[:1], params, deltas[v0:v0 + step])[:, 0]
            n = len(t)
            items = np.stack(np.meshgrid(np.arange(n), np.arange(G), indexing="ij"),
                             -1).reshape(-1, 2)
            m = eng.trace_reduce_many(t, [(y, u, None) for _, y, u in fb], items,
                                      clip=False, rot0=rot0, exact=exact)
            focus[v0:v0 + n] = focus_shifts(m.reshape(n, G, 20), [w for w, _, _ in fb])
    finally:
        for _, y, u in fb:
            y.free(), u.free()
    return focus


def check_fields(system, heights, wavelengths, compensate, chunk):
    """(heights, wavelengths) as lists, after the refusals of the arguments
    every tolerance analysis takes (ValueError)"""
    if compensate not in (None, "focus"):
        raise ValueError("compensate must be None or 'focus', got %r" % (compensate,))
    if chunk is not None and int(chunk) < 1:
        raise ValueError("chunk must be >= 1, got %r" % (chunk,))
    heights = list(heights)
    wavelengths = list(system.wavelengths if wavelengths is None else wavelengths)
    if not heights or not wavelengths:
        raise ValueError("need at least one height and one wavelength")
    return heights, wavelengths


class VariantMarch:
    """The host side of every tolerance analysis, whose arguments it takes
    (heights and wavelengths from check_fields).  On construction: the
    nominal lens packed per wavelength (`nominal` (W, S), `rot0`),
    perturbed_tables' refusals of `params` and `deltas` (V, P) and, for a
    `wavefront` analysis, of a shape or tilt of the image surface (it
    changes only the reference sphere), all before any device work; then
    the launch bundles of the nominal lens (`dev`, height-major, `chiefs`
    their chief rays, `counts` (H, W) their rays) and, for a `wavefront`
    analysis, the chief-ray reference `ref` on the device.  Everything it
    put on the device is freed when the ``with`` block it opens ends, or
    when construction fails."""

    def __init__(self, system, params, deltas, heights, wavelengths, nrays, distribution,
                 compensate, chunk, engine, exact, wavefront=False):
        self.nominal, self.rot0 = _nominal(system, wavelengths)
        S = self.nominal.shape[1]
        self.params = list(params)
        deltas = np.asarray(deltas, np.float64)
        self.deltas = deltas[None] if deltas.ndim == 1 else deltas
        perturbed_tables(self.nominal, self.params, self.deltas[:0])
        for j, kind in self.params:
            if wavefront and j == S and kind != "distance":
                raise ValueError("%s of the image surface %d changes only the reference sphere"
                                 % (kind, j))
        self.V, self.H, self.W = len(self.deltas), len(heights), len(wavelengths)
        self.heights, self.wavelengths = heights, wavelengths
        self.compensate, self.chunk, self.exact = compensate, chunk, exact
        self.focus = None
        self.eng = engine or default_engine()
        # System.pupil's result depends on the calls made before it: the focus
        # bundle is aimed on a copy taken before any
        self.fsys = copy.deepcopy(system) if compensate == "focus" else None
        self.bundles, self.chiefs = launch_bundles(system, heights, wavelengths, nrays,
                                                   distribution, self.eng)
        self.dev = [(y, u, None) for y, u in self.bundles]
        self.counts = np.array([y.shape[0] for y, _ in self.bundles],
                               np.float64).reshape(self.H, self.W)
        self.ref = None
        try:
            if wavefront:
                self.ref = _WavefrontRef(system, self.nominal, wavelengths, self.chiefs)
                self.ref.upload(self.eng)
        except BaseException:
            self.close()
            raise

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def close(self):
        for y, u in self.bundles:
            y.free(), u.free()
        self.bundles = []
        if self.ref is not None:
            self.ref.free()

    def chunks(self, row_bytes=160, items_per_variant=0):
        """Refocus every variant when compensating, then yield (v0, t, items)
        for each chunk of n variants v0 .. v0+n-1: t (n, W, S) their
        perturbed tables with the image surface moved by each one's focus
        shift, items (n*H*W, 2) the (table, bundle) of every variant and
        bundle, (v*W + w, h*W + w).  A chunk is `chunk` variants, or as many
        as fit in 1 GiB of tables, tile rows and `items_per_variant` item
        rows of `row_bytes` each."""
        nb = len(self.bundles)
        W, S = self.nominal.shape[:2]
        tiles = sum(-(-y.shape[0]//512) for y, _ in self.bundles)
        step = int(self.chunk) if self.chunk else _variant_chunk(W*S*512, tiles, 2**30, row_bytes,
                                                                 items_per_variant)
        if self.compensate == "focus":
            self.focus = _focus(self.eng, self.fsys, self.nominal, self.params, self.deltas,
                                self.wavelengths[0], self.rot0, step, self.exact)
        for v0 in range(0, self.V, step):
            t = perturbed_tables(self.nominal, self.params, self.deltas[v0:v0 + step])
            n = len(t)
            if self.focus is not None:                         # system[-1].distance += shift
                t["offset"][:, :, -1, 2] = _move_distance(t["offset"][:, :, -1, 2],
                                                          self.focus[v0:v0 + n, None])
            v, b = (a.reshape(-1) for a in np.meshgrid(np.arange(n), np.arange(nb), indexing="ij"))
            yield v0, t, np.stack([v*W + b % W, b], -1)

    def result(self, out):
        """`out` with heights, wavelengths, params, deltas and, when
        compensated, focus"""
        out.update(heights=np.asarray(self.heights, np.float64),
                   wavelengths=np.asarray(self.wavelengths, np.float64), params=self.params,
                   deltas=self.deltas)
        if self.focus is not None:
            out["focus"] = self.focus
        return out


def tolerance(system, params, deltas, heights=(0., .707, 1.), wavelengths=None, nrays=1000,
              distribution="hexapolar", compensate=None, engine=None, exact=False, chunk=None):
    """Spot rms, transmission and centroid of every perturbed lens at every
    field height and wavelength, on the device.

    `system` a rayopt ``System``; `params` [(j, kind)] and `deltas` (V, P) as
    ``perturbed_tables``.  Each (height, wavelength) bundle is aimed once for
    the NOMINAL lens and shared by all V variants (no re-aiming); the rays are
    clipped by the perturbed lens.  ``compensate="focus"`` first refocuses
    each variant as Analysis does (13 Radau rays on axis at wavelengths[0],
    unclipped) and moves its image surface by the shift.  `chunk`: variants
    per launch (default: as many as fit in 1 GiB of tables and tile sums);
    the results do not depend on it.

    Returns a dict: rms (V, H, W) about the mean of the rays that reach the
    image, transmitted (V, H, W) the fraction that does, centroid (V, H, W,
    2) relative to the nominal chief ray, moments (V, H, W, 20), focus (V,)
    when compensated, and heights, wavelengths, params, deltas."""
    heights, wavelengths = check_fields(system, heights, wavelengths, compensate, chunk)
    with VariantMarch(system, params, deltas, heights, wavelengths, nrays, distribution,
                      compensate, chunk, engine, exact) as r:
        centers = _centers(r.eng, r.nominal, r.rot0, r.chiefs, exact)
        H, W, S = r.H, r.W, r.nominal.shape[1]
        m = np.empty((r.V, H, W, 20))
        for v0, t, items in r.chunks():
            n = len(t)
            m[v0:v0 + n] = r.eng.trace_reduce_many(
                t.reshape(n*W, S), r.dev, items, centers[items[:, 1]], clip=True, rot0=r.rot0,
                exact=exact).reshape(n, H, W, 20)
    with np.errstate(all="ignore"):
        out = dict(rms=Engine.rms_finite_from_moments(m), transmitted=m[..., 4]/m[..., 5],
                   centroid=np.stack([m[..., 1]/m[..., 0], m[..., 2]/m[..., 0]], -1), moments=m)
    return r.result(out)


def _otf_targets(targets, shape):
    """`targets` broadcast to (H, 2, F), ValueError when it does not"""
    try:
        return np.broadcast_to(np.asarray(targets, np.float64), shape)
    except ValueError:
        raise ValueError("targets of shape %s does not broadcast to (heights, 2, freqs) = %s"
                         % (np.shape(targets), shape)) from None


def mtf_tolerance_result(sums, count, weights, targets=None):
    """tolerance_mtf's result from the OTF sums (V, H, W, K, 2, F) complex
    and counts (V, H, W, K): otf = sums/count (NaN where nothing counted),
    mtf, poly (V, H, K, 2, F) (mtf.poly_otf with the spectral `weights`)
    and poly_mtf; with `targets` (broadcast to (H, 2, F)) passed (V, K),
    true where every poly MTF of the plane is at or above its target (NaN
    fails), and yield (K,) the fraction of variants that pass"""
    from .mtf import _otf, poly_otf
    sums = np.asarray(sums, np.complex128)
    count = np.asarray(count, np.int64)
    V, H, W, K, _, F = sums.shape
    otf = _otf(sums, count)
    poly = poly_otf(otf.reshape(V*H, W, K, 2, F), count.reshape(V*H, W, K),
                    weights).reshape(V, H, K, 2, F)
    out = dict(otf=otf, mtf=np.abs(otf), count=count, poly=poly, poly_mtf=np.abs(poly))
    if targets is not None:
        t = _otf_targets(targets, (H, 2, F))
        with np.errstate(invalid="ignore"):
            ok = out["poly_mtf"] >= t[:, None]
        out["passed"] = ok.all(axis=(1, 3, 4))
        out["yield"] = out["passed"].mean(0)
    return out


def tolerance_mtf(system, params, deltas, freqs, heights=(0., .707, 1.), wavelengths=None,
                  nrays=1000, distribution="hexapolar", defocus=(0.,), compensate=None,
                  spectral_weights=None, targets=None, engine=None, exact=False, chunk=None):
    """Geometric OTF and MTF of every perturbed lens at the frequencies
    `freqs` (cycles per length unit), every field height, wavelength and
    defocus plane, on the device: the MTF counterpart of ``tolerance``.

    `params` [(j, kind)] and `deltas` (V, P) are ``perturbed_tables``'.
    Each (height, wavelength) bundle is aimed once for the NOMINAL lens and
    marched through all V variants with clipping (no re-aiming); every
    variant's bundles are reduced to their OTF sums in the same launch as
    the march (rtx_trace_otf_many).  As in geometric_mtf, every wavelength
    of a height is centred on the nominal chief ray at wavelengths[0]; the
    MTF does not depend on the centre.  `defocus` are up to 16 plane
    distances from the image surface.  ``compensate="focus"`` refocuses each
    variant first, as ``tolerance`` does.  `targets` (broadcast to (H, 2,
    F)) are the minimum polychromatic MTF of an accepted lens.  `chunk`:
    variants per launch (default: as many as fit in 1 GiB of tables and tile
    rows); the results do not depend on it.

    Returns a dict: freq (F,), z (K,), otf complex (V, H, W, K, 2, F)
    (axis 0: x, sagittal; 1: y, tangential), mtf = |otf|, count (V, H, W,
    K), poly (V, H, K, 2, F) the `spectral_weights` mean of the
    wavelengths' OTFs (mtf.poly_otf), poly_mtf = |poly|, focus (V,) when
    compensated, heights, wavelengths, params, deltas; with `targets`
    also passed (V, K) (every poly MTF of the plane at or above its target,
    NaN failing) and yield (K,), the fraction of variants that pass.
    Every argument is checked before any device work."""
    from .engine import OTF_MAX_PLANES
    from .mtf import _check_freqs, _spectral
    heights, wavelengths = check_fields(system, heights, wavelengths, compensate, chunk)
    H, W = len(heights), len(wavelengths)
    nu = _check_freqs(freqs)
    z = np.atleast_1d(np.asarray(defocus, np.float64))
    if z.ndim != 1 or not 1 <= len(z) <= OTF_MAX_PLANES or not np.isfinite(z).all():
        raise ValueError("defocus must be 1..%d finite distances, got %r" % (OTF_MAX_PLANES, defocus))
    F, K = len(nu), len(z)
    sw = _spectral(spectral_weights, W)
    if targets is not None:
        targets = _otf_targets(targets, (H, 2, F))
    with VariantMarch(system, params, deltas, heights, wavelengths, nrays, distribution,
                      compensate, chunk, engine, exact) as r:
        # the chief ray of each height at wavelengths[0], for every wavelength
        centers = _centers(r.eng, r.nominal[:1], r.rot0, r.chiefs[::W], exact)[:, :2]
        S = r.nominal.shape[1]
        sums = np.empty((r.V, H, W, K, 2, F), np.complex128)
        count = np.empty((r.V, H, W, K), np.int64)
        for v0, t, items in r.chunks(8*(4*K*F + K), H*W):
            n = len(t)
            s, c = r.eng.trace_otf_many(t.reshape(n*W, S), r.dev, items, centers[items[:, 1]//W],
                                        z, nu, clip=True, rot0=r.rot0, exact=exact)
            sums[v0:v0 + n] = s.reshape(n, H, W, K, 2, F)
            count[v0:v0 + n] = c.reshape(n, H, W, K)
    out = mtf_tolerance_result(sums, count, sw, targets)
    out.update(freq=nu, z=z)
    return r.result(out)


# ---- the rms wavefront ------------------------------------------------------
def wavefront_specs(base, tables, chief, Ri, origin0, image):
    """The rtx_opd records (OPD_DTYPE, (n,)) of opd()'s reference sphere for
    n variants of one wavelength, each centred on its own chief ray.

    `base` the nominal lens's spec (lazy.opd_spec): its radius, launch ray
    and n0 are kept.  `tables` (n, S) the variants' full tables (row S-1 the
    image), `chief` (n, 2) each variant's chief-ray image point x, y (its z
    is the sag of `image`, the nominal image record: the image surface's
    shape is not perturbed), `Ri` the image surface's rot_normal and
    `origin0` the object's offset.  Per variant, as opd_spec makes them from
    a System with the same change: n_after = record S-2's n, M = rot(record
    S-2) @ Ri.T (a tilt of the last lens surface turns it), and d =
    (origins[after] - origins[image]) @ Ri.T - Y with the origins the
    cumulative offsets."""
    from .engine import OPD_DTYPE, _opd_record
    from .optimize import _image_sag
    tables = np.asarray(tables, SURFACE_DTYPE)
    n, S = tables.shape
    rec = np.repeat(_opd_record(base), n)
    rec["n_after"] = tables[:, S - 2]["n"]
    Ri = np.asarray(Ri, np.float64)
    rec["M"] = (tables[:, S - 2]["rot"].reshape(n, 3, 3) @ Ri.T).reshape(n, 9)
    off = np.concatenate([np.broadcast_to(np.asarray(origin0, np.float64), (n, 1, 3)),
                          tables["offset"]], axis=1)
    origins = np.cumsum(off, axis=1)                          # System.origins
    chief = np.asarray(chief, np.float64).reshape(n, 2)
    x, y = chief[:, 0], chief[:, 1]
    Y = np.stack([x, y, _image_sag(image, x, y)], -1)
    rec["d"] = (origins[:, S - 1] - origins[:, S]) @ Ri.T - Y
    return rec.astype(OPD_DTYPE)


def _tilt_fit(s):
    """(SSR, Caa, n) of the least-squares fit of 1, x, y to a from the 10
    sums s (..., 10) (rtx_trace_opd_many's order), formed from the centred
    second moments in long double; a rank-deficient pupil (all points on
    one line or one point) takes the minimum-norm fit.  SSR is clamped to
    >= 0"""
    s = np.asarray(s, np.longdouble)
    n, sa, saa, sx, sy, sxx, sxy, syy, sax, say = np.moveaxis(s, -1, 0)
    with np.errstate(all="ignore"):
        ma, mx, my = sa/n, sx/n, sy/n
        Caa = saa - sa*ma
        Cxx, Cxy, Cyy = sxx - sx*mx, sxy - sx*my, syy - sy*my
        Cax, Cay = sax - sx*ma, say - sy*ma
        det = Cxx*Cyy - Cxy*Cxy
        full = det > 1e-12*Cxx*Cyy
        fit2 = (Cyy*Cax*Cax - 2*Cxy*Cax*Cay + Cxx*Cay*Cay)/det
        lam = Cxx + Cyy                                       # rank 1: C = lam e e^T
        fit1 = np.where(lam > 0, (Cxx*Cax*Cax + 2*Cxy*Cax*Cay + Cyy*Cay*Cay)/(lam*lam), 0)
        ssr = Caa - np.where(full, fit2, fit1)
        ssr = np.where(ssr < 0, 0, ssr)
    return ssr, Caa, n


def _wfe_targets(targets, H):
    """`targets` broadcast to (H,), ValueError when it does not"""
    try:
        t = np.broadcast_to(np.asarray(targets, np.float64), (H,))
    except ValueError:
        raise ValueError("targets of shape %s does not broadcast to (heights,) = (%d,)"
                         % (np.shape(targets), H)) from None
    return t


def wavefront_tolerance_result(sums, wl, N, weights, chief=None, targets=None):
    """tolerance_wavefront's result from the sums (V, H, W, 10), the
    wavelengths `wl` (W,) in lens units, the bundles' ray counts N (H, W),
    the spectral `weights` (W,), `chief` (V, H, W) bool (None: all true) and
    `targets` (broadcast to (H,), waves rms tilt removed).  An item whose
    chief ray is lost has NaN for every value; rms and rms_tilt are NaN
    where no ray entered"""
    sums = np.array(sums, np.float64)
    V, H, W, _ = sums.shape
    chief = np.ones((V, H, W), bool) if chief is None else np.asarray(chief, bool)
    sums[~chief] = np.nan
    wl = np.asarray(wl, np.float64).reshape(W)
    n = sums[..., 0]
    with np.errstate(all="ignore"):
        dbar = sums[..., 1]/n                                  # gauss_newton_wavefront's rms
        rms = np.sqrt(np.maximum((sums[..., 2]/n - dbar*dbar)/(wl*wl), 0.))
        rms = np.where(np.isnan(dbar), np.nan, rms)
        ssr, _, nl = _tilt_fit(sums)
        # the fit never raises the rms; rounding may, by an ulp, where the tilt is 0
        rms_tilt = np.minimum((np.sqrt(ssr/nl)/wl).astype(np.float64), rms)
        strehl = np.exp(-(2*np.pi*rms_tilt)**2)
        transmitted = n/np.asarray(N, np.float64).reshape(H, W)
        w = np.asarray(weights, np.float64).reshape(W)
        poly_rms = np.sqrt((rms*rms*w).sum(-1)/w.sum())
        poly_rms_tilt = np.sqrt((rms_tilt*rms_tilt*w).sum(-1)/w.sum())
    out = dict(rms=rms, rms_tilt=rms_tilt, strehl=strehl, transmitted=transmitted,
               chief=chief, poly_rms=poly_rms, poly_rms_tilt=poly_rms_tilt, sums=sums)
    if targets is not None:
        t = _wfe_targets(targets, H)
        with np.errstate(invalid="ignore"):
            out["passed"] = (poly_rms_tilt <= t).all(-1)
        out["yield"] = float(out["passed"].mean())
    return out


class _WavefrontRef:
    """The chief-ray reference of the rms wavefront, shared by
    tolerance_wavefront and tolerance_zernike: each (height, wavelength)
    bundle's nominal opd() spec (`base`), the image surface's rot_normal
    `Ri` and the object's offset `origin0`; `chief` makes the per-chunk
    launches that refer every variant's rays to its own chief ray"""

    def __init__(self, system, nominal, wavelengths, chiefs):
        from .lazy import opd_spec
        W, S = len(wavelengths), nominal.shape[1]
        after, image = S - 1, S                                # System indices
        ei = system[image]
        self.Ri = np.asarray(ei.rot_normal, float) if getattr(ei, "rotated", False) else np.eye(3)
        self.origin0 = np.asarray(system[0].offset, np.float64)
        self.base = [opd_spec(system, system.track, system.origins, after, image,
                              system.refractive_index(wavelengths[b % W], 0),
                              float(nominal[b % W, S - 2]["n"]), np.reshape(y0, 3),
                              np.reshape(u0, 3), np.zeros(3))
                     for b, (y0, u0) in enumerate(chiefs)]
        self.nominal, self.chiefs, self.W = nominal, chiefs, W
        self.cdev = []

    def upload(self, eng):
        """the chief rays as 1-ray device bundles (freed by `free`)"""
        for y0, u0 in self.chiefs:
            self.cdev.append((eng.to_device(np.reshape(y0, (1, 3))),
                              eng.to_device(np.reshape(u0, (1, 3))), None))
        return self.cdev

    def free(self):
        for y, u, _ in self.cdev:
            y.free(), u.free()
        self.cdev = []

    def chief(self, eng, t, rot0, exact):
        """For the variants' full tables t (n, W, S): (march (n*W, S-1),
        items (n*nb, 2) variant-major, specs (n*nb,), a0 (n*nb,), centres
        (n*nb, 2), ok (n, nb)) -- the march tables and the per-item
        arguments of rtx_trace_opd_many or rtx_trace_zernike_many whose
        residuals are opd()'s chief-referenced t and py; ok is false where
        the chief ray is lost (a0 and the centre are 0 there)"""
        from .engine import WFE_NSUMS
        n, W, S = t.shape
        nb = len(self.chiefs)
        nominal, base, Ri, origin0, cdev = self.nominal, self.base, self.Ri, self.origin0, self.cdev
        v, b = (a.reshape(-1) for a in np.meshgrid(np.arange(n), np.arange(nb), indexing="ij"))
        items = np.stack([v*W + b % W, b], -1)
        # 1. each variant's chief-ray image point
        m = eng.trace_reduce_many(t.reshape(n*W, S), cdev, items, clip=True, rot0=rot0,
                                  exact=exact).reshape(n, nb, 20)
        ok = m[..., 4] == 1
        xy = np.where(ok[..., None], m[..., 1:3], 0.)
        # 2. its reference sphere
        specs = np.empty((n, nb), wavefront_specs(base[0], t[:1, 0], xy[:1, 0], Ri, origin0,
                                                  nominal[0, S - 1]).dtype)
        for bi in range(nb):
            w = bi % W
            specs[:, bi] = wavefront_specs(base[bi], t[:, w], xy[:, bi], Ri, origin0,
                                           nominal[w, S - 1])
        specs = specs.reshape(-1)
        march = t[:, :, :-1].reshape(n*W, S - 1)
        # 3. the chief ray's path and sphere point, exactly (single-term sums)
        c = eng.trace_opd_many(march, cdev, items, specs, clip=True, rot0=rot0,
                               exact=exact).reshape(n, nb, WFE_NSUMS)
        ok &= c[..., 0] == 1
        a0 = np.where(ok, c[..., 1], 0.).reshape(-1)
        cen = np.where(ok[..., None], c[..., 3:5], 0.).reshape(-1, 2)
        return march, items, specs, a0, cen, ok


def tolerance_wavefront(system, params, deltas, heights=(0., .707, 1.), wavelengths=None,
                        nrays=1000, distribution="hexapolar", compensate=None,
                        spectral_weights=None, targets=None, engine=None, exact=False, chunk=None):
    """The rms wavefront error of every perturbed lens at every field height
    and wavelength, on the device: the wavefront counterpart of
    ``tolerance`` and ``tolerance_mtf``.

    `params` [(j, kind)] and `deltas` (V, P) are ``perturbed_tables``'; a
    shape or tilt of the image surface is refused (it changes only the
    reference sphere), its distance (a defocus) is not.  Each (height,
    wavelength) bundle is aimed once for the NOMINAL lens and marched through
    all V variants with clipping (no re-aiming).  Each variant has its own
    reference sphere: opd()'s default radius of the nominal lens, centred on
    the variant's chief-ray image point and turned by its last lens
    surface's tilt.  Per chunk of variants there are three launches: the
    chief rays to the image (rtx_trace_reduce_many), the chief rays' path
    and sphere point (rtx_trace_opd_many), then every ray's residuals about
    them, opd()'s chief-referenced t and py, reduced to the sums of a fit of
    piston and tilt (rtx_trace_opd_many).  ``compensate="focus"`` refocuses
    each variant first, as ``tolerance`` does.  `targets` (broadcast to (H,))
    are the largest accepted polychromatic rms_tilt in waves.  `chunk`:
    variants per launch (default: as many as fit in 1 GiB of tables and
    tile rows); the results do not depend on it.  FP64 only.

    Returns a dict: rms (V, H, W) the piston-removed rms in waves (lambda =
    l/system.scale), rms_tilt (V, H, W) the residual rms after the
    least-squares fit of 1, x, y (tilt removed), strehl = exp(-(2 pi
    rms_tilt)^2) (Marechal), transmitted (V, H, W) the fraction of the rays
    that enter, chief (V, H, W) true where the variant's chief ray reaches
    the image (elsewhere every value is NaN), poly_rms and poly_rms_tilt
    (V, H) the `spectral_weights` mean of rms^2 over the wavelengths,
    square-rooted, sums (V, H, W, 10) rtx_trace_opd_many's, focus (V,) when
    compensated, heights, wavelengths, params, deltas; with `targets` also
    passed (V,) (every height within its target, NaN failing) and yield,
    the fraction of variants that pass.  Every argument is checked before
    any device work."""
    from .engine import WFE_NSUMS
    from .mtf import _spectral
    heights, wavelengths = check_fields(system, heights, wavelengths, compensate, chunk)
    H, W = len(heights), len(wavelengths)
    sw = _spectral(spectral_weights, W)
    if targets is not None:
        targets = _wfe_targets(targets, H)
    with VariantMarch(system, params, deltas, heights, wavelengths, nrays, distribution,
                      compensate, chunk, engine, exact, wavefront=True) as r:
        sums = np.empty((r.V, H, W, WFE_NSUMS))
        chief = np.empty((r.V, H, W), bool)
        for v0, t, _ in r.chunks(160, 3*H*W):
            n = len(t)
            march, items, specs, a0, cen, ok = r.ref.chief(r.eng, t, r.rot0, exact)
            # 4. every ray's residuals about the chief ray's
            s = r.eng.trace_opd_many(march, r.dev, items, specs, a0, cen, clip=True, rot0=r.rot0,
                                     exact=exact)
            sums[v0:v0 + n] = s.reshape(n, H, W, WFE_NSUMS)
            chief[v0:v0 + n] = ok.reshape(n, H, W)
    wl = np.array([l/system.scale for l in wavelengths])
    return r.result(wavefront_tolerance_result(sums, wl, r.counts, sw, chief, targets))
