"""Lens optimisation on the device: exact derivatives of the spot and a
damped-least-squares (Levenberg-Marquardt) optimiser built on them.

``spot_jacobian`` marches every (height, wavelength) bundle of the lens once
with forward-mode tangents (rtx_trace_jacobian) and reduces the image points
and their derivatives to the Gauss-Newton sums on the device
(rtx_jacobian_sums).  With the residuals of a bundle r_k = (q_k - qbar)/sqrt(n)
(q_k the image point of ray k, qbar the centroid of the n rays that reach the
image with finite derivatives), rms^2 = sum |r_k|^2 and

    J^T J = (K - G G^T/n)/n,   J^T r = (H - dbar . G)/n,   d rms^2/dp = 2 J^T r

from the device sums K, G, H, dbar (include/rtx.h).  The derivatives are
those of the march on fixed launch rays: nothing flows through ray aiming,
which ``optimize_spot`` redoes at every iteration instead.

``optimize_spot`` minimises sum_b w_b rms_b^2 over curvatures, conics,
distances and aspheric coefficients (the image surface's distance is the
focus).  Each iteration re-aims the lens, takes the Jacobian, solves
(J^T J + lambda diag J^T J) delta = -J^T r for a few lambda, scores every
trial step in one rtx_trace_reduce_many launch on the same bundles and takes
the best one if it lowers the merit.
"""
import copy

import numpy as np

from .engine import Engine, default_engine, jacobian_sums_unpack
from .surface_table import RTX_MAX_ASPH, pack_system
from .tolerance import _chief, launch_bundles, perturbed_tables, record_tangents

OPT_KINDS = ("curvature", "conic", "distance") + tuple("asph%d" % i for i in range(RTX_MAX_ASPH))


def _nominal(system, wavelengths):
    packs = [pack_system(system, l, 1, None, n0=system.refractive_index(l, 0)) for l in wavelengths]
    return np.stack([t for t, _, _ in packs]), packs[0][2]


class _Bundles:
    """The launch rays of every (height, wavelength) of `system`, aimed once
    (height-major), and each bundle's guess centre: its chief ray at the
    image.  Frees its device arrays on close()."""

    def __init__(self, system, heights, wavelengths, nrays, distribution, eng, exact):
        self.nominal, self.rot0 = _nominal(system, wavelengths)
        self.W = len(wavelengths)
        self.rays, chiefs = launch_bundles(system, heights, wavelengths, nrays, distribution, eng)
        try:
            self.centers = np.array([_chief(eng, self.nominal[b % self.W], self.rot0, y, u, exact)
                                     for b, (y, u) in enumerate(chiefs)])
        except Exception:
            self.close()
            raise

    def close(self):
        for y, u in self.rays:
            y.free(), u.free()
        self.rays = []


def _sums(eng, B, moves, clip, chunk, exact):
    """(bundles, W) device sums of every bundle, its ray chunks added on the
    host in chunk order"""
    P = len(moves)
    out = np.zeros((len(B.rays), 5 + 3*P + P*(P + 1)//2))
    for b, (y0, u0) in enumerate(B.rays):
        w = b % B.W
        mv = [[(row, rec[w]) for row, rec in m] for m in moves]
        N = y0.shape[0]
        for r0 in range(0, N, chunk):
            r1 = min(N, r0 + chunk)
            q, J = eng.trace_jacobian(B.nominal[w], y0.rows(r0, r1), u0.rows(r0, r1), mv,
                                      clip=clip, rot0=B.rot0, exact=exact)
            try:
                out[b] += eng.jacobian_sums(q, J, B.centers[b, :2])["out"]
            finally:
                q.free(), J.free()
    return out


def gauss_newton(out, P):
    """rms^2 about the centroid, J^T J, J^T r and the gradient of rms^2 of
    one bundle from its rtx_jacobian_sums row `out` (the module docstring's
    formulas)"""
    s = jacobian_sums_unpack(out, P)
    n, G = s["n"], s["G"]
    with np.errstate(all="ignore"):
        dbar = s["sum_d"]/n
        rms2 = s["sum_d2"]/n - dbar @ dbar
        JtJ = (s["K"] - G @ G.T/n)/n
        Jtr = (s["H"] - G @ dbar)/n
    return rms2, JtJ, Jtr, 2*Jtr


def spot_jacobian(system, params, heights=(0., .707, 1.), wavelengths=None, nrays=1000,
                  distribution="hexapolar", clip=False, chunk=1 << 20, engine=None, exact=False):
    """Exact derivatives of the spot of every (height, wavelength) bundle
    with respect to the parameters `params` [(j, kind)] (tolerance's
    vocabulary), on the device.

    The launch rays of each bundle are generated in HBM for the nominal lens
    (tolerance.launch_bundles) and marched in chunks of `chunk` rays; the
    sums are about each bundle's chief ray and added on the host in chunk
    order.  Returns a dict: rms (H, W) about each bundle's own centroid,
    grad (H, W, P) of rms^2, JtJ (H, W, P, P), Jtr (H, W, P), n (H, W) the
    rays that enter, bad (H, W) the rays with a finite image point and a
    non-finite derivative, sums (H, W, .) the device rows, and heights,
    wavelengths, params."""
    eng = engine or default_engine()
    wavelengths = list(system.wavelengths if wavelengths is None else wavelengths)
    heights = list(heights)
    params = list(params)
    chunk = int(chunk)
    if chunk < 1:
        raise ValueError("chunk must be >= 1")
    moves = record_tangents(_nominal(system, wavelengths)[0], params)  # refusals first
    B = _Bundles(system, heights, wavelengths, nrays, distribution, eng, exact)
    try:
        out = _sums(eng, B, moves, clip, chunk, exact)
    finally:
        B.close()
    return _result(out, len(heights), len(wavelengths), len(params),
                   dict(heights=np.asarray(heights, np.float64),
                        wavelengths=np.asarray(wavelengths, np.float64), params=params))


def _result(out, H, W, P, extra):
    gn = [gauss_newton(o, P) for o in out]
    res = dict(rms=np.sqrt(np.maximum([g[0] for g in gn], 0.)).reshape(H, W),
               JtJ=np.array([g[1] for g in gn]).reshape(H, W, P, P),
               Jtr=np.array([g[2] for g in gn]).reshape(H, W, P),
               grad=np.array([g[3] for g in gn]).reshape(H, W, P),
               n=out[:, 0].reshape(H, W), bad=out[:, -1].reshape(H, W),
               sums=out.reshape(H, W, -1))
    res.update(extra)
    return res


def lm_step(JtJ, Jtr, lam):
    """the Levenberg-Marquardt step with Marquardt's scaling:
    (JtJ + lam D) delta = -Jtr, D = diag JtJ.  A parameter that does not
    move the spot has a zero row and column; its D entry is floored at
    1e-12 of the largest (1 when all are 0), so that the system stays
    solvable and that parameter's step is 0."""
    A = np.array(JtJ, np.float64)
    d = np.diag(A).copy()
    top = d.max() if d.size and d.max() > 0 else 1.
    A[np.diag_indices_from(A)] += lam*np.maximum(d, 1e-12*top)
    return np.linalg.solve(A, -np.asarray(Jtr, np.float64))


def apply_deltas(system, params, delta):
    """`system` with the parameter changes `delta` made (in place), as
    perturbed_tables makes them on the records, then system.update()"""
    for (j, kind), d in zip(params, delta):
        e = system[j]
        d = float(d)
        if kind == "curvature":
            e.curvature = e.curvature + d
        elif kind == "conic":
            e.conic = e.conic + d
        elif kind == "distance":
            e.distance = e.distance + d
        else:
            i = int(kind[4:])
            a = list(e.aspherics) if e.aspherics is not None else []
            a += [0.]*(i + 1 - len(a))
            a[i] = a[i] + d
            e.aspherics = a
    system.update()
    return system


def _merits(eng, B, params, deltas, weights, clip, exact):
    """sum_b w_b rms_b^2 of each row of `deltas` (V, P) on the fixed bundles
    B, in one rtx_trace_reduce_many launch"""
    t = perturbed_tables(B.nominal, params, deltas)
    V, W, S = t.shape
    nb = len(B.rays)
    v, b = np.meshgrid(np.arange(V), np.arange(nb), indexing="ij")
    v, b = v.reshape(-1), b.reshape(-1)
    items = np.stack([v*W + b % W, b], -1)
    m = eng.trace_reduce_many(t.reshape(V*W, S), [(y, u, None) for y, u in B.rays], items,
                              B.centers[b], clip=clip, rot0=B.rot0, exact=exact)
    rms = Engine.rms_finite_from_moments(m).reshape(V, nb)
    return (weights.reshape(-1)*rms**2).sum(1)


def optimize_spot(system, params, heights=(0., .707, 1.), wavelengths=None, weights=None,
                  iterations=20, damping=1e-3, nrays=1000, distribution="hexapolar", clip=False,
                  lambdas=(.1, 1., 10., 100.), chunk=1 << 20, engine=None, exact=False):
    """Levenberg-Marquardt on the merit sum_b w_b rms_b^2 over the (height,
    wavelength) bundles, rms about each bundle's centroid.

    `params` [(j, kind)] with kind in OPT_KINDS; the image surface's
    ``distance`` is the focus.  `weights` (H, W), default 1.  Each iteration
    re-aims the current lens, takes spot_jacobian's normal equations, tries
    lambda = damping*f for f in `lambdas`, scores the trial steps on the same
    bundles in one launch and applies the best one if it lowers the merit
    (then damping = its lambda; otherwise damping grows 100-fold).  The
    caller's System is not modified.

    Returns a dict: system (the optimised copy), deltas (P,) the cumulative
    change, merit (iterations + 1,) the re-aimed merit before each iteration
    and at the end, lam and step (iterations,) the lambda and step taken (0
    where none was accepted), trial (iterations,) the fixed-bundle merit of
    the accepted step (or of the lens when none was)."""
    params = [(int(j), kind) for j, kind in params]
    for j, kind in params:
        if kind not in OPT_KINDS:
            raise ValueError("cannot optimise %r: the kinds are %s" % (kind, ", ".join(OPT_KINDS[:4])
                                                                        + ", asph<i>"))
    eng = engine or default_engine()
    wavelengths = list(system.wavelengths if wavelengths is None else wavelengths)
    heights = list(heights)
    H, W, P = len(heights), len(wavelengths), len(params)
    weights = np.ones((H, W)) if weights is None else np.broadcast_to(
        np.asarray(weights, np.float64), (H, W))
    system = copy.deepcopy(system)
    record_tangents(_nominal(system, wavelengths)[0], params)  # refusals before any device work
    total = np.zeros(P)
    hist = dict(merit=[], lam=[], step=[], trial=[])
    lam = float(damping)
    for it in range(iterations + 1):
        B = _Bundles(system, heights, wavelengths, nrays, distribution, eng, exact)
        try:
            if it == iterations:               # the final lens, re-aimed
                hist["merit"].append(float(_merits(eng, B, params, np.zeros((1, P)), weights,
                                                   clip, exact)[0]))
                break
            moves = record_tangents(B.nominal, params)
            res = _result(_sums(eng, B, moves, clip, int(chunk), exact), H, W, P, {})
            w = weights[..., None, None]
            JtJ = (w*res["JtJ"]).sum((0, 1))
            Jtr = (w[..., 0]*res["Jtr"]).sum((0, 1))
            lams = [lam*f for f in lambdas]
            steps = np.array([lm_step(JtJ, Jtr, x) for x in lams])
            merit = _merits(eng, B, params, np.vstack([np.zeros(P), steps]), weights, clip, exact)
        finally:
            B.close()
        hist["merit"].append(float(merit[0]))
        k = int(np.nanargmin(merit[1:])) if np.isfinite(merit[1:]).any() else -1
        if k >= 0 and merit[1 + k] < merit[0]:
            lam = lams[k]
            apply_deltas(system, params, steps[k])
            total += steps[k]
            hist["lam"].append(lam)
            hist["step"].append(steps[k])
            hist["trial"].append(float(merit[1 + k]))
        else:
            lam *= 100
            hist["lam"].append(0.)
            hist["step"].append(np.zeros(P))
            hist["trial"].append(float(merit[0]))
    return dict(system=system, deltas=total, merit=np.array(hist["merit"]),
                lam=np.array(hist["lam"]), step=np.array(hist["step"]).reshape(-1, P),
                trial=np.array(hist["trial"]), params=params)
