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

``wavefront_jacobian`` and ``optimize_wavefront`` do the same for the rms
wavefront error, piston removed and referenced to the chief ray: the
per-ray path A of ``opd()`` (rtx_trace_opd_jacobian, to surface after =
len(system) - 2, the default reference sphere) in waves W_k = -(A_k -
A_ref)/lambda.  With d_k = A_k - a0 (a0 the chief ray's A) and the
one-component sums of rtx_wavefront_sums,

    rms^2 = (sum d^2/n - dbar^2)/lambda^2,   J^T J = (K - G G^T/n)/(n lambda^2),
    J^T r = (H - dbar G)/(n lambda^2)

The sphere's radius and the frame change to the image surface are held at
their values for the current lens; its centre, the chief ray's image point,
moves with the parameters.

``mtf_jacobian`` and ``optimize_mtf`` do the same for the geometric MTF at
chosen frequencies: with d_k = q_k - c along one axis, S(nu) = sum_k
exp(-2 pi i nu d_k) and dS/dp = sum_k -2 pi i nu dq_k/dp exp(-2 pi i nu d_k)
(rtx_otf_jacobian_sums, c held fixed).  Moving the centre c multiplies S by a
phase, so MTF = |S|/n and d MTF/dp = Re(conj(S) dS/dp)/(|S| n) need no
derivative of c, and neither does the polychromatic MTF of wavelengths that
share one centre.
"""
import copy

import numpy as np

from .engine import (Engine, default_engine, jacobian_sums_unpack, otf_jacobian_sums_unpack,
                     wavefront_sums_unpack)
from .lazy import opd_spec
from .mtf import _check_freqs, _spectral, poly_otf
from .surface_table import RTX_MAX_ASPH, SURFACE_DTYPE
from .tolerance import _centers, _nominal, launch_bundles, perturbed_tables, record_tangents

OPT_KINDS = ("curvature", "conic", "distance") + tuple("asph%d" % i for i in range(RTX_MAX_ASPH))


class _Bundles:
    """The launch rays of every (height, wavelength) of `system`, aimed once
    (height-major), and each bundle's guess centre: its chief ray at the
    image.  Frees its device arrays on close()."""

    def __init__(self, system, heights, wavelengths, nrays, distribution, eng, exact):
        self.nominal, self.rot0 = _nominal(system, wavelengths)
        self.W = len(wavelengths)
        self.wavelengths = list(wavelengths)
        self.rays, chiefs = launch_bundles(system, heights, wavelengths, nrays, distribution, eng)
        self.chiefs = chiefs
        try:
            self.centers = _centers(eng, self.nominal, self.rot0, chiefs, exact)
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


def _check_kinds(params):
    params = [(int(j), kind) for j, kind in params]
    for j, kind in params:
        if kind not in OPT_KINDS:
            raise ValueError("cannot optimise %r: the kinds are %s" % (kind, ", ".join(OPT_KINDS[:4])
                                                                        + ", asph<i>"))
    return params


def _bundle_weights(weights, H, W):
    """the per-bundle weights (H, W) of optimize_spot and optimize_wavefront"""
    return np.ones((H, W)) if weights is None else np.broadcast_to(
        np.asarray(weights, np.float64), (H, W))


def _weighted_normal(res, weights):
    """sum_b w_b of the per-bundle normal equations res["JtJ"] (H, W, P, P)
    and res["Jtr"] (H, W, P)"""
    w = weights[..., None, None]
    return (w*res["JtJ"]).sum((0, 1)), (w[..., 0]*res["Jtr"]).sum((0, 1))


def _lm(system, params, heights, wavelengths, iterations, damping, nrays, distribution,
        lambdas, eng, exact, prepare, normal, merits):
    """The Levenberg-Marquardt loop of optimize_spot, optimize_wavefront and
    optimize_mtf on a copy of `system`.  Per iteration, on the re-aimed
    bundles B: state = prepare(system, B, final) (freed by state.close()
    when it has one; `final`: only the merit of the last, re-aimed lens is
    wanted), normal(B, state) the weighted normal equations (JtJ (P, P),
    Jtr (P,)), merits(B, state, deltas) the weighted merit of each row of
    deltas on the fixed bundles."""
    P = len(params)
    system = copy.deepcopy(system)
    total = np.zeros(P)
    hist = dict(merit=[], lam=[], step=[], trial=[])
    lam = float(damping)
    for it in range(iterations + 1):
        B = _Bundles(system, heights, wavelengths, nrays, distribution, eng, exact)
        state = None
        try:
            state = prepare(system, B, it == iterations)
            if it == iterations:               # the final lens, re-aimed
                hist["merit"].append(float(merits(B, state, np.zeros((1, P)))[0]))
                break
            JtJ, Jtr = normal(B, state)
            lams = [lam*f for f in lambdas]
            steps = np.array([lm_step(JtJ, Jtr, x) for x in lams])
            merit = merits(B, state, np.vstack([np.zeros(P), steps]))
        finally:
            if state is not None and hasattr(state, "close"):
                state.close()
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
    params = _check_kinds(params)
    eng = engine or default_engine()
    wavelengths = list(system.wavelengths if wavelengths is None else wavelengths)
    heights = list(heights)
    H, W, P = len(heights), len(wavelengths), len(params)
    weights = _bundle_weights(weights, H, W)
    record_tangents(_nominal(system, wavelengths)[0], params)  # refusals before any device work

    def normal(B, state):
        moves = record_tangents(B.nominal, params)
        return _weighted_normal(_result(_sums(eng, B, moves, clip, int(chunk), exact), H, W, P, {}),
                                weights)

    return _lm(system, params, heights, wavelengths, iterations, damping, nrays, distribution,
               lambdas, eng, exact, lambda system, B, final: None, normal,
               lambda B, state, deltas: _merits(eng, B, params, deltas, weights, clip, exact))


# ---- the rms wavefront error ---------------------------------------------
def _wavefront_checked(system, wavelengths, params):
    """record_tangents' refusals, then the ones of the wavefront: shape
    parameters of the image surface (they change only the reference) and
    tilts of the last two surfaces (they change the frame change M, which is
    held fixed).  ValueError before any device work."""
    L = len(system)
    record_tangents(_nominal(system, wavelengths)[0], params)
    for j, kind in params:
        if j == L - 1 and kind not in ("distance",):
            raise ValueError("%s of the image surface %d changes only the reference sphere"
                             % (kind, j))
        if j >= L - 2 and kind in ("tilt_x", "tilt_y"):
            raise ValueError("%s of surface %d changes the frame change to the image, "
                             "which the wavefront derivative holds fixed" % (kind, j))


def _image_slope(rec, x, y):
    """e of the normal (x e, y e, 1) of record `rec` at (x, y): the sag's
    gradient is -(x e, y e)"""
    r2 = x*x + y*y
    c, kc2 = float(rec["c"]), float(rec["kc2"])
    e = -c/np.sqrt(1 - kc2*r2)
    for j in range(max(int(rec["n_asph"]), 0)):
        e -= float(rec["dasph"][j])*r2**j
    return e


def _image_sag(rec, x, y):
    """z of record `rec`'s surface at (x, y)"""
    r2 = x*x + y*y
    c, kc2 = float(rec["c"]), float(rec["kc2"])
    z = c*r2/(1 + np.sqrt(1 - kc2*r2))
    for j in range(max(int(rec["n_asph"]), 0)):
        z += float(rec["asph"][j])*r2**(j + 1)
    return z


class _Wavefront:
    """Per bundle of B: the rtx_opd record of opd()'s default sphere (or of
    `radius`), its derivative dopd (P, 4), the piston guess a0 (the chief
    ray's A), the wavelength in lens units and the chief rays on the device.
    `moves` the full-table moves of record_tangents(B.nominal) (None: no
    derivatives)."""

    def __init__(self, eng, system, B, heights, moves, radius, clip, exact):
        L = len(system)
        self.after, self.image = L - 2, L - 1
        ei = system[self.image]
        self.Ri = np.asarray(ei.rot_normal, float) if getattr(ei, "rotated", False) else np.eye(3)
        S = B.nominal.shape[1]
        self.chief = []
        self.specs, self.dopd, self.a0, self.wl, self.yimg = [], [], [], [], []
        try:
            for b, (y0, u0) in enumerate(B.chiefs):
                self.chief.append((eng.to_device(np.reshape(y0, (1, 3))),
                                   eng.to_device(np.reshape(u0, (1, 3)))))
            for b, (y0, u0) in enumerate(B.chiefs):
                w = b % B.W
                table = B.nominal[w]
                l = B.wavelengths[w]
                Y = eng.trace(table, np.reshape(y0, (1, 3)), np.reshape(u0, (1, 3)), clip=True,
                              rot0=B.rot0, keep_last=True, exact=exact, want=("y",))[0][0, 0]
                if not np.all(np.isfinite(Y)):
                    raise ValueError("the chief ray of height %g at wavelength %g does not reach "
                                     "the image" % (heights[b//B.W], l))
                spec = opd_spec(system, system.track, system.origins, self.after, self.image,
                                system.refractive_index(l, 0), float(table[S - 2]["n"]),
                                np.reshape(y0, 3), np.reshape(u0, 3), Y, radius)
                self.specs.append(spec)
                self.yimg.append(Y)
                self.wl.append(l/system.scale)
                if moves is not None:
                    self.dopd.append(self._dopd(eng, system, B, b, table, moves, Y, exact))
                A, Pp = eng.empty((1,)), eng.empty((1, 3))
                try:
                    cy, cu = self.chief[b]
                    eng.trace_opd(table[:-1], cy, cu, spec, A, Pp, clip=clip, rot0=B.rot0,
                                  exact=exact)
                    self.a0.append(float(A.download()[0]))
                finally:
                    A.free(), Pp.free()
        except Exception:
            self.close()
            raise

    def _dopd(self, eng, system, B, b, table, moves, Y, exact):
        """d(spec d) and d(n_after) per parameter: the image surface's offset
        and the chief ray's image point move the sphere's centre"""
        S = len(table)
        w = b % B.W
        mv = [[(row, rec[w]) for row, rec in m] for m in moves]
        cy, cu = self.chief[b]
        q, J = eng.trace_jacobian(table, cy, cu, mv, clip=True, rot0=B.rot0, exact=exact)
        try:
            dq = J.download()[:, :, 0]
        finally:
            q.free(), J.free()
        J = dq
        Ri = self.Ri
        e = _image_slope(table[S - 1], Y[0], Y[1])
        out = np.zeros((len(mv), 4))
        for p, m in enumerate(mv):
            dy = np.array([J[p, 0], J[p, 1], -e*(Y[0]*J[p, 0] + Y[1]*J[p, 1])])
            doff = sum((np.asarray(rec["offset"], float) for row, rec in m if row == S - 1),
                       np.zeros(3))
            out[p, :3] = -doff @ Ri.T - dy
            out[p, 3] = sum(float(rec["n"]) for row, rec in m if row == S - 2)
        return out

    def close(self):
        for y, u in self.chief:
            y.free(), u.free()
        self.chief = []


def _opd_moves(moves, w, S):
    """the moves of wavelength w on the OPD march's rows 0..S-2; a
    parameter that moves only the image row gets a zero move on row S-2"""
    out = []
    for m in moves:
        mv = [(row, rec[w]) for row, rec in m if row < S - 1]
        out.append(mv or [(S - 2, np.zeros((), SURFACE_DTYPE))])
    return out


def _wavefront_sums(eng, B, st, moves, clip, chunk, exact):
    """(bundles, W) device wavefront sums of every bundle, its ray chunks
    added on the host in chunk order"""
    P = len(moves)
    S = B.nominal.shape[1]
    out = np.zeros((len(B.rays), 4 + 2*P + P*(P + 1)//2))
    for b, (y0, u0) in enumerate(B.rays):
        w = b % B.W
        mv = _opd_moves(moves, w, S)
        N = y0.shape[0]
        for r0 in range(0, N, chunk):
            r1 = min(N, r0 + chunk)
            A, dA = eng.trace_opd_jacobian(B.nominal[w, :-1], y0.rows(r0, r1), u0.rows(r0, r1),
                                           st.specs[b], mv, st.dopd[b], clip=clip, rot0=B.rot0,
                                           exact=exact)
            try:
                out[b] += eng.wavefront_sums(A, dA, st.a0[b])["out"]
            finally:
                A.free(), dA.free()
    return out


def gauss_newton_wavefront(out, P, wl):
    """rms^2 in waves^2 about the mean, J^T J, J^T r and the gradient of
    rms^2 of one bundle from its rtx_wavefront_sums row `out` and the
    wavelength wl in lens units (the module docstring's formulas)"""
    s = wavefront_sums_unpack(out, P)
    n, G = s["n"], s["G"]
    k = 1/(wl*wl)
    with np.errstate(all="ignore"):
        dbar = s["sum_d"]/n
        rms2 = (s["sum_d2"]/n - dbar*dbar)*k
        JtJ = (s["K"] - np.outer(G, G)/n)/n*k
        Jtr = (s["H"] - dbar*G)/n*k
    return rms2, JtJ, Jtr, 2*Jtr


def _wavefront_result(out, wl, H, W, P, extra):
    gn = [gauss_newton_wavefront(o, P, x) for o, x in zip(out, wl)]
    res = dict(rms=np.sqrt(np.maximum([g[0] for g in gn], 0.)).reshape(H, W),
               JtJ=np.array([g[1] for g in gn]).reshape(H, W, P, P),
               Jtr=np.array([g[2] for g in gn]).reshape(H, W, P),
               grad=np.array([g[3] for g in gn]).reshape(H, W, P),
               n=out[:, 0].reshape(H, W), bad=out[:, -1].reshape(H, W),
               sums=out.reshape(H, W, -1))
    res.update(extra)
    return res


def wavefront_jacobian(system, params, heights=(0., .707, 1.), wavelengths=None, nrays=1000,
                       distribution="hexapolar", clip=False, radius=None, chunk=1 << 20,
                       engine=None, exact=False):
    """Exact derivatives of the rms wavefront error of every (height,
    wavelength) bundle with respect to the parameters `params` [(j, kind)]
    (tolerance's vocabulary), on the device: the piston-removed rms of opd()'s
    per-ray wavefront, chief-ray referenced, over the rays whose path and
    derivatives are finite.

    The sphere is opd()'s default (or of `radius`), centred on the chief
    ray's image point; its radius and the frame change to the image are held
    fixed, its centre follows the parameters.  Shape parameters of the image
    surface and tilts of the last two surfaces are refused (ValueError).  The
    bundles are generated as spot_jacobian's.  Returns a dict: rms (H, W) in
    waves, grad (H, W, P) of rms^2, JtJ (H, W, P, P), Jtr (H, W, P), n, bad,
    sums (H, W, .) the device rows, and heights, wavelengths, params."""
    eng = engine or default_engine()
    wavelengths = list(system.wavelengths if wavelengths is None else wavelengths)
    heights = list(heights)
    params = list(params)
    chunk = int(chunk)
    if chunk < 1:
        raise ValueError("chunk must be >= 1")
    _wavefront_checked(system, wavelengths, params)
    B = _Bundles(system, heights, wavelengths, nrays, distribution, eng, exact)
    st = None
    try:
        moves = record_tangents(B.nominal, params)
        st = _Wavefront(eng, system, B, heights, moves, radius, clip, exact)
        out = _wavefront_sums(eng, B, st, moves, clip, chunk, exact)
    finally:
        if st is not None:
            st.close()
        B.close()
    return _wavefront_result(out, st.wl, len(heights), len(wavelengths), len(params),
                             dict(heights=np.asarray(heights, np.float64),
                                  wavelengths=np.asarray(wavelengths, np.float64),
                                  params=params))


def _wavefront_merits(eng, B, st, params, deltas, weights, clip, exact):
    """sum_b w_b rms_b^2 (waves^2) of each row of `deltas` (V, P) on the
    fixed bundles B: each variant's sphere centred on its chief rays, all
    marched in one rtx_trace_reduce_many launch; then rtx_trace_opd and
    rtx_wavefront_sums (P = 0) per variant and bundle, the radius and a0
    the current lens's"""
    t = perturbed_tables(B.nominal, params, deltas)
    V, W, S = t.shape
    nb = len(B.rays)
    v, b = np.meshgrid(np.arange(V), np.arange(nb), indexing="ij")
    v, b = v.reshape(-1), b.reshape(-1)
    items = np.stack([v*W + b % W, b], -1)
    m = eng.trace_reduce_many(t.reshape(V*W, S), [(y, u, None) for y, u in st.chief], items,
                              clip=True, rot0=B.rot0, exact=exact).reshape(V, nb, 20)
    Nmax = max(y.shape[0] for y, _ in B.rays)
    A, Pp = eng.empty((Nmax,)), eng.empty((Nmax, 3))
    rms2 = np.full((V, nb), np.inf)
    try:
        for vi in range(V):
            for bi, (y0, u0) in enumerate(B.rays):
                w = bi % W
                if m[vi, bi, 4] != 1:                  # the chief ray is lost
                    continue
                spec = dict(st.specs[bi])
                ti = t[vi, w, -1]
                t0 = ei = B.nominal[w, -1]
                x, y = m[vi, bi, 1], m[vi, bi, 2]
                Y0 = st.yimg[bi]
                dy = np.array([x - Y0[0], y - Y0[1],
                               _image_sag(ei, x, y) - _image_sag(ei, Y0[0], Y0[1])])
                doff = np.asarray(ti["offset"], float) - np.asarray(t0["offset"], float)
                spec["d"] = np.asarray(spec["d"], float) - doff @ st.Ri.T - dy
                spec["n_after"] = float(t[vi, w, S - 2]["n"])
                N = y0.shape[0]
                eng.trace_opd(t[vi, w, :-1], y0, u0, spec, A, Pp, N=N, clip=clip, rot0=B.rot0,
                              exact=exact)
                s = eng.wavefront_sums(A, None, st.a0[bi], N=N)
                with np.errstate(all="ignore"):
                    dbar = s["sum_d"]/s["n"]
                    r2 = (s["sum_d2"]/s["n"] - dbar*dbar)/st.wl[bi]**2
                rms2[vi, bi] = r2 if s["n"] > 0 else np.inf
    finally:
        A.free(), Pp.free()
    return (weights.reshape(-1)*rms2).sum(1)


def optimize_wavefront(system, params, heights=(0., .707, 1.), wavelengths=None, weights=None,
                       iterations=20, damping=1e-3, nrays=1000, distribution="hexapolar",
                       clip=False, lambdas=(.1, 1., 10., 100.), chunk=1 << 20, engine=None,
                       exact=False):
    """optimize_spot on the merit sum_b w_b rms_b^2 with rms_b the rms
    wavefront error in waves (wavefront_jacobian's): the same parameters,
    loop and returns.  Each iteration takes the sphere of the re-aimed lens;
    the trial steps are scored on the same bundles with that sphere's radius
    and each variant's own chief-ray centre."""
    params = _check_kinds(params)
    eng = engine or default_engine()
    wavelengths = list(system.wavelengths if wavelengths is None else wavelengths)
    heights = list(heights)
    H, W, P = len(heights), len(wavelengths), len(params)
    weights = _bundle_weights(weights, H, W)
    _wavefront_checked(system, wavelengths, params)

    def prepare(system, B, final):
        moves = None if final else record_tangents(B.nominal, params)
        st = _Wavefront(eng, system, B, heights, moves, None, clip, exact)
        st.moves = moves
        return st

    def normal(B, st):
        out = _wavefront_sums(eng, B, st, st.moves, clip, int(chunk), exact)
        return _weighted_normal(_wavefront_result(out, st.wl, H, W, P, {}), weights)

    return _lm(system, params, heights, wavelengths, iterations, damping, nrays, distribution,
               lambdas, eng, exact, prepare, normal,
               lambda B, st, deltas: _wavefront_merits(eng, B, st, params, deltas, weights, clip,
                                                       exact))


# ---- the geometric MTF at chosen frequencies -------------------------------
def _per_residual(name, x, shape):
    """`x` broadcast to (H, 2, F), ValueError when it does not"""
    try:
        return np.broadcast_to(np.asarray(x, np.float64), shape)
    except ValueError:
        raise ValueError("%s of shape %s does not broadcast to (heights, 2, freqs) = %s"
                         % (name, np.shape(x), shape)) from None


def _otf_sums(eng, B, moves, freqs, clip, chunk, exact):
    """(bundles, W) rtx_otf_jacobian_sums rows of every bundle about its
    height's chief ray at wavelengths[0], its ray chunks added on the host in
    chunk order"""
    P, F = len(moves), len(freqs)
    out = np.zeros((len(B.rays), 2 + 4*F + 4*P*F))
    for b, (y0, u0) in enumerate(B.rays):
        w = b % B.W
        mv = [[(row, rec[w]) for row, rec in m] for m in moves]
        N = y0.shape[0]
        for r0 in range(0, N, chunk):
            r1 = min(N, r0 + chunk)
            q, J = eng.trace_jacobian(B.nominal[w], y0.rows(r0, r1), u0.rows(r0, r1), mv,
                                      clip=clip, rot0=B.rot0, exact=exact)
            try:
                out[b] += eng.otf_jacobian_sums(q, J, freqs, B.centers[b - w, :2])["out"]
            finally:
                q.free(), J.free()
    return out


def _abs_grad(S, dS):
    """|S| and d|S| = Re(conj(S) dS)/|S|: S (..., 2, F), dS (..., P, 2, F)
    complex; the gradient (..., 2, F, P), NaN where |S| = 0"""
    a = np.abs(S)
    with np.errstate(invalid="ignore", divide="ignore"):
        g = (np.conj(S)[..., None, :, :]*dS).real/a[..., None, :, :]
        g = np.where(a[..., None, :, :] > 0, g, np.nan)
    return a, np.moveaxis(g, -3, -1)


def _mtf_result(out, H, W, P, F, sw):
    u = [otf_jacobian_sums_unpack(o, P, F) for o in out]
    n = np.array([x["n"] for x in u]).reshape(H, W)
    S = np.array([x["S"] for x in u]).reshape(H, W, 2, F)
    dS = np.array([x["dS"] for x in u]).reshape(H, W, P, 2, F)
    with np.errstate(invalid="ignore", divide="ignore"):
        otf = S/n[..., None, None]
        dotf = dS/n[..., None, None, None]
    _, grad = _abs_grad(otf, dotf)
    poly = poly_otf(otf[:, :, None], n[:, :, None], sw)[:, 0]
    wk = np.where(n > 0, sw, 0.)
    with np.errstate(invalid="ignore", divide="ignore"):
        dpoly = np.einsum("hw,hwpaf->hpaf", wk, np.where(wk[..., None, None, None] > 0, dotf, 0)) \
            / wk.sum(1)[:, None, None, None]
    poly_mtf, poly_grad = _abs_grad(poly, dpoly)
    return dict(otf=otf, mtf=np.abs(otf), grad=grad, poly=poly, poly_mtf=poly_mtf,
                poly_grad=poly_grad, n=n, bad=out[:, -1].reshape(H, W), sums=out.reshape(H, W, -1))


def mtf_jacobian(system, params, freqs, heights=(0., .707, 1.), wavelengths=None, nrays=1000,
                 distribution="hexapolar", clip=True, spectral_weights=None, chunk=1 << 20,
                 engine=None, exact=False):
    """Exact derivatives of the geometric MTF of every (height, wavelength)
    bundle at the frequencies `freqs` (cycles per length unit) with respect
    to the parameters `params` [(j, kind)] (tolerance's vocabulary), on the
    device.

    The bundles are spot_jacobian's; each is marched with tangents in chunks
    of `chunk` rays (rtx_trace_jacobian) and reduced to the OTF sums S and
    their derivatives dS (rtx_otf_jacobian_sums), the chunks added on the
    host in order.  As in geometric_mtf, every wavelength of a height is
    centred on that height's chief ray at wavelengths[0].  The MTF |S|/n does
    not depend on the centre, so its derivative Re(conj(S) dS)/(|S| n) needs
    none of the centre's.  With clip=True (the default) the MTF is
    geometric_mtf's at defocus 0.

    Returns a dict: freq (F,), otf complex (H, W, 2, F) (axis 0: x, 1: y),
    mtf = |otf|, grad (H, W, 2, F, P) of the MTF, poly (H, 2, F) the
    `spectral_weights` mean of the wavelengths' OTFs (mtf.poly_otf),
    poly_mtf = |poly|, poly_grad (H, 2, F, P), n (H, W) the rays that enter,
    bad (H, W) the rays with a finite image point and a non-finite
    derivative, sums (H, W, .) the device rows, and heights, wavelengths,
    params.  Where |S| = 0 the MTF has no derivative: grad (and poly_grad
    where |poly| = 0) is NaN there."""
    eng = engine or default_engine()
    wavelengths = list(system.wavelengths if wavelengths is None else wavelengths)
    heights = list(heights)
    params = list(params)
    nu = _check_freqs(freqs)
    sw = _spectral(spectral_weights, len(wavelengths))
    chunk = int(chunk)
    if chunk < 1:
        raise ValueError("chunk must be >= 1")
    moves = record_tangents(_nominal(system, wavelengths)[0], params)  # refusals first
    B = _Bundles(system, heights, wavelengths, nrays, distribution, eng, exact)
    try:
        out = _otf_sums(eng, B, moves, nu, clip, chunk, exact)
    finally:
        B.close()
    res = _mtf_result(out, len(heights), len(wavelengths), len(params), len(nu), sw)
    res.update(freq=nu, heights=np.asarray(heights, np.float64),
               wavelengths=np.asarray(wavelengths, np.float64), params=params)
    return res


def mtf_normal(mtf, grad, targets, weights):
    """The Gauss-Newton normal equations of sum w (t - M)^2 over the
    residuals (any shape; `targets` and `weights` broadcast to it):
    JtJ = sum w g g^T, Jtr = -sum w g (t - M) with g = grad (..., P) =
    dM/dp.  Residuals with a non-finite M or gradient are left out."""
    M = np.asarray(mtf, np.float64)
    g = np.asarray(grad, np.float64)
    ok = np.isfinite(g).all(-1) & np.isfinite(M)
    g, w = g[ok], np.broadcast_to(np.asarray(weights, np.float64), M.shape)[ok]
    r = (np.broadcast_to(np.asarray(targets, np.float64), M.shape) - M)[ok]
    return np.einsum("k,ka,kb->ab", w, g, g), -np.einsum("k,ka,k->a", w, g, r)


def _trial_mtf(eng, B, params, deltas, freqs, sw, clip, exact):
    """the polychromatic MTF (V, H, 2, F) of each row of `deltas` (V, P) on
    the fixed bundles B: every variant marched keep-LAST (rtx_trace_batch,
    up to 8 bundles per launch), then rtx_otf_jacobian_sums with P = 0 about
    the current lens's centres"""
    t = perturbed_tables(B.nominal, params, deltas)
    V, W = t.shape[:2]
    nb, F = len(B.rays), len(freqs)
    Ns = [y.shape[0] for y, _ in B.rays]
    ld = max(64, -(-max(Ns)//64)*64)
    Ys = [eng.empty((1, ld, 3)) for _ in range(min(nb, 8))]
    out = np.zeros((V, nb, 2 + 4*F))
    try:
        for v in range(V):
            for b0 in range(0, nb, 8):
                bs = range(b0, min(nb, b0 + 8))
                eng.trace_device_batch([t[v, b % W] for b in bs], [B.rays[b][0] for b in bs],
                                       [B.rays[b][1] for b in bs], Ys[:len(bs)], None, None, None,
                                       Ns=[Ns[b] for b in bs], ld=ld, clip=clip, keep_last=True,
                                       rot0=B.rot0, exact=exact)
                for i, b in enumerate(bs):
                    out[v, b] = eng.otf_jacobian_sums(Ys[i].rows(0), None, freqs,
                                                      B.centers[b - b % W, :2], N=Ns[b])["out"]
    finally:
        for y in Ys:
            y.free()
    return np.array([_mtf_result(o, nb//W, W, 0, F, sw)["poly_mtf"] for o in out])


def _mtf_merits(eng, B, params, deltas, freqs, sw, targets, weights, clip, exact):
    """sum w (t - polyMTF)^2 of each row of `deltas` (V, P) on the fixed
    bundles B (_trial_mtf); a residual without rays counts as inf"""
    M = _trial_mtf(eng, B, params, deltas, freqs, sw, clip, exact)
    r2 = np.where(np.isfinite(M), (targets - M)**2, np.inf)
    return np.where(weights > 0, weights*r2, 0.).sum((1, 2, 3))


def optimize_mtf(system, params, freqs, targets=1., heights=(0., .707, 1.), wavelengths=None,
                 weights=None, iterations=20, damping=1e-3, nrays=1000, distribution="hexapolar",
                 clip=True, spectral_weights=None, lambdas=(.1, 1., 10., 100.), chunk=1 << 20,
                 engine=None, exact=False):
    """Levenberg-Marquardt on sum_h sum_a sum_j w (t_j - polyMTF_h,a(nu_j))^2,
    the polychromatic MTF of mtf_jacobian at the frequencies `freqs`, both
    axes (x, y) and every height.

    `targets` and `weights` (default 1) broadcast to (H, 2, F).  The
    parameters, loop and returns are optimize_spot's: each iteration re-aims
    the lens, takes mtf_jacobian's poly_grad g and solves with
    JtJ = sum w g g^T and Jtr = -sum w g (t - M) (mtf_normal; residuals with
    a NaN gradient are left out), scores the trial steps on the same bundles
    with the current lens's centres and applies the best one if it lowers
    the merit.  A residual at a height that no ray reaches counts as inf.
    The caller's System is not modified."""
    params = _check_kinds(params)
    eng = engine or default_engine()
    wavelengths = list(system.wavelengths if wavelengths is None else wavelengths)
    heights = list(heights)
    H, W, P = len(heights), len(wavelengths), len(params)
    nu = _check_freqs(freqs)
    F = len(nu)
    targets = _per_residual("targets", targets, (H, 2, F))
    weights = _per_residual("weights", 1. if weights is None else weights, (H, 2, F))
    sw = _spectral(spectral_weights, W)
    chunk = int(chunk)
    if chunk < 1:
        raise ValueError("chunk must be >= 1")
    record_tangents(_nominal(system, wavelengths)[0], params)  # refusals before any device work

    def normal(B, state):
        out = _otf_sums(eng, B, record_tangents(B.nominal, params), nu, clip, chunk, exact)
        res = _mtf_result(out, H, W, P, F, sw)
        return mtf_normal(res["poly_mtf"], res["poly_grad"], targets, weights)

    return _lm(system, params, heights, wavelengths, iterations, damping, nrays, distribution,
               lambdas, eng, exact, lambda system, B, final: None, normal,
               lambda B, state, deltas: _mtf_merits(eng, B, params, deltas, nu, sw, targets,
                                                    weights, clip, exact))
