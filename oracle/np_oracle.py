"""numpy restatement of rayopt's geometric propagate loop -- THE ORACLE.

TEST INFRASTRUCTURE ONLY.  Only tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs may import this file.  The product
(rayopt_b200/) never does: it fails loudly when the CUDA library is missing.

This is a CPU restatement of the reference algorithm for the hot path, written
against the same per-surface POD table (`rtx_surface`, include/rtx.h) that the
CUDA engine consumes, so that reference -> table -> {oracle, CUDA} can be
compared array by array.  Every function cites the reference lines it follows
(paths relative to the reference tree, quartiq/rayopt @ a51f1db).  It keeps
numpy's evaluation order expression by expression, so on this NumPy build it is
BIT-IDENTICAL to the live reference for unrotated systems (pinned by
tests/test_oracle_vs_reference.py when /root/reference is present, and by the
committed fixtures tests/golden/*.npz generated from the live reference by
tests/golden/make_golden.py).

The aspheric intercept restates scipy.optimize.newton (SciPy 1.18.1,
scipy/optimize/_zeros_py.py, scalar Newton-Raphson branch) -- a third-party
dependency of the reference (elements.py:345-346) -- as a vectorised loop with
identical per-ray semantics (<= 5 iterations, F==0 exit, F'==0 -> NaN,
|p-p0| <= 1e-7 exit, otherwise NaN).
"""
import numpy as np

NEWTON_TOL = 1e-7      # elements.py:346
NEWTON_MAXITER = 5     # elements.py:346

F_ROTATED = 1
F_ALT = 2


def _aspherics(rec):
    n = int(rec["n_asph"])
    if n < 0:
        return None
    return [float(a) for a in rec["asph"][:n]]


def surface_sag(rec, xyz):
    """Spheroid.surface_sag, elements.py:440-455."""
    c = float(rec["c"])
    asph = _aspherics(rec)
    e = xyz[..., 2].copy()
    if not c and asph is None:
        return e
    xy = xyz[..., :2]
    r2 = xy[..., 0]*xy[..., 0] + xy[..., 1]*xy[..., 1]   # einsum, :445
    if c:
        e -= c*r2/(1 + np.sqrt(1 - float(rec["kc2"])*r2))  # :448
    if asph is not None:
        d = 0.
        for ai in reversed(asph):                          # :451-453
            d += ai
            d *= r2
        e -= d
    return e


def surface_normal(rec, xyz):
    """Spheroid.surface_normal, elements.py:457-475 (un-normalised)."""
    c = float(rec["c"])
    asph = _aspherics(rec)
    q = np.zeros_like(xyz)
    q[..., 2] = 1
    if not c and asph is None:
        return q
    xy = xyz[..., :2]
    r2 = xy[..., 0]*xy[..., 0] + xy[..., 1]*xy[..., 1]   # einsum, :463
    e = 0.
    if c:
        e -= c/np.sqrt(1 - float(rec["kc2"])*r2)         # :467
    if asph is not None:
        d = 0.
        for i in reversed(range(len(asph))):               # :470-472
            d *= r2
            d += float(rec["dasph"][i])
        e -= d
    q[..., :2] = xy*e[..., None]
    return q


def intercept_plane(y, u):
    """Element.intercept, elements.py:195-201."""
    return -y[:, 2]/u[:, 2]


def intercept_newton(rec, y, u):
    """Interface.intercept, elements.py:333-349, with scipy.optimize.newton
    (fprime given, tol=1e-7, maxiter=5, rtol=0) restated per ray."""
    with np.errstate(all="ignore"):
        p0 = intercept_plane(y, u)
        out = np.full_like(p0, np.nan)
        active = np.ones(p0.shape, bool)
        for _ in range(NEWTON_MAXITER):
            pos = y + p0[:, None]*u                       # :339 yi + si*ui
            fval = surface_sag(rec, pos)
            hit = active & (fval == 0)                    # "if fval == 0"
            out[hit] = p0[hit]
            active &= ~hit
            q = surface_normal(rec, pos)
            fder = (q[:, 0]*u[:, 0] + q[:, 1]*u[:, 1]) + q[:, 2]*u[:, 2]  # :342
            zero = active & (fder == 0)                   # RuntimeError -> NaN
            active &= ~zero
            p = p0 - fval/fder
            tol = NEWTON_TOL
            if p.dtype == np.float32:
                # 1e-7 is below float32 resolution for |p| > 1: a few ulp of the
                # iterate instead, the FP32 engine's rule (rtx_device.cuh)
                tol = np.maximum(np.float32(NEWTON_TOL), np.float32(4*2.0**-23)*np.abs(p))
            conv = active & (np.abs(p - p0) <= tol)        # np.isclose rtol=0
            conv |= active & (p == p0)                    # equal infinities
            out[conv] = p[conv]
            active &= ~conv
            p0 = p
        return out


def intercept(rec, y, u):
    """Spheroid.intercept, elements.py:477-501."""
    if int(rec["n_asph"]) >= 0:
        return intercept_newton(rec, y, u)                # :478-479
    c, k = float(rec["c"]), float(rec["k"])
    if c == 0:
        return -y[:, 2]/u[:, 2]                           # :483
    if not k:
        uy = (u*y).sum(1)                                 # :485
        uu = 1.
        yy = np.square(y).sum(1)
    else:
        kk = np.array([(1, 1, 1 + k)], y.dtype)           # :489 (float64 in the reference)
        uy = (u*y*kk).sum(1)
        uu = (np.square(u)*kk).sum(1)
        yy = (np.square(y)*kk).sum(1)
    d = c*uy - u[:, 2]
    e = c*uu
    f = c*yy - 2*y[:, 2]
    g = np.sqrt(np.square(d) - e*f)
    if int(rec["flags"]) & F_ALT:
        g *= -1                                           # :497-498
    s = -(d + g)/e
    return s


def clip(rec, y, u):
    """Element.clip, elements.py:206-209."""
    good = np.square(y[:, :2]).sum(1) <= float(rec["radius2"])
    return np.where(good[:, None], u, np.nan)


def refract(rec, y, u0):
    """Interface.refract, elements.py:351-369."""
    mu = float(rec["mu"])
    if mu == 1:
        return u0
    r = surface_normal(rec, y)
    r2 = np.square(r).sum(1)
    muf = float(rec["muf"])
    a = muf*(u0*r).sum(1)/r2
    if mu == -1:
        u = u0 - 2*a[:, None]*r
    else:
        b = float(rec["mu2m1"])/r2
        g = -a + float(rec["sgn"])*np.sqrt(np.square(a) - b)
        u = muf*u0 + g[:, None]*r
    return u


def propagate_surface(rec, y0, u0, do_clip):
    """Interface.propagate, elements.py:306-315."""
    t = intercept(rec, y0, u0)
    y = y0 + t[:, None]*u0
    if do_clip:
        u0 = clip(rec, y, u0)
    u = u0
    if float(rec["mu"]):
        u = refract(rec, y, u0)
    return y, u, t*float(rec["n0"])


def trace(table, y0, u0, clip=False, rot0=None, dtype=np.float64):
    """GeometricTrace.propagate + System.propagate, geometric_trace.py:72-80,
    system.py:459-464.  Returns Y,U,I (S,N,3) and T (S,N) in `dtype`
    arithmetic.  float64 is the reference.  float32 evaluates the SAME
    expressions entirely in float32 (the table scalars enter as Python floats,
    weak under NEP 50, so nothing is promoted): the error budget of "the
    reference's formulas in single precision" that the FP32 engine is held
    against in tests/test_gpu_parity.py."""
    dtype = np.dtype(dtype)
    y = np.array(y0, dtype)
    u = np.array(u0, dtype)
    S, N = len(table), y.shape[0]
    Y = np.empty((S, N, 3), dtype)
    U = np.empty_like(Y)
    I = np.empty_like(Y)
    T = np.empty((S, N), dtype)
    with np.errstate(all="ignore"):
        if rot0 is not None:
            r = np.asarray(rot0, dtype).reshape(3, 3)
            y, u = np.dot(y, r), np.dot(u, r)             # geometric_trace.py:76
        for j, rec in enumerate(table):
            rotated = int(rec["flags"]) & F_ROTATED
            y = y - np.asarray(rec["offset"], dtype)      # system.py:461
            i = u
            if rotated:                                   # elements.py:156-163
                r = np.asarray(rec["rot"], dtype).reshape(3, 3)
                y, i = np.dot(y, r.T), np.dot(u, r.T)
            y, u, t = propagate_surface(rec, y, i, clip)  # system.py:462
            Y[j], U[j], I[j], T[j] = y, u, i, t           # system.py:463
            if rotated:
                y, u = np.dot(y, r), np.dot(u, r)         # system.py:464
    return Y, U, I, T


def rms(y_last, w=None, ref=None):
    """GeometricTrace.rms, geometric_trace.py:171-183 (not NaN-masked)."""
    y = y_last[:, :2]
    y0 = y.mean(0) if ref is None else y[ref]
    r = np.square(y - y0).sum(1)
    if w is None:
        w = np.ones_like(r)/r.shape[0]
    return np.sqrt((r*w).sum())
