"""Forward-mode restatement of np_oracle.trace: each ray's image point and its
derivatives with respect to P lens parameters -- THE JACOBIAN ORACLE.

TEST INFRASTRUCTURE ONLY (as np_oracle).  A parameter is a list of moves
(row, record): the derivative of table[row] with respect to it, the unit
rtx_trace_jacobian takes (rayopt_b200.tolerance.record_tangents builds them).
The primal is np_oracle's, expression by expression; the tangents follow it
with the same linearisation the kernel states in include/rtx.h: the
intercept is differentiated implicitly at the primal hit point p = y + s u
of Phi(p; record) = 0, with Phi the sag form z - sag(r2) on plane and Newton
surfaces and the quadric c (x^2 + y^2 + (1+k) z^2) - 2 z on spheres and
conics (either sheet); clipping passes the tangents through and a clipped
direction's tangent is NaN.  tests/test_jacobian_host.py checks it against
Richardson-extrapolated central differences of np_oracle.trace.
"""
import numpy as np

import np_oracle


def _dense(moves, S):
    """per parameter: {row: summed derivative record fields}"""
    out = []
    for mv in moves:
        d = {}
        for row, rec in mv:
            f = d.setdefault(int(row), dict(off=np.zeros(3), rot=np.zeros((3, 3)), c=0., k=0.,
                                             kc2=0., muf=0., mu2m1=0., asph=np.zeros(10),
                                             dasph=np.zeros(10)))
            f["off"] += np.asarray(rec["offset"], float)
            f["rot"] += np.asarray(rec["rot"], float).reshape(3, 3)
            for k in ("c", "k", "kc2", "muf", "mu2m1"):
                f[k] += float(rec[k])
            f["asph"] += np.asarray(rec["asph"], float)
            f["dasph"] += np.asarray(rec["dasph"], float)
        out.append(d)
    return out


def _dot(a, b):
    return (a*b).sum(-1)


def trace(table, y0, u0, moves, clip=False, rot0=None):
    """q (N, 2) at the last surface of `table` (np_oracle.trace's Y[-1, :,
    :2]) and J (P, 2, N) = dq/dp"""
    S = len(table)
    tans = _dense(moves, S)
    P = len(tans)
    y = np.array(y0, np.float64)
    u = np.array(u0, np.float64)
    N = y.shape[0]
    dy = np.zeros((P, N, 3))
    du = np.zeros((P, N, 3))
    with np.errstate(all="ignore"):
        if rot0 is not None:
            r = np.asarray(rot0, np.float64).reshape(3, 3)
            y, u = np.dot(y, r), np.dot(u, r)
        for j, rec in enumerate(table):
            rotated = int(rec["flags"]) & np_oracle.F_ROTATED
            R = np.asarray(rec["rot"], np.float64).reshape(3, 3)
            T = [t.get(j) for t in tans]
            y1 = y - np.asarray(rec["offset"], np.float64)
            ui = u
            y2, u2 = (np.dot(y1, R.T), np.dot(ui, R.T)) if rotated else (y1, ui)
            for p, t in enumerate(T):
                a, b = dy[p], du[p]
                if t is not None:
                    a = a - t["off"]
                if rotated:
                    a, b = np.dot(a, R.T), np.dot(b, R.T)
                if t is not None:
                    a, b = a + np.dot(y1, t["rot"].T), b + np.dot(ui, t["rot"].T)
                dy[p], du[p] = a, b
            # ---- primal step (np_oracle.propagate_surface)
            s = np_oracle.intercept(rec, y2, u2)
            h = y2 + s[:, None]*u2
            uc = np_oracle.clip(rec, h, u2) if clip else u2
            uo = np_oracle.refract(rec, h, uc) if float(rec["mu"]) else uc
            # ---- the intercept's implicit derivative
            c, k, kc2 = float(rec["c"]), float(rec["k"]), float(rec["kc2"])
            na = max(int(rec["n_asph"]), 0)
            x_, y_, z_ = h[:, 0], h[:, 1], h[:, 2]
            r2 = x_*x_ + y_*y_
            w = 1 - kc2*r2
            sq = np.sqrt(w)
            e = -c/sq - sum(float(rec["dasph"][i])*r2**i for i in range(na))
            e_r2 = -c*kc2/(2*w*sq) - sum(i*float(rec["dasph"][i])*r2**(i - 1)
                                         for i in range(1, na))
            quad = int(rec["n_asph"]) < 0 and c != 0
            if quad:
                g = np.stack([2*c*x_, 2*c*y_, 2*c*(1 + k)*z_ - 2], -1)
                phi = dict(c=r2 + (1 + k)*z_*z_, k=c*z_*z_, kc2=0.*r2)
                hz = g[:, 2]
            else:
                g = np.stack([x_*e, y_*e, np.ones_like(e)], -1)
                phi = dict(c=-r2/(1 + sq), k=0.*r2, kc2=-c*r2*r2/(2*sq*(1 + sq)**2))
                hz = np.ones_like(e)
            gu = _dot(g, u2)
            n = np.stack([x_*e, y_*e, np.ones_like(e)], -1)
            rr2 = _dot(n, n)
            mu, muf, sgn, mu2m1 = (float(rec[f]) for f in ("mu", "muf", "sgn", "mu2m1"))
            dotn = _dot(u2, n)
            A = muf*dotn/rr2
            Bq = mu2m1/rr2
            root = np.sqrt(A*A - Bq)
            G = -A + sgn*root
            for p, t in enumerate(T):
                m = dy[p] + s[:, None]*du[p]
                num = _dot(g, m)
                de = 0.*r2
                dmuf = dmu2m1 = 0.
                if t is not None:
                    da = sum(t["asph"][i]*r2**(i + 1) for i in range(10))
                    num = num + phi["c"]*t["c"] + phi["k"]*t["k"] + phi["kc2"]*t["kc2"] - hz*da
                    de = (-t["c"]/sq - c*r2*t["kc2"]/(2*w*sq)
                          - sum(t["dasph"][i]*r2**i for i in range(10)))
                    dmuf, dmu2m1 = t["muf"], t["mu2m1"]
                ds = -num/gu
                dh = m + ds[:, None]*u2
                dv = du[p]
                if float(rec["mu"]) and mu != 1:
                    de = de + e_r2*2*(x_*dh[:, 0] + y_*dh[:, 1])
                    dn = np.stack([dh[:, 0]*e + x_*de, dh[:, 1]*e + y_*de, 0.*de], -1)
                    drr2 = 2*_dot(n, dn)
                    ddot = _dot(du[p], n) + _dot(u2, dn)
                    dA = (dmuf*dotn + muf*ddot)/rr2 - A*drr2/rr2
                    if mu == -1:
                        dv = du[p] - 2*(dA[:, None]*n + A[:, None]*dn)
                    else:
                        dB = dmu2m1/rr2 - Bq*drr2/rr2
                        dG = -dA + sgn*(2*A*dA - dB)/(2*root)
                        dv = dmuf*u2 + muf*du[p] + dG[:, None]*n + G[:, None]*dn
                dv = np.where(np.isnan(uo[:, :1]), np.nan, dv)
                dy[p], du[p] = dh, dv
            y, u = h, uo
            if j + 1 < S:
                for p, t in enumerate(T):
                    a, b = dy[p], du[p]
                    if rotated:
                        a, b = np.dot(a, R), np.dot(b, R)
                    if t is not None:
                        a, b = a + np.dot(h, t["rot"]), b + np.dot(uo, t["rot"])
                    dy[p], du[p] = a, b
                if rotated:
                    y, u = np.dot(y, R), np.dot(u, R)
    return y[:, :2].copy(), np.transpose(dy[:, :, :2], (0, 2, 1)).copy()
