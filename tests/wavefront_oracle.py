"""Forward-mode restatement of rtx_trace_opd_jacobian: each ray's optical
path A (epi_oracle.opd_epilogue of np_oracle's march) and its derivatives
dA (P, N) with respect to P lens parameters -- THE WAVEFRONT ORACLE.

TEST INFRASTRUCTURE ONLY.  The march is oracle/jac_oracle.py's, expression
by expression, keeping the whole (y, u) and their tangents, plus the path
tangent dT += n0 ds + s dn0 of every surface; the epilogue's derivative
follows include/rtx.h: dq = dy M + dd, dv = du M, the sphere root ti of
Phi(x) = c |x|^2 - 2 x_z differentiated implicitly at P = q + ti v, and
dA = dT + n_after dti + ti dn_after, with M and the radius held fixed and
the centre moved by `dopd` (P, 4).  tests/test_wavefront_host.py checks it
against Richardson-extrapolated central differences of the host chain
(tests/wavefront_chain.py).
"""
import numpy as np

import epi_oracle
import jac_oracle
import np_oracle

_dot = jac_oracle._dot


def _dn0(moves):
    """per parameter: {row: summed d(n0)}"""
    out = []
    for mv in moves:
        d = {}
        for row, rec in mv:
            d[int(row)] = d.get(int(row), 0.) + float(rec["n0"])
        out.append(d)
    return out


def trace_opd(table, y0, u0, moves, spec, dopd, clip=False, rot0=None):
    """A (N,) as rtx_trace_opd gives it for the march `table` (rows 0 ..
    after) and dA (P, N)"""
    S = len(table)
    tans = jac_oracle._dense(moves, S)
    dn0s = _dn0(moves)
    P = len(tans)
    dopd = np.asarray(dopd, np.float64).reshape(P, 4)
    y = np.array(y0, np.float64)
    u = np.array(u0, np.float64)
    N = y.shape[0]
    dy = np.zeros((P, N, 3))
    du = np.zeros((P, N, 3))
    dT = np.zeros((P, N))
    acc = np.zeros(N)
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
            s = np_oracle.intercept(rec, y2, u2)
            h = y2 + s[:, None]*u2
            acc = acc + s*float(rec["n0"])                 # np_oracle's t, summed in order
            uc = np_oracle.clip(rec, h, u2) if clip else u2
            uo = np_oracle.refract(rec, h, uc) if float(rec["mu"]) else uc
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
                dT[p] = dT[p] + float(rec["n0"])*ds + s*dn0s[p].get(j, 0.)
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
        Aout = epi_oracle.opd_epilogue(y0, y, u, acc, spec)[0]
        # ---- the epilogue's tangents
        M = np.asarray(spec["M"], np.float64).reshape(3, 3)
        d = np.asarray(spec["d"], np.float64).reshape(3)
        radius, n_after = float(spec["radius"]), float(spec["n_after"])
        q = np.dot(y, M) + d
        q[:, 2] += radius
        v = np.dot(u, M)
        c = 1/radius
        uyv, yyv = _dot(v, q), _dot(q, q)
        dd = c*uyv - v[:, 2]
        ff = c*yyv - 2*q[:, 2]
        ti = -(dd + np.sqrt(dd*dd - c*ff))/c
        Pt = q + ti[:, None]*v
        g = c*Pt - np.array([0., 0., 1.])
        gv = _dot(g, v)
        dA = np.empty((P, N))
        for p in range(P):
            dq = np.dot(dy[p], M) + dopd[p, :3]
            dv = np.dot(du[p], M)
            dti = -_dot(g, dq + ti[:, None]*dv)/gv
            dA[p] = dT[p] + n_after*dti + ti*dopd[p, 3]
    return Aout, dA
