"""The wavefront chain on the host, for the derivative tests: np_oracle's
march to surface `after`, its path summed left to right, and rtx_trace_opd's
epilogue (epi_oracle.opd_epilogue's formulas), with Richardson-extrapolated
central differences of the path A along a parameter.  The differences are
taken in long double, so that their rounding (eps |A| / h) stays far below
the derivatives they are compared with."""
import numpy as np

import np_oracle
from rayopt_b200.tolerance import perturbed_tables

LD = np.longdouble


def epilogue(y0, y, u, acc, spec):
    """epi_oracle.opd_epilogue's A in the arithmetic of `y`"""
    dt = y.dtype
    f = lambda a: np.asarray(a).astype(dt)               # noqa: E731
    y0, y0r, u0r = f(y0), f(spec["y0_ref"]).reshape(3), f(spec["u0_ref"]).reshape(3)
    M, d = f(spec["M"]).reshape(3, 3), f(spec["d"]).reshape(3)
    n0, n_after, radius = (dt.type(spec[k]) for k in ("n0", "n_after", "radius"))
    A = acc
    if spec["infinite"]:
        A = A - ((y0r - y0)*u0r).sum(1)*n0
    q = np.dot(y, M) + d
    q[:, 2] += radius
    v = np.dot(u, M)
    c = 1/radius
    dd = c*(v*q).sum(1) - v[:, 2]
    ff = c*(q*q).sum(1) - 2*q[:, 2]
    ti = -(dd + np.sqrt(dd*dd - c*ff))/c
    return A + ti*n_after


def path(table, y0, u0, spec, clip=False, rot0=None, dtype=LD):
    """A (N,) of rtx_trace_opd for the OPD march `table` (rows 0..after)"""
    Y, U, _, T = np_oracle.trace(table, y0, u0, clip=clip, rot0=rot0, dtype=dtype)
    acc = np.zeros(T.shape[1], T.dtype)
    for t in T:                                       # the kernel's order
        acc = acc + t
    return epilogue(y0, Y[-1], U[-1], acc, spec)


def richardson(f, h):
    """(4 D(h/2) - D(h))/3 of the central differences D of f at 0"""
    D = [(f(x) - f(-x))/(2*x) for x in (h, h/2)]
    return np.asarray((4*D[1] - D[0])/3, np.float64)


def march_column(table, y0, u0, spec, j, kind, h, clip=False, rot0=None, dopd=None):
    """dA/dp by differences: the OPD march table perturbed along (j, kind)
    and, with `dopd` (4,), the spec's d and n_after moved along it"""
    def f(x):
        t = perturbed_tables(table, [(j, kind)], [[x]])[0, 0]
        sp = dict(spec)
        if dopd is not None:
            sp["d"] = np.asarray(spec["d"], LD) + LD(x)*np.asarray(dopd[:3], LD)
            sp["n_after"] = LD(spec["n_after"]) + LD(x)*LD(dopd[3])
        return path(t, y0, u0, sp, clip, rot0)
    with np.errstate(all="ignore"):
        return richardson(f, h)
