"""The long-double oracle of rtx_trace_zernike_many: the exact Gram sums of
(a, Z_1 .. Z_J) over one item's rays and include/rtx.h's bound on each."""
import math

import numpy as np

from rayopt_b200.zernike import noll, nterms, radial_coefficients, zernike_basis

EPS = 2.0**-52


def basis_bound(J, r):
    """(N, J) rtx.h's bound (a) on each device basis value at the
    normalised radii r: (n+2)^2 eps N_j A_j max(1, r)^n"""
    R = np.maximum(1., np.asarray(r, np.float64))
    out = np.empty((len(R), J))
    for j, (n, m) in enumerate(noll(J)):
        N = math.sqrt(n + 1) if m == 0 else math.sqrt(2*(n + 1))
        A = sum(abs(c) for c in radial_coefficients(n, m))
        out[:, j] = (n + 2)**2*EPS*N*A*R**n
    return out


def oracle(A, P, a0, c, rho, order):
    """(sums (E,) long double, bound (E,), n, r2max) of one item's per-ray
    path A (N,) and sphere point P (N, 3): a = A - a0, x = P_x - c_x, y =
    P_y - c_y formed in FP64 as the device forms them (so the same rays
    enter and r2max is the same bits), then the exact Zernike values at
    (x, y)/rho in long double"""
    J = nterms(order)
    with np.errstate(all="ignore"):
        a = A - a0
        x = P[:, 0] - c[0]
        y = P[:, 1] - c[1]
    ok = np.isfinite(a) & np.isfinite(x) & np.isfinite(y)
    a, x, y = a[ok], x[ok], y[ok]
    r2max = float((x*x + y*y).max()) if ok.any() else 0.
    ld = np.longdouble
    u, v = np.asarray(x, ld)/ld(rho), np.asarray(y, ld)/ld(rho)
    Z = zernike_basis(J, u, v)
    V = np.concatenate([np.asarray(a, ld)[:, None], Z], 1)
    Eb = np.concatenate([np.zeros((len(a), 1)),
                         basis_bound(J, np.sqrt((u*u + v*v).astype(np.float64)))], 1)
    iu = np.triu_indices(J + 1)
    sums = np.einsum("ij,ik->jk", V, V)[iu]
    Vf = np.abs(V.astype(np.float64))
    mag = np.einsum("ij,ik->jk", Vf, Vf)[iu]
    basis = (np.einsum("ij,ik->jk", Eb, Vf) + np.einsum("ij,ik->jk", Vf, Eb)
             + np.einsum("ij,ik->jk", Eb, Eb))[iu]
    N = len(A)
    # (b) on the device's products, whose magnitudes are within (a) of these
    bound = (512 + -(-N//512))*EPS*(mag + basis) + basis
    return sums, bound, int(ok.sum()), r2max
