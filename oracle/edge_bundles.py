"""Launch bundles on the numerical decision boundaries of the trace.

TEST INFRASTRUCTURE ONLY (tests/test_edge_oracle.py, tests/test_gpu_domain_edges.py).

Every case is a small hand-made surface table (the boundary sits at surface 0,
a plane at z = 10 follows so that a NaN reaches the last surface and the
vignetting mask) and a bundle of launch rays.  A *walked* family varies one
launch coordinate: bisection over the doubles finds two adjacent values on
which np_oracle.trace decides differently (ray kept / lost at surface 0), and
the family holds the last kept ray, the first lost ray, W more ulps on either
side and a few rays far from the boundary.  A *fixed* family is a handful of
rays placed on a representable boundary (discriminant exactly 0, F' exactly 0,
signed zeros, infinities).

Per ray, `margin` is the distance from the oracle's boundary in ulps of the
walked coordinate (1 for the edge pair; 0: placed on a boundary; inf: no
boundary nearby), which is what
the fast-mode and FP32 mask rules of tests/test_gpu_domain_edges.py are stated
in.  Near a boundary one ulp of the coordinate moves the boundary quantity
(r2 - radius2, the discriminant, a^2 - b) by one or two of its own ulps.
"""
import types
from fractions import Fraction

import numpy as np

import np_oracle
from rayopt_b200.surface_table import SURFACE_DTYPE, pack_element

W = 3                       # ulps walked on either side of the transition
FAR = (1e-9, 1e-3)          # relative offsets of the far rays
LIFT = 10.                  # z of the plane after the boundary surface


def surface(c=0., k=0., asph=None, radius=np.inf, n0=1., n=None, mirror=False, z=0.,
            alt=False):
    """one record, filled by the packer from a duck-typed element"""
    e = types.SimpleNamespace(offset=(0., 0., z), rotated=False, curvature=c, conic=k,
                              aspherics=asph, radius=radius, alternate_intersection=alt)
    if mirror:
        e.get_n_mu = lambda n0_, l: (n0_, -1.)
    elif n is not None:
        e.get_n_mu = lambda n0_, l: (n, n0_/n)
    rec = np.zeros(1, SURFACE_DTYPE)
    pack_element(rec[0], e, n0, 5.876e-7)
    return rec, e


def table(*recs):
    return np.concatenate([r for r, _ in recs])


def key(x):
    """monotone integer order of doubles (-0 and +0 share 0)"""
    i = np.asarray(x, np.float64).view(np.int64)
    return np.where(i >= 0, i, -(i & 0x7fffffffffffffff))


def lost(tab, y0, u0, clip, at="U", j=0):
    """per ray: the oracle loses it at surface j (NaN in U, or in Y)"""
    Y, U, I, T = np_oracle.trace(tab, y0, u0, clip=clip)
    return np.isnan((U if at == "U" else Y)[j]).any(1)


class Case:
    def __init__(self, name, tab, clip, elements):
        self.name, self.table, self.clip, self.elements = name, tab, clip, elements
        self.y0, self.u0 = np.empty((0, 3)), np.empty((0, 3))
        self.margin = np.empty(0)
        self.edges = []         # (i_kept, i_lost, at): adjacent rays straddling the boundary

    def add(self, y0, u0, margin):
        y0, u0 = np.atleast_2d(np.asarray(y0, float)), np.atleast_2d(np.asarray(u0, float))
        n = len(self.y0)
        self.y0, self.u0 = np.vstack([self.y0, y0]), np.vstack([self.u0, u0])
        self.margin = np.concatenate([self.margin, np.broadcast_to(margin, (len(y0),))])
        return n

    def walk(self, family, lo, hi, at="U"):
        """bisect family(x) -> (y0, u0) between lo and hi (decided differently)"""
        dec = lambda x: bool(lost(self.table, *family(np.array([x])), self.clip, at)[0])  # noqa: E731
        dlo, dhi = dec(lo), dec(hi)
        assert dlo != dhi, (self.name, lo, hi)
        while True:
            mid = lo + (hi - lo)/2
            if mid in (lo, hi):
                break
            if dec(mid) == dlo:
                lo = mid
            else:
                hi = mid
        xs = [lo, hi]
        for _ in range(W):
            xs = [np.nextafter(xs[0], -np.inf)] + xs + [np.nextafter(xs[-1], np.inf)]
        scale = max(abs(lo), 1.)
        far = [lo - d*scale for d in FAR] + [hi + d*scale for d in FAR]
        xs = np.array(xs + far)
        k = key(xs)
        margin = np.minimum(abs(k - key(lo)), abs(k - key(hi))) + 1.   # 1 at the edge pair
        n = self.add(*family(xs), margin.astype(float))
        ik, il = (n + W, n + W + 1) if not dlo else (n + W + 1, n + W)
        self.edges.append((ik, il, at))
        return self


def _axial(yv):
    def fam(x):
        y0 = np.stack([x, np.full_like(x, yv), np.full_like(x, -1.)], 1)
        return y0, np.tile([0., 0., 1.], (len(x), 1))
    return fam


def _oblique(yv, ux):
    uz = np.sqrt(1 - ux*ux)

    def fam(x):
        y0 = np.stack([x, np.full_like(x, yv), np.full_like(x, -1.)], 1)
        return y0, np.tile([ux, 0., uz], (len(x), 1))
    return fam


def _direction(yv):
    """u = (x, 0, sqrt(1 - x^2)) from (yv, 0, -1): walks the incidence angle"""
    def fam(x):
        y0 = np.tile([yv, 0., -1.], (len(x), 1))
        return y0, np.stack([x, np.zeros_like(x), np.sqrt(1 - x*x)], 1)
    return fam


def fused_flip_rim(rad2, xs, yv):
    """rays whose clip decision flips when r2 = x*x + y*y fuses the y product
    (the kernel's fast r2: fma(y, y, x*x)); exact, in Fraction"""
    out = []
    yy = Fraction(yv)**2
    for x in xs:
        ref = float(x)*float(x) + yv*yv <= rad2
        fused = float(yy + Fraction(float(x)*float(x))) <= rad2
        out.append(ref != fused)
    return np.array(out)


def _rim_yv(R):
    """a y for the axial rim family at which the fused r2 flips a walked ray"""
    for yv in np.linspace(.11, .97, 400)*R:
        c = Case("probe", table(surface(radius=R), surface(z=LIFT)), True, None)
        c.walk(_axial(yv), 0., R)
        fin = np.isfinite(c.margin)
        if fused_flip_rim(R*R, c.y0[fin, 0], yv).any():
            return float(yv)
    raise AssertionError("no fused-flip ray found")


def cases():
    """all boundary cases (deterministic)"""
    out = []
    # ---- aperture rim: r2 == radius2 exactly (3^2 + 4^2 = 5^2) and walked
    s0 = surface(radius=5.)
    c = Case("rim_exact", table(s0, surface(z=LIFT)), True, [s0])
    c.walk(_axial(4.), 2.5, 3.5)
    out.append(c)
    R = 1.3
    s0 = surface(radius=R)
    yv = _rim_yv(R)
    c = Case("rim_axial", table(s0, surface(z=LIFT)), True, [s0])
    c.walk(_axial(yv), 0., R)
    out.append(c)
    s0 = surface(radius=R)
    c = Case("rim_oblique", table(s0, surface(z=LIFT)), True, [s0])
    c.walk(_oblique(.4, .28), 0., 1.2)
    c.walk(_oblique(-.7, -.6), -.5, 1.2)
    out.append(c)
    s0 = surface(c=.05, radius=5., n=1.5)
    c = Case("rim_sphere_axial", table(s0, surface(z=LIFT, n0=1.5)), True, [s0])
    c.walk(_axial(4.), 2.5, 3.5)
    c.walk(_axial(1.7), 4., 4.9)
    out.append(c)
    # ---- tangent intercept: sphere c = 1/8, x = 8 along z: discriminant 0
    for alt in (False, True):
        s0 = surface(c=.125, alt=alt)
        c = Case("tangent_sphere" + "_alt"*alt, table(s0, surface(z=LIFT)), False, [s0])
        c.add([[8., 0., -1.], [-8., 0., -1.], [0., 8., -1.]], [[0., 0., 1.]]*3, 0.)
        c.walk(_axial(0.), 7., 9., at="Y")
        c.walk(_oblique(1., .6), -6., 9., at="Y")
        out.append(c)
    # ... and its refraction: w = 1 - c^2 r2 -> 0 at the hemisphere rim
    s0 = surface(c=.125, n=1.5)
    c = Case("hemisphere_rim", table(s0, surface(z=LIFT, n0=1.5)), False, [s0])
    c.add([[8., 0., -1.], [0., -8., -1.]], [[0., 0., 1.]]*2, 0.)
    c.walk(_axial(0.), 7., 9., at="U")
    out.append(c)
    # conics: ellipsoids (k > -1) along z, hyperboloid (k < -1) obliquely
    for k in (-.5, .7, -3.):
        for alt in (False, True):
            s0 = surface(c=.1, k=k, alt=alt)
            c = Case("tangent_conic_k%g" % k + "_alt"*alt, table(s0, surface(z=LIFT)), False,
                     [s0])
            if k > -1:
                rmax = 1/(.1*np.sqrt(1 + k))
                c.walk(_axial(0.), .5*rmax, 1.5*rmax, at="Y")
                c.walk(_axial(.3*rmax), .5*rmax, 1.5*rmax, at="Y")
            else:
                c.walk(_oblique(0., .9), 10., 20., at="Y")
            out.append(c)
    # ---- critical angle, dense to thin (mu = 1.5): plane and sphere
    s0 = surface(n0=1.5, n=1.)
    c = Case("critical_plane", table(s0, surface(z=LIFT)), False, [s0])
    c.walk(_direction(.2), .5, .9)
    c.walk(_direction(-.3), -.9, -.5)
    out.append(c)
    s0 = surface(c=.1, n0=1.5, n=1.)
    c = Case("critical_sphere", table(s0, surface(z=LIFT)), False, [s0])
    c.walk(_axial(0.), 5., 9.)
    c.walk(_axial(.5), -9., -5.)
    out.append(c)
    # ---- mirror at normal incidence, and mu == 1 exactly (the early return)
    s0 = surface(mirror=True)
    s1 = surface(c=-.05, mirror=True)
    for name, s in (("mirror_plane", s0), ("mirror_sphere", s1)):
        c = Case(name, table(s, surface(z=-LIFT)), True, [s])
        z, m = 0., -0.
        c.add([[z, z, -1.], [m, z, -1.], [z, m, -1.], [m, m, -1.], [.3, .2, -1.]],
              [[z, z, 1.], [z, m, 1.], [m, z, 1.], [m, m, 1.], [z, z, 1.]], np.inf)
        out.append(c)
    s0 = surface(c=.125, n0=1.5, n=1.5)
    c = Case("mu_one", table(s0, surface(z=LIFT, n0=1.5)), False, [s0])
    c.add([[8., 0., -1.], [0., 0., -1.], [3., 4., -1.]], [[0., 0., 1.]]*3, 0.)
    out.append(c)
    # ---- paraboloid: the axis ray has e = c uu = 0 (0/0 or x/0), one ulp off is finite
    for alt in (False, True):
        s0 = surface(c=.1, k=-1., alt=alt, n=1.5)
        c = Case("paraboloid" + "_alt"*alt, table(s0, surface(z=LIFT, n0=1.5)), False, [s0])
        t = np.nextafter(0., 1.)*2.**60
        c.add([[0., 0., -1.], [1., .5, -1.], [1., .5, -1.], [0., 0., -1.]],
              [[0., 0., 1.], [0., 0., 1.], [t, 0., np.sqrt(1 - t*t)], [0., -t, 1.]], 0.)
        out.append(c)
    # ---- planes: parallel rays (u.z = +-0) and rays starting on the plane (y.z = +-0)
    s0 = surface(n=1.5)
    c = Case("plane_zeros", table(s0, surface(z=0., n0=1.5), surface(z=LIFT, n0=1.5)), False,
             [s0])
    z, m = 0., -0.
    for y in ([.3, .2, z], [.3, .2, m], [z, m, z], [m, z, m], [m, m, z], [.3, .2, -1.],
              [z, z, -1.]):
        for u in ([z, z, 1.], [z, z, -1.], [.6, z, .8], [m, .6, -.8], [1., z, z], [1., z, m],
                  [.8, .6, z], [m, -1., m]):
            c.add([y], [u], np.inf)
    out.append(c)
    # ---- Newton surfaces
    # a start already on the surface: F == 0 on the first iteration (a flat
    # base with an empty list makes the reference's surface_normal raise, so
    # the flat one has a zero coefficient)
    s0 = surface(asph=[0.])
    c = Case("newton_flat_root", table(s0, surface(z=LIFT)), False, [s0])
    c.add([[.3, .2, -1.], [z, m, -1.], [.3, .2, z], [.3, .2, m]], [[z, z, 1.], [.6, z, .8],
          [z, z, 1.], [z, z, 1.]], np.inf)
    out.append(c)
    s0 = surface(c=.2, asph=[], n=1.5)                      # sphere through Newton
    c = Case("newton_sphere_empty", table(s0, surface(z=LIFT, n0=1.5)), True, [s0])
    c.add([[z, z, -1.], [m, z, -1.], [1., .5, -1.], [z, z, z]], [[z, z, 1.]]*4, np.inf)
    out.append(c)
    # flat base with aspherics: F' = e (x ux + y uy) + uz = 0 exactly at the
    # first iterate (1, 0, 0): e = -2 a0 = -1, u = (1/2, 0, 1/2)
    s0 = surface(asph=[.5], n=1.5)
    c = Case("newton_zero_slope", table(s0, surface(z=LIFT, n0=1.5)), False, [s0])
    x1 = np.nextafter(0., 1.)*2.**1000
    c.add([[0., 0., -1.], [x1, 0., -1.], [-x1, 0., -1.], [0., 1e-300, -1.]], [[.5, 0., .5]]*4, 0.)
    out.append(c)
    # F == 0 exactly where F' is NaN: the first iterate (8, 0, 0) is on the
    # rim (w = 0) of a sphere whose aspheric term cancels its sag there; the
    # reference returns the start before it looks at F'
    s0 = surface(c=.125, asph=[-.125], n=1.5)
    c = Case("newton_root_at_rim", table(s0, surface(z=LIFT, n0=1.5)), False, [s0])
    c.add([[8., 0., -1.], [np.nextafter(8., 9.), 0., -1.], [0., -8., -1.]], [[0., 0., 1.]]*3,
          0.)
    out.append(c)
    # convergence on exactly the 5th iteration / one more needed: a steep
    # asphere, rays walked across the oracle's convergence boundary
    s0 = surface(c=.1, asph=[1e-2, 1e-3], n=1.5)
    c = Case("newton_fifth", table(s0, surface(z=LIFT, n0=1.5)), False, [s0])
    fam = _oblique(0., .6)
    xs = np.linspace(2., 3., 1001)
    it = _newton_iterations(c.table, *fam(xs))
    c.add(*fam(xs[it == 5][:2]), 0.)
    c.add(*fam(xs[it == 6][:2]), 0.)
    j = int(np.flatnonzero(it >= 6)[0])
    c.walk(fam, xs[j - 1], xs[j], at="Y")
    out.append(c)
    return out


def _newton_iterations(tab, y0, u0):
    """per ray: the iteration on which the oracle's Newton at surface 0
    converges (1..6; 7 = not within 6)"""
    rec = tab[0]
    y = y0 - rec["offset"]
    it = np.full(len(y0), 7)
    old = np_oracle.NEWTON_MAXITER
    try:
        for n in range(6, 0, -1):
            np_oracle.NEWTON_MAXITER = n
            ok = ~np.isnan(np_oracle.intercept_newton(rec, y, u0))
            it[ok] = n
    finally:
        np_oracle.NEWTON_MAXITER = old
    return it


NONFINITE = [np.nan, np.inf, -np.inf]


def mixed_bundle(y0, u0, seed=5):
    """finite launch rays with one component of every fourth ray replaced by
    NaN, +inf, -inf, +0 or -0 (so that early retirement and clamped lanes sit
    in warps of finite rays); returns y0, u0 and the per-ray finite flag"""
    rng = np.random.default_rng(seed)
    y0, u0 = y0.copy(), u0.copy()
    vals = NONFINITE + [0., -0.]
    for n, i in enumerate(range(1, len(y0), 4)):
        a = y0 if rng.integers(2) else u0
        a[i, rng.integers(3)] = vals[n % len(vals)]
    fin = np.isfinite(y0).all(1) & np.isfinite(u0).all(1)
    return y0, u0, fin
