"""Launch-ray generation for aimed bundles: host numpy restatements, which the
tests and the benchmark compare the device generator (rtx_aim_rays) against,
and the per-field `rtx_aim` records that generator reads.

Restates, for the cases the benchmark workloads need, what the reference does
upstream of the hot path:  ``InfiniteConjugate.aim`` with the rectilinear
projection (rayopt/conjugates.py:208-213, 236-255), ``Pupil.map`` with
``filter=False`` (rayopt/pupils.py:97-107) and ``sagittal_meridional``
(rayopt/utils.py:102-114), given a pupil-aiming solution ``(z, p)`` that the
reference's ``System.pupil`` solved on the host (rayopt/system.py:585-593).
The object surface (``system[0]``) is taken to be a plane, as in every fixture.
"""
import numpy as np


def disc(n, seed):
    """uniform pupil coordinates in the unit disc: r = sqrt(U), phi = 2 pi U"""
    rng = np.random.default_rng(seed)
    r = np.sqrt(rng.random(n))
    phi = 2*np.pi*rng.random(n)
    return np.c_[r*np.cos(phi), r*np.sin(phi)]


def hexapolar(nrays):
    """pupil_distribution("hexapolar", nrays) (rayopt/utils.py:174-180):
    returns (rings, xy (N,2)); N = 1 + 3 rings (rings + 1)"""
    n = int(np.sqrt(nrays/3. - 1/12.) - 1/2.)
    l = [np.zeros((2, 1))]
    for i in range(1, n + 1):
        a = np.linspace(0, 2*np.pi, 6*i, endpoint=False)
        l.append([np.sin(a)*i/n, np.cos(a)*i/n])
    return n, np.concatenate(l, axis=1).T


def hexapolar_xy(idx, rings):
    """pupil coordinates of rays `idx` of the hexapolar grid with `rings`
    rings (rayopt/utils.py:174-180) without building the whole grid: ray 0 on
    axis; ring i = 1..rings holds rays 3 i (i-1) < j <= 3 i (i+1) at angles
    k 2 pi/(6 i) -- the index arithmetic of the device generator (pupil_xy in
    rtx_device.cuh), used to check samples of 1e8-ray device-generated bundles"""
    idx = np.asarray(idx, np.int64)
    i = np.floor((1 + np.sqrt(1 + 4*np.maximum(idx - 1, 0)/3.))/2).astype(np.int64)
    i = np.where(3*i*(i + 1) < idx, i + 1, i)
    i = np.where(3*i*(i - 1) >= idx, i - 1, i)
    i = np.maximum(i, 1)
    k = idx - 1 - 3*i*(i - 1)
    a = k*(2*np.pi/(6*i))
    xy = np.c_[np.sin(a)*i/rings, np.cos(a)*i/rings]
    xy[idx == 0] = 0
    return xy


def aim_infinite(yo, yp, z, p, angle):
    """Rays (y, u), each (N, 3), for fractional object coordinate `yo` (2,),
    fractional pupil coordinates `yp` (N, 2), pupil distance `z`, pupil
    half-apertures `p` (2, 2) and object semi-angle `angle` (radians)."""
    yo = np.atleast_2d(np.asarray(yo, float))
    yp = np.atleast_2d(np.asarray(yp, float))
    p = np.asarray(p, float)
    yp = yp*np.fabs(p).max()                               # pupils.py:100-101
    yo, yp = np.broadcast_arrays(yo, yp)
    n = yo.shape[0]
    yt = yo*np.tan(angle)                                  # conjugates.py:211
    u = np.hstack((yt, np.ones((n, 1))))
    u /= np.sqrt(np.square(u).sum(-1))[:, None]
    yz = np.array((0, 0, z), float)
    y = yz - z*u                                           # conjugates.py:249
    s = np.cross(u, yz)                                    # utils.py:103-110
    axial = np.all(s == 0, axis=-1)[..., None]
    s = np.where(axial, (1., 0, 0), s)
    m = np.cross(u, s)
    s /= np.sqrt(np.square(s).sum(-1))[..., None]
    m /= np.sqrt(np.square(m).sum(-1))[..., None]
    y += yp[..., 0, None]*s + yp[..., 1, None]*m           # conjugates.py:252
    y += (-y[:, 2]/u[:, 2])[..., None]*u                   # plane object surface, :254
    return y, u


def finite_frame(yo, z, radius, telecentric=False, surface=None):
    """Per-field constants of FiniteConjugate.aim: object point y (3,), chief
    direction u = (0,0,z) - y, or (0,0,z) for a `telecentric` pupil (3,),
    normalised sagittal and meridional axes s, m (3,).  `surface`: a curved
    object surface, on which the object point lies."""
    yo = np.atleast_2d(np.asarray(yo, float))
    y = np.zeros((1, 3))
    y[..., :2] = -yo*radius                                # conjugates.py:151
    if surface is not None:
        y[..., 2] = -surface.surface_sag(y)                # :153
    uz = np.array((0, 0, z), float)
    u = np.tile(uz, (1, 1)) if telecentric else uz - y    # :155-158
    s, m = _sagittal_meridional(u, uz)
    return y[0], u[0], s[0], m[0]


def aim_finite(yo, yp, z, p, radius):
    """FiniteConjugate.aim (rayopt/conjugates.py:137-166) for a non-telecentric
    pupil, a plane object surface and ``filter=False``: object point at
    ``-yo*radius``, pupil coordinates mapped through the pupil half-angles
    ``arctan2(p, z)`` (Pupil.map, rayopt/pupils.py:97-101), direction
    ``normalize(u + z tan(yp_x) s + z tan(yp_y) m)``, flipped if z < 0."""
    yp = np.atleast_2d(np.asarray(yp, float))
    a = np.arctan2(np.asarray(p, float), z)                # conjugates.py:146
    yp = yp*np.fabs(a).max()                               # pupils.py:100-101
    yp = z*np.tan(yp)                                      # conjugates.py:149
    y0, u0, s, m = finite_frame(yo, z, radius)
    n = yp.shape[0]
    y = np.broadcast_to(y0, (n, 3)).copy()
    u = np.broadcast_to(u0, (n, 3)).copy()
    u += yp[..., 0, None]*s + yp[..., 1, None]*m           # conjugates.py:161
    u /= np.sqrt(np.square(u).sum(-1))[..., None]          # normalize, utils.py:97-98
    if z < 0:
        u *= -1
    return y, u


# --------------------------------------------------------------------------
# General device generator (rtx_aim_plan / rtx_aim_rays): the host side builds
# one `rtx_aim` record per field point with the reference's own expressions.

GRID_GIVEN, GRID_HEXAPOLAR, GRID_SQUARE, GRID_TRIANGULAR, GRID_RANDOM, GRID_LINES = range(6)


def aim_dtype():
    """numpy mirror of `struct rtx_aim` (include/rtx.h)"""
    from .surface_table import SURFACE_DTYPE
    return np.dtype([("conjugate", "<i4"), ("grid", "<i4"), ("filter", "<i4"), ("curved", "<i4"),
                     ("n", "<i8"), ("seed", "<u8"), ("seg", "<f8", (2, 4)), ("seg_m", "<i8", (2,)),
                     ("frame", "<f8", (12,)), ("pmax", "<f8"), ("z", "<f8"), ("fc", "<f8", (2,)),
                     ("fd2", "<f8", (2,)), ("surface", SURFACE_DTYPE)], align=True)


def grid_spec(distribution, nrays):
    """pupil_distribution (rayopt/utils.py:118-199) as a grid description the
    device evaluates per ray: returns (ref, dict(grid, n, seg, seg_m)) or
    (ref, None) for the distributions that stay on the host (one ray; the
    Gauss-Radau / Lobatto quadrature nodes)."""
    d, n = distribution, int(nrays)
    z4 = (0., 0., 0., 0.)
    if n == 1 or d in ("radau", "lobatto"):
        return 0, None
    if d == "half-meridional":
        return 0, dict(grid=GRID_LINES, seg=((0., 0., 0., 1.), z4), seg_m=(n, 0))
    if d == "meridional":
        n -= n % 2
        return 0, dict(grid=GRID_LINES, seg=((0., -1., 0., 1.), z4), seg_m=(n + 1, 0))
    if d == "sagittal":
        n -= n % 2
        return n//2, dict(grid=GRID_LINES, seg=((-1., 0., 1., 0.), z4), seg_m=(n + 1, 0))
    if d == "cross":
        n -= n % 4
        return n//4, dict(grid=GRID_LINES, seg=((0., -1., 0., 1.), (-1., 0., 1., 0.)),
                          seg_m=(n//2 + 1, n//2 + 1))
    if d == "tee":
        n = (n - 2)//3
        return 2*n + 1, dict(grid=GRID_LINES, seg=((0., -1., 0., 1.), (0., 0., 1., 0.)),
                             seg_m=(2*n + 1, n + 1))
    if d == "random":
        return 0, dict(grid=GRID_RANDOM, n=n)
    if d in ("square", "triangular"):
        return 0, dict(grid=GRID_SQUARE if d == "square" else GRID_TRIANGULAR,
                       n=int(np.sqrt(n*4/np.pi)))
    if d == "hexapolar":
        return 0, dict(grid=GRID_HEXAPOLAR, n=int(np.sqrt(n/3. - 1/12.) - 1/2.))
    raise ValueError("unknown ray distribution", d)


def pupil_grid(yp, nrays=None, rings=None):
    """`grid` of a bundle whose pupil coordinates are the device array `yp`
    (None: GRID_GIVEN), or else of the hexapolar grid with `rings` rings or
    about `nrays` rays"""
    if yp is not None:
        return None
    if rings is None:
        _, g = grid_spec("hexapolar", nrays)
        rings = 0 if g is None else g["n"]       # one ray: the axial ray alone
    return dict(grid=GRID_HEXAPOLAR, n=rings)


def project(yo, angle, projection="rectilinear"):
    """InfiniteConjugate.map (rayopt/conjugates.py:208-234): field -> direction"""
    yo = np.atleast_2d(np.asarray(yo, float))
    n, p, a = yo.shape[0], projection, angle
    if p == "rectilinear":
        y = yo*np.tan(a)
        u = np.hstack((y, np.ones((n, 1))))
        u /= np.sqrt(np.square(u).sum(-1))[:, None]
    elif p == "stereographic":
        y = yo*(2*np.tan(a/2))
        r = np.square(y).sum(-1)[:, None]/4
        u = np.hstack((y, 1 - r))/(r + 1)
    elif p == "equisolid":
        y = yo*(2*np.sin(a/2))
        r = np.square(y).sum(-1)[:, None]
        u = np.hstack((y*np.sqrt(1 - r/4), 1 - r/2))
    elif p == "orthographic":
        # (the reference raises here: its hstack of ``np.sqrt(1 - r)[:, None]``
        # with r already (n,1) has mismatched dimensions, conjugates.py:225-226;
        # this is the evident intent u = (y, sqrt(1 - |y|^2)))
        y = yo*np.sin(a)
        r = np.square(y).sum(-1)[:, None]
        u = np.hstack((y, np.sqrt(1 - r)))
    elif p == "equidistant":
        y = yo*a
        b = np.square(y).sum(-1) > (np.pi/2)**2
        y = np.sin(y)
        z = np.sqrt(np.square(y).sum(-1))
        u = np.hstack((y, np.where(b, -z, z)[:, None]))
    else:
        raise ValueError("unknown projection", p)
    return u


def _sagittal_meridional(u, z):
    """rayopt/utils.py:102-114 for one direction"""
    s = np.cross(u, z)
    if np.all(s == 0):
        s = np.array([[1., 0, 0]])
    m = np.cross(u, s)
    s = s/np.sqrt(np.square(s).sum(-1))[..., None]
    m = m/np.sqrt(np.square(m).sum(-1))[..., None]
    return s, m


def _curved(surface):
    return surface is not None and (getattr(surface, "curvature", 0.) or
                                    getattr(surface, "aspherics", None) is not None)


def _record(conjugate, frame, a, z, grid, filter, seed):
    """the `rtx_aim` record of one field point with pupil half-apertures (or,
    finite, half-angles) `a` (2, 2)"""
    rec = np.zeros(1, aim_dtype())
    r = rec[0]
    r["conjugate"] = conjugate
    r["frame"] = np.concatenate(frame)
    r["pmax"] = np.fabs(a).max()                           # pupils.py:100
    r["z"] = z
    r["filter"] = int(bool(filter))
    c, d = np.sum(a, axis=0)/2, np.diff(a, axis=0)[0]/2    # pupils.py:103-104
    r["fc"], r["fd2"] = c, d**2
    g = grid or dict(grid=GRID_GIVEN)
    r["grid"] = g["grid"]
    r["n"] = g.get("n", 0)
    r["seed"] = seed
    r["seg"] = g.get("seg", np.zeros((2, 4)))
    r["seg_m"] = g.get("seg_m", (0, 0))
    return rec


def infinite_record(yo, z, p, angle, projection="rectilinear", grid=None, filter=False,
                    surface=None, seed=0):
    """`rtx_aim` record of InfiniteConjugate.aim (conjugates.py:236-255) for
    field point `yo` of an object at semi-angle `angle` in `projection`;
    frame (u, ybase = yz - z*u, s, m)"""
    u = project(yo, angle, projection)
    yz = np.array((0, 0, z), float)
    s, m = _sagittal_meridional(u, yz)
    frame = u[0], (yz - z*u)[0], s[0], m[0]                # :249
    rec = _record(0, frame, np.asarray(p, float).reshape(2, 2), z, grid, filter, seed)
    if _curved(surface):
        from .elements import _Bare
        from .surface_table import pack_element
        r = rec[0]
        r["curved"] = 1
        pack_element(r["surface"], _Bare(surface, mu=1.), 1., None)
    return rec


def finite_record(yo, z, p, radius, telecentric=False, grid=None, filter=False, surface=None,
                  seed=0):
    """`rtx_aim` record of FiniteConjugate.aim (conjugates.py:137-166) for
    field point `yo` of an object of `radius`; frame as finite_frame"""
    a = np.arctan2(np.asarray(p, float).reshape(2, 2), z)  # conjugates.py:146
    frame = finite_frame(yo, z, radius, telecentric, surface if _curved(surface) else None)
    return _record(1, frame, a, z, grid, filter, seed)


def aim_record(obj, yo, z, p, grid=None, filter=False, surface=None, seed=0):
    """One `rtx_aim` record for field point `yo` of a rayopt conjugate `obj`
    (``system.object``: InfiniteConjugate or FiniteConjugate, duck-typed) with
    the pupil-aiming solution ``(z, p)`` of ``System.pupil``; `grid` from
    grid_spec() (None: pupil coordinates are given), `surface` = ``system[0]``."""
    if getattr(obj, "finite", False):
        return finite_record(yo, z, p, obj.radius, obj.pupil.telecentric, grid, filter, surface,
                             seed)
    return infinite_record(yo, z, p, obj.angle, getattr(obj, "projection", "rectilinear"), grid,
                           filter, surface, seed)
