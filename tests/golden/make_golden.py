#!/usr/bin/env python
"""Generate tests/golden/*.npz and systems.json FROM THE LIVE REFERENCE.

Needs the reference tree (oracle/ref_shim.py: $RAYOPT_REFERENCE or oracle/_ref):

    python tests/golden/make_golden.py                  # *.npz, systems.json
    python tests/golden/make_golden.py --vs-reference   # vs_reference/*.npz

For every case the reference's own System / GeometricTrace (imported through
oracle/ref_shim.py) produces launch rays and the full trace; the case file
stores the packed surface table (rayopt_b200.surface_table.pack_system), the
launch rays and the reference outputs y,u,i,t,n.  Nothing in these files is
produced by the oracle or the CUDA engine.

systems.json additionally stores, per fixture system and wavelength, the
packed table and the reference's pupil-aiming solution (z, p) per field, so
that the benchmark can generate aimed bundles without the reference.
"""
import json
import os
import sys
import warnings

import numpy as np
import yaml

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, HERE)

import ref_shim  # noqa: E402
import systems_yaml  # noqa: E402
from rayopt_b200.surface_table import pack_system, table_to_json  # noqa: E402

warnings.simplefilter("ignore")
R = ref_shim.load()


def build(text):
    s = R.System(**yaml.safe_load(text))
    s.update()
    s.paraxial.refocus()
    return s


def disc(n, seed):
    """uniform pupil coordinates in the unit disc (SURVEY 8d)"""
    rng = np.random.default_rng(seed)
    r = np.sqrt(rng.random(n))
    phi = 2*np.pi*rng.random(n)
    return np.c_[r*np.cos(phi), r*np.sin(phi)]


def save(name, system, g, clip, start=1, stop=None, meta=None):
    table, n, rot0 = pack_system(system, g.l, start, stop, n0=g.n[start - 1])
    sl = slice(start, stop)
    out = dict(
        table=table, n=n,
        rot0=np.zeros((0, 3)) if rot0 is None else rot0,
        y0=g.y[start - 1].copy(), u0=g.u[start - 1].copy(),
        clip=np.array(bool(clip)),
        Y=g.y[sl].copy(), U=g.u[sl].copy(), I=g.i[sl].copy(), T=g.t[sl].copy(),
        w=np.asarray(g.w, float) if g.w is not None else np.zeros(0),
        meta=np.array(json.dumps(meta or {})),
    )
    assert np.array_equal(n, g.n[sl])
    path = os.path.join(HERE, name + ".npz")
    np.savez_compressed(path, **out)
    nan = np.isnan(out["U"][-1, :, 0]).mean()
    print("%-28s S=%2d N=%4d clip=%d nan(last u)=%.2f  %6.1f kB" % (
        name, len(table), out["y0"].shape[0], clip, nan,
        os.path.getsize(path)/1e3))


def trace_aimed(system, yo, l, yp, clip, weight=None):
    g = R.GeometricTrace(system)
    z, p = system.pupil(yo, l=l)
    y, u = system.aim(yo, yp, z, p, filter=False)
    g.rays_given(y, u, l, weight)
    g.propagate(clip=clip)
    return g, z, p


def trace_given(system, y, u, clip, l=None, **kw):
    y, u = np.atleast_2d(y, u)
    if y.shape[1] == 3 and u.shape[1] == 2:
        u = np.c_[u, np.sqrt(1 - np.square(u).sum(1))]
    g = R.GeometricTrace(system)
    g.rays_given(y, u, l)
    g.propagate(clip=clip, **kw)
    return g


def main():
    systems = {k: build(v) for k, v in systems_yaml.SYSTEMS.items()}
    sysjson = {}

    # ---- systems.json: tables per wavelength + aim solutions per field ----
    for name, s in systems.items():
        ent = {"S": len(s) - 1, "wavelengths": [float(l) for l in s.wavelengths],
               "tables": [], "n": [], "aim": [],
               "object_angle": float(getattr(s.object, "angle", 0.)),
               "object_finite": bool(s.object.finite)}
        fields = [0., .25, .5, .7, .75, 1.]
        for l in s.wavelengths:
            table, n, rot0 = pack_system(s, l)
            ent["tables"].append(table_to_json(table))
            ent["n"].append([float(s.refractive_index(l, 0))] + [float(x) for x in n])
            aims = []
            for f in fields:
                try:
                    z, p = s.pupil((0, f), l=l)
                    aims.append({"field": [0., f], "z": float(z),
                                 "p": np.asarray(p, float).tolist()})
                except Exception as ex:  # aiming can fail for odd systems
                    aims.append({"field": [0., f], "error": repr(ex)})
            ent["aim"].append(aims)
        sysjson[name] = ent
    with open(os.path.join(HERE, "systems.json"), "w") as f:
        json.dump(sysjson, f, indent=0)

    # ---- C1: singlet, rays_point hexapolar 1000 -> 919 rays (SURVEY 8d) ----
    s = systems["singlet"]
    g = R.GeometricTrace(s)
    g.rays_point((0, 0.), nrays=1000, distribution="hexapolar")
    save("singlet_c1", s, g, False, meta={"config": "C1", "rms": float(g.rms())})
    g = R.GeometricTrace(s)
    g.rays_point((0, 1.), nrays=200, distribution="hexapolar", clip=True)
    save("singlet_field1_clip", s, g, True)

    # ---- Cooke: the reference's own known answer (test_raytrace.py:189-199) ----
    s = systems["cooke"]
    g = R.GeometricTrace(s)
    g.rays_point((0, 1.), nrays=13, distribution="radau", clip=False,
                 filter=False)
    save("cooke_radau13", s, g, False,
         meta={"rms": float(g.rms()), "known_answer": 0.052,
               "source": "rayopt/test/test_raytrace.py:192-195"})
    g = R.GeometricTrace(s)
    g.rays_point((0, 1.), nrays=500, distribution="square", clip=False,
                 filter=True)
    save("cooke_square500", s, g, False, meta={"rms": float(g.rms())})
    g, z, p = trace_aimed(s, (0, .7), s.wavelengths[2], disc(256, 3), True)
    save("cooke_f07_clip", s, g, True)

    # ---- C2: Double-Gauss, 3 wavelengths, field (0,.7), clip (~6% vignetted) ----
    s = systems["double_gauss"]
    for j, l in enumerate(s.wavelengths):
        g, z, p = trace_aimed(s, (0, .7), l, disc(256, 0), True)
        save("double_gauss_l%d_clip" % j, s, g, True, meta={"z": float(z),
             "p": np.asarray(p).tolist(), "field": [0, .7]})
    g, z, p = trace_aimed(s, (0, 1.), s.wavelengths[0], disc(256, 1), False)
    save("double_gauss_f1_noclip", s, g, False)
    # sub-range propagate(start, stop)
    g, z, p = trace_aimed(s, (0, .5), s.wavelengths[0], disc(64, 2), True)
    g2 = R.GeometricTrace(s)
    g2.rays_given(g.y[0], g.u[0], g.l)
    g2.propagate(clip=True)
    g2.propagate(start=4, stop=9, clip=True)
    save("double_gauss_sub_4_9", s, g2, True, start=4, stop=9)

    # ---- C3: Cooke + even aspheres (Newton intercept) ----
    s = systems["cooke_asph"]
    g, z, p = trace_aimed(s, (0, .7), s.wavelengths[0], disc(256, 1), True)
    save("cooke_asph_f07_clip", s, g, True)
    g, z, p = trace_aimed(s, (0, 0.), s.wavelengths[1], disc(128, 4), False)
    save("cooke_asph_axis", s, g, False)

    # ---- C5: zoom, fields x wavelengths ----
    s = systems["zoom"]
    for fi, f in enumerate((0., .5, 1.)):
        l = s.wavelengths[(2*fi) % 5]
        g, z, p = trace_aimed(s, (0, f), l, disc(192, 10 + fi), True)
        save("zoom_f%d_clip" % fi, s, g, True)

    # ---- mirror + rotated frames ----
    s = systems["mirror"]
    g, z, p = trace_aimed(s, (0, 1.), s.wavelengths[0], disc(128, 5), False)
    save("mirror_folded", s, g, False)

    # ---- tilted / decentred surfaces (test_elements.py:31-32 style) ----
    s = R.System(elements=[
        dict(material="air"),
        dict(distance=2., direction=(.02, .05, 1.), angles=(.03, -.02, .1),
             roc=12., material=1.5, radius=4.),
        dict(distance=1.5, direction=(-.03, .01, 1.), angles=(-.05, .04, 0.),
             roc=-15., conic=-.4, material=1.0, radius=4.),
        dict(distance=3., angles=(.1, 0, 0), material="mirror", radius=6.),
        dict(distance=-2., direction=(0, .1, 1.), radius=8.),
    ])
    s.update()
    rng = np.random.default_rng(7)
    y = np.c_[rng.normal(0, .8, (200, 2)), np.zeros(200)]
    u = rng.normal(0, .05, (200, 2))
    for clip in (False, True):
        g = trace_given(s, y, u, clip, l=587.56e-9)
        save("tilted_clip%d" % clip, s, g, clip)
    # rotated start frame: propagate(start=3) begins in a rotated frame (rot0)
    g = trace_given(s, y, u, False, l=587.56e-9)
    g.propagate(start=3, clip=False)
    save("tilted_start3", s, g, False, start=3)

    # ---- conics, alternate intersection, planes, degenerate NaNs ----
    rng = np.random.default_rng(11)
    n = 160
    y = np.c_[rng.uniform(-6, 6, (n, 2)), rng.uniform(-1, 0, n)]
    u = rng.normal(0, .15, (n, 2))
    s = R.System(elements=[
        dict(material=1.0),
        dict(distance=3., roc=9., conic=.35, material=1.7, radius=5.),   # oblate
        dict(distance=2., roc=-11., conic=-.6, material=1.0, radius=5.),  # prolate
        dict(distance=1., material=1.6, radius=5.5),                      # plane refracting
        dict(distance=2., roc=-7., conic=-1., material=1.0, radius=5.5),  # paraboloid
        dict(distance=1., roc=30., conic=-2.5, material=1.45, radius=6.),  # hyperboloid
        dict(distance=4., roc=-8., material=1.0, radius=6.),              # strong sphere: TIR + misses
        dict(distance=6., radius=3.),
    ])
    s.update()
    for clip in (False, True):
        g = trace_given(s, y, u, clip, l=550e-9)
        save("conics_clip%d" % clip, s, g, clip)

    # paraboloid hit by axis-parallel rays: e = 0 -> 0/0 (SURVEY A.5,
    # TODO.rst:3-4); alternate_intersection on a sphere
    s = R.System(elements=[
        dict(material=1.0),
        dict(distance=2., roc=-20., conic=-1., material="mirror", radius=5.),
        dict(distance=-5., roc=10., alternate_intersection=True, material=1.5,
             radius=9.),
        dict(distance=30., radius=20.),
    ])
    s.update()
    y = np.c_[rng.uniform(-3, 3, (64, 2)), np.zeros(64)]
    u = np.zeros((64, 2))
    u[32:] = rng.normal(0, .02, (32, 2))
    g = trace_given(s, y, u, False, l=550e-9)
    save("parabola_axis_alt", s, g, False)

    # Newton edge cases: aspherics=[0, 0] (pure conic through Newton), strong
    # asphere where some rays fail to converge in 5 iterations, grazing rays
    s = R.System(elements=[
        dict(material=1.0),
        dict(distance=2., roc=8., conic=-.5, aspherics=[0., 0.], material=1.5,
             radius=5.),
        dict(distance=3., roc=-6., aspherics=[1e-3, -4e-4, 2e-5, 3e-6],
             material=1.0, radius=5.),
        dict(distance=2., aspherics=[2e-2, 0, 1e-4], material=1.8, radius=5.),
        dict(distance=1., roc=4., aspherics=[0, 5e-3], material=1.0,
             radius=4.),
        dict(distance=10., radius=30.),
    ])
    s.update()
    y = np.c_[rng.uniform(-4.5, 4.5, (160, 2)), np.zeros(160)]
    u = rng.normal(0, .25, (160, 2))
    for clip in (False, True):
        g = trace_given(s, y, u, clip, l=550e-9)
        save("newton_edge_clip%d" % clip, s, g, clip)

    # single ray and 2-D (N,2) input padding (geometric_trace.py:62-67)
    s = systems["cooke"]
    g = trace_given(s, [[0., 1.5]], [[0., .05]], False)
    save("cooke_single_ray", s, g, False)


VS_REFERENCE = [("cooke", 20000, False), ("double_gauss", 20000, True),
                ("zoom", 10000, True), ("cooke_asph", 400, True), ("mirror", 5000, False),
                ("singlet", 5000, True)]


def vs_reference(keep=32):
    """vs_reference/<system>.npz: the reference's packed table, launch rays and
    full trace for the first two wavelengths of each fixture system (field
    (0, .7), n pupil points uniform in the disc), for a seeded sample of `keep`
    of those rays (tests/test_oracle_vs_reference.py)"""
    os.makedirs(os.path.join(HERE, "vs_reference"), exist_ok=True)
    for name, n, clip in VS_REFERENCE:
        s = build(systems_yaml.SYSTEMS[name])
        out = {"clip": np.array(bool(clip)), "n_rays": np.array(n)}
        for j, l in enumerate(s.wavelengths[:2]):
            g, z, p = trace_aimed(s, (0, .7), l, disc(n, 1), clip)
            table, nn, rot0 = pack_system(s, l)
            assert np.array_equal(nn, g.n[1:])
            idx = np.sort(np.random.default_rng(j).choice(n, min(n, keep), replace=False))
            out.update({"table%d" % j: table, "n%d" % j: nn,
                        "rot0%d" % j: np.zeros((0, 3)) if rot0 is None else rot0,
                        "idx%d" % j: idx, "y0%d" % j: g.y[0][idx], "u0%d" % j: g.u[0][idx],
                        "Y%d" % j: g.y[1:, idx], "U%d" % j: g.u[1:, idx],
                        "I%d" % j: g.i[1:, idx], "T%d" % j: g.t[1:, idx]})
        path = os.path.join(HERE, "vs_reference", name + ".npz")
        np.savez_compressed(path, **out)
        print("%-14s %6.1f kB" % (name, os.path.getsize(path)/1e3))


if __name__ == "__main__":
    if "--vs-reference" in sys.argv:
        vs_reference()
    else:
        main()
