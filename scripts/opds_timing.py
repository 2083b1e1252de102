#!/usr/bin/env python
"""Times of the OPD regridding with the exit-pupil points kept in HBM
(rtx_opd_points) against the host round trip it replaces, and of
rayopt_b200.opds, in one run.

    python scripts/opds_timing.py [--nrays 1e4 1e5 1e6] [--reps 5] [--out FILE]

Workload (as psf_timing.py): Cooke triplet at field 0.7, hexapolar bundle,
resident trace (ResidentTrace), resample 4, device triangulation.  Needs the
reference's System (its tree staged by build() under oracle/_ref) and an H100.

- old: ``opd_rays`` (rtx_trace_opd and the download of every ray's A, P),
  numpy's reference subtraction and finite filter, the upload of the points
  and values, rtx_delaunay and rtx_grid_linear;
- new: ``_opd_grid`` (rtx_trace_opd, rtx_opd_points, rtx_delaunay and
  rtx_grid_linear on the arrays in HBM), split into the points stage and the
  triangulation + regridding stage;
- opds: ``rayopt_b200.opds`` for heights 0, .707 and 1 (contour OPD, PSF,
  encircled energy and MTF per height).

Each row gives the median, min and max over --reps repetitions of the wall
time (host clock around work that ends in a device synchronise) and of the
CUDA-event time of the same window (rtx_timer_*), after one warm-up of every
shape.  The old and new grids are compared bit for bit in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests", "golden")):
    sys.path.insert(0, p)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nrays", type=float, nargs="+", default=[1e4, 1e5, 1e6])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out")
    a = ap.parse_args()
    warnings.simplefilter("ignore")
    np.seterr(all="ignore")
    import yaml
    import ref_shim
    import systems_yaml
    import rayopt_b200
    from rayopt_b200 import ResidentTrace
    from rayopt_b200.engine import Engine
    from rayopt_b200.lazy import regrid
    R = ref_shim.load()
    eng = Engine(0)
    info = card()
    print("card: %s (name, power limit)" % info)
    s = R.System(**yaml.safe_load(systems_yaml.SYSTEMS["cooke"]))
    s.update()
    s.paraxial.refocus()
    g = ResidentTrace(s, engine=eng)
    rows = []

    def timed(fn):
        """(result, wall s, CUDA-event ms) of fn, which ends synchronised"""
        eng.sync()
        eng.timer_start()
        t0 = time.perf_counter()
        r = fn()
        eng.sync()
        t1 = time.perf_counter()
        return r, t1 - t0, eng.timer_stop()

    for nr in a.nrays:
        g.rays_point((0, .7), nrays=int(nr), distribution="hexapolar", clip=True)
        n = int(4*g.nrays**.5)

        def old():
            st = {}
            (x, y, t), st["old_opd_rays_s"], st["old_opd_rays_ev_ms"] = timed(g.opd_rays)

            def up():
                ok = np.isfinite(x) & np.isfinite(y) & np.isfinite(t)
                xo, yo, to = x[ok], y[ok], t[ok]
                h = np.fabs((xo, yo)).max()
                return (eng.to_device(np.stack([xo, yo], axis=-1)), eng.to_device(to),
                        int(to.size), h)
            pts, st["old_filter_upload_s"], st["old_filter_upload_ev_ms"] = timed(up)
            (_, _, o), st["old_regrid_s"], st["old_regrid_ev_ms"] = timed(
                lambda: regrid(eng, *pts, n, False, "device"))
            st["old_total_s"] = st["old_opd_rays_s"] + st["old_filter_upload_s"] + st["old_regrid_s"]
            st["old_total_ev_ms"] = (st["old_opd_rays_ev_ms"] + st["old_filter_upload_ev_ms"]
                                     + st["old_regrid_ev_ms"])
            return st, o

        def new():
            st = {}

            def points():
                A, P = g._trace_opd(None, -2, -1)
                try:
                    return eng.opd_points(A, P, int(g.ref), g.l/s.scale)
                finally:
                    A.free(), P.free()
            pts, st["new_points_s"], st["new_points_ev_ms"] = timed(points)
            (_, _, o), st["new_regrid_s"], st["new_regrid_ev_ms"] = timed(
                lambda: regrid(eng, *pts, n, False, "device"))
            (_, _, o2), st["new_opd_grid_s"], st["new_opd_grid_ev_ms"] = timed(
                lambda: g._opd_grid(None, -2, -1, 4, download=False, triangulation="device"))
            o2.free()
            return st, o

        def report():
            st = {}
            _, st["opds_3_heights_s"], st["opds_3_heights_ev_ms"] = timed(
                lambda: rayopt_b200.opds(s, (0., .707, 1.), nrays=int(nr), engine=eng))
            return st

        reps = []
        for k in range(a.reps + 1):                   # the first pass warms every shape
            so, oo = old()
            sn, on = new()
            same = oo.download().tobytes() == on.download().tobytes()
            oo.free(), on.free()
            if k:
                reps.append(dict(so, **sn, **report(), same_grid=same))
            else:
                report()
        row = dict(nrays=g.nrays, n=n, card=info, reps=a.reps,
                   same_grid_bits=all(r.pop("same_grid") for r in reps))
        for key in reps[0]:
            v = [r[key] for r in reps]
            row[key] = (statistics.median(v), min(v), max(v))
        rows.append(row)
        print(json.dumps(row))
    g.free()
    eng.close()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
