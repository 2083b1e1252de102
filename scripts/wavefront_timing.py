#!/usr/bin/env python
"""Times of the device wavefront Jacobian (rtx_trace_opd_jacobian,
rtx_wavefront_sums) next to the spot Jacobian (rtx_trace_jacobian,
rtx_jacobian_sums) at the same P, of a whole wavefront_jacobian call and of
one optimize_wavefront iteration.

    python scripts/wavefront_timing.py [--params 4 20 40] [--nrays 1e4 1e6]
                                       [--reps 5] [--out FILE]

Workload: the Double-Gauss lens (tests/golden/systems.json), 3 field heights
(0, 0.7, 1) x 3 wavelengths, P parameters (curvatures, distances and conics
of its curved surfaces, then other distances and aspherics), clip off, FP64
fast mode; the OPD march is the table without its image row and the sphere
(radius -100) is centred on each bundle's first ray.  The launch rays are
generated on the host (aim_infinite of a disc).  For each P and bundle
size it prints one JSON line: the median kernel ms (CUDA events) of each
call summed over the 9 bundles, and the card's name and power limit read
in the same run.  With the reference staged, the whole wavefront_jacobian
call on the Double-Gauss System and one optimize_wavefront iteration of the
Cooke triplet (1e4 rays per bundle) are timed on the host clock.
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests"),
          os.path.join(ROOT, "tests", "golden"), os.path.join(ROOT, "scripts")):
    sys.path.insert(0, p)

from jacobian_timing import card, reference_system  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--params", type=int, nargs="+", default=[4, 20, 40])
    ap.add_argument("--nrays", type=float, nargs="+", default=[1e4, 1e6])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out")
    a = ap.parse_args()
    np.seterr(all="ignore")
    from conftest import load_systems
    from rayopt_b200.engine import Engine
    from rayopt_b200.rays import aim_infinite, disc
    from rayopt_b200.tolerance import record_tangents
    eng = Engine(0)
    gpu = card()
    ent = load_systems()["double_gauss"]
    nominal = np.stack(ent["tables"][:3])
    W, S = nominal.shape
    curved = [j for j in range(1, S) if nominal[0]["c"][j - 1] != 0]
    lines = []
    for nr in a.nrays:
        n = int(nr)
        bundles = []
        for li in range(W):
            for h in range(3):
                aim = ent["aim"][li][h]
                y0, u0 = aim_infinite(aim["field"], disc(n, 10*li + h)*.95, aim["z"], aim["p"],
                                      ent["object_angle"])
                spec = dict(y0_ref=y0[0], u0_ref=u0[0], n0=1., n_after=1., M=np.eye(3),
                            d=np.array([0., 0., 0.]), radius=-100., infinite=1)
                bundles.append((li, eng.to_device(y0), eng.to_device(u0), spec))
        for P in a.params:
            cands = ([(j, k) for k in ("curvature", "distance", "conic") for j in curved]
                     + [(j, "distance") for j in range(1, S) if j not in curved]
                     + [(j, x) for x in ("asph0", "asph1") for j in curved])
            params = cands[:P]
            opd_moves = record_tangents(nominal[:, :-1], params)
            spot_moves = record_tangents(nominal, params)
            dopd = np.zeros((P, 4))
            t = {k: [] for k in ("opd_jacobian", "wavefront_sums", "spot_jacobian", "spot_sums")}
            for rep in range(a.reps + 1):                 # rep 0 warms up
                acc = dict.fromkeys(t, 0.)
                for li, y0, u0, spec in bundles:
                    mv = [[(r, rec[li]) for r, rec in m] for m in opd_moves]
                    A, dA = eng.trace_opd_jacobian(nominal[li, :-1], y0, u0, spec, mv, dopd)
                    eng.sync()
                    acc["opd_jacobian"] += eng.last_kernel_ms()
                    eng.wavefront_sums(A, dA, 0.)
                    acc["wavefront_sums"] += eng.last_kernel_ms()
                    A.free(), dA.free()
                    mv = [[(r, rec[li]) for r, rec in m] for m in spot_moves]
                    q, J = eng.trace_jacobian(nominal[li], y0, u0, mv)
                    eng.sync()
                    acc["spot_jacobian"] += eng.last_kernel_ms()
                    eng.jacobian_sums(q, J)
                    acc["spot_sums"] += eng.last_kernel_ms()
                    q.free(), J.free()
                if rep:
                    for k in t:
                        t[k].append(acc[k])
            line = dict(P=P, nrays_per_bundle=n, bundles=len(bundles),
                        **{k + "_kernel_ms": statistics.median(v) for k, v in t.items()}, gpu=gpu)
            print(json.dumps(line), flush=True)
            lines.append(line)
        for _, y, u, _ in bundles:
            y.free(), u.free()
    import ref_shim
    if ref_shim.available():
        lines += whole_calls(eng, gpu, a.params, a.nrays, a.reps)
    if a.out:
        with open(a.out, "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")
    eng.close()


def whole_calls(eng, gpu, Ps, nrays, reps):
    """wavefront_jacobian on the Double-Gauss System and one
    optimize_wavefront iteration of the Cooke triplet, host clock, medians
    after a warm-up"""
    from rayopt_b200 import optimize as opt
    from rayopt_b200.surface_table import pack_system
    out = []
    s = reference_system("double_gauss")
    t = pack_system(s, s.wavelengths[0], 1, None)[0]
    S = len(t)
    curved = [j for j in range(1, S) if t["c"][j - 1] != 0]
    cands = ([(j, k) for k in ("curvature", "distance", "conic") for j in curved]
             + [(j, "distance") for j in range(1, S + 1) if j not in curved]
             + [(j, x) for x in ("asph0", "asph1") for j in curved])
    for nr in nrays:
        for P in Ps:
            ms = []
            for rep in range(reps + 1):
                t0 = time.perf_counter()
                opt.wavefront_jacobian(s, cands[:P], (0., .7, 1.), nrays=int(nr), engine=eng)
                if rep:
                    ms.append(1e3*(time.perf_counter() - t0))
            line = dict(what="wavefront_jacobian call, Double-Gauss System, 3 heights x 3 "
                        "wavelengths", P=P, nrays_per_bundle=int(nr),
                        call_ms=statistics.median(ms), gpu=gpu)
            print(json.dumps(line), flush=True)
            out.append(line)
    c = reference_system("cooke")
    t = pack_system(c, c.wavelengths[0], 1, None)[0]
    params = [(j, "curvature") for j in range(1, len(t)) if t["c"][j - 1] != 0][:6]
    params.append((len(t), "distance"))
    kw = dict(heights=(0., .7, 1.), nrays=10000, engine=eng)
    opt.optimize_wavefront(c, params, iterations=1, **kw)          # warm-up
    ms = []
    for _ in range(3):
        t0 = time.perf_counter()
        opt.optimize_wavefront(c, params, iterations=1, **kw)
        ms.append(1e3*(time.perf_counter() - t0))
    line = dict(what="optimize_wavefront iteration, Cooke, P=7, 9 bundles x 1e4 rays",
                iteration_ms=statistics.median(ms), gpu=gpu)
    print(json.dumps(line), flush=True)
    out.append(line)
    return out


if __name__ == "__main__":
    main()
