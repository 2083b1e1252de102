#!/usr/bin/env python
"""Times of the device Jacobian (rtx_trace_jacobian, rtx_jacobian_sums), of
spot_jacobian and of one optimize_spot iteration, next to the central-
difference gradient through rtx_trace_reduce_many.

    python scripts/jacobian_timing.py [--params 4 20 40] [--nrays 1e4 1e6]
                                      [--reps 5] [--out FILE]

Workload: the Double-Gauss lens (tests/golden/systems.json), 3 field heights
(0, 0.7, 1) x 3 wavelengths, P parameters (curvatures, distances and conics
of its curved surfaces, then other distances and aspherics), clip off, FP64
fast mode.  The launch rays are generated on the host (aim_infinite of a
disc) so that no System is needed.
For each P and bundle size it prints one JSON line: the median kernel ms
(CUDA events) of rtx_trace_jacobian and rtx_jacobian_sums summed over the 9
bundles, the host-clock ms of the whole Jacobian (both calls per bundle,
synchronised), the median kernel ms of the difference gradient (2P+1
variants of every bundle in one rtx_trace_reduce_many launch), and the
card's name and power limit read in the same run.  With the reference
staged, the whole spot_jacobian call on the Double-Gauss System (hexapolar
bundles aimed by the System and generated in HBM) is timed for the same P
and bundle sizes, and one optimize_spot iteration of the Cooke triplet (six curvatures and
the image distance, 1e4 rays per bundle) is split into host aiming and the
rest.  The registers and spills of the new kernels come from -Xptxas -v
(DESIGN.md 3.12), not from this script.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests"),
          os.path.join(ROOT, "tests", "golden")):
    sys.path.insert(0, p)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def med(xs):
    return statistics.median(xs)


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
    from rayopt_b200.tolerance import record_tangents, sensitivity_deltas, perturbed_tables
    eng = Engine(0)
    gpu = card()
    ent = load_systems()["double_gauss"]
    nominal = np.stack(ent["tables"][:3])
    W, S = nominal.shape
    H = 3
    curved = [j for j in range(1, S + 1) if nominal[0]["c"][j - 1] != 0]
    kinds = ("curvature", "distance", "conic")
    lines = []
    for nr in a.nrays:
        n = int(nr)
        bundles = []
        for li in range(W):
            for h in range(H):
                aim = ent["aim"][li][h]
                y0, u0 = aim_infinite(aim["field"], disc(n, 10*li + h)*.95, aim["z"], aim["p"],
                                      ent["object_angle"])
                bundles.append((li, eng.to_device(y0), eng.to_device(u0)))
        centers = np.zeros((len(bundles), 4))
        for P in a.params:
            cands = ([(j, k) for k in kinds for j in curved]
                     + [(j, "distance") for j in range(1, S + 1) if j not in curved]
                     + [(j, a) for a in ("asph0", "asph1") for j in curved])
            params = cands[:P]
            moves = record_tangents(nominal, params)
            kj, ks, wall = [], [], []
            for rep in range(a.reps + 1):
                tj = tsum = 0.
                eng.sync()
                t0 = time.perf_counter()
                for li, y0, u0 in bundles:
                    mv = [[(r, rec[li]) for r, rec in m] for m in moves]
                    q, J = eng.trace_jacobian(nominal[li], y0, u0, mv)
                    eng.sync()
                    tj += eng.last_kernel_ms()
                    eng.jacobian_sums(q, J, (0., 0.))
                    tsum += eng.last_kernel_ms()
                    q.free(), J.free()
                t1 = time.perf_counter()
                if rep:                                        # rep 0 warms up
                    kj.append(tj), ks.append(tsum), wall.append(1e3*(t1 - t0))
            d = sensitivity_deltas([1e-5]*P)
            t = perturbed_tables(nominal, params, d)
            V = len(d)
            vv, bb = np.meshgrid(np.arange(V), np.arange(len(bundles)), indexing="ij")
            items = np.stack([vv.reshape(-1)*W + np.array([b[0] for b in bundles])[bb.reshape(-1)],
                              bb.reshape(-1)], -1)
            kd = []
            for rep in range(a.reps + 1):
                eng.trace_reduce_many(t.reshape(V*W, S), [(y, u, None) for _, y, u in bundles],
                                      items, centers[bb.reshape(-1)])
                if rep:
                    kd.append(eng.last_kernel_ms())
            line = dict(P=P, nrays_per_bundle=n, bundles=len(bundles),
                        jacobian_kernel_ms=med(kj), sums_kernel_ms=med(ks),
                        jacobian_call_ms=med(wall), jacobian_call_ms_range=[min(wall), max(wall)],
                        difference_kernel_ms=med(kd), difference_variants=V, gpu=gpu)
            print(json.dumps(line), flush=True)
            lines.append(line)
        for _, y, u in bundles:
            y.free(), u.free()
    import ref_shim
    if ref_shim.available():
        lines += spot_jacobian_calls(eng, gpu, a.params, a.nrays, a.reps)
        lines.append(optimize_iteration(eng, gpu))
    if a.out:
        with open(a.out, "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")
    eng.close()


def reference_system(name):
    import warnings
    import yaml
    import ref_shim
    import systems_yaml
    warnings.simplefilter("ignore")
    R = ref_shim.load()
    s = R.System(**yaml.safe_load(systems_yaml.SYSTEMS[name]))
    s.update()
    return s


def spot_jacobian_calls(eng, gpu, Ps, nrays, reps):
    """the whole spot_jacobian call on the Double-Gauss System (host aiming,
    launch rays generated in HBM, the Jacobian and its sums per bundle, the
    host formulas), host clock, medians after a warm-up"""
    from rayopt_b200 import optimize as opt
    from rayopt_b200.surface_table import pack_system
    s = reference_system("double_gauss")
    t = pack_system(s, s.wavelengths[0], 1, None)[0]
    S = len(t)
    curved = [j for j in range(1, S + 1) if t["c"][j - 1] != 0]
    cands = ([(j, k) for k in ("curvature", "distance", "conic") for j in curved]
             + [(j, "distance") for j in range(1, S + 1) if j not in curved]
             + [(j, a) for a in ("asph0", "asph1") for j in curved])
    out = []
    for nr in nrays:
        for P in Ps:
            kw = dict(heights=(0., .7, 1.), nrays=int(nr), engine=eng)
            ms = []
            for rep in range(reps + 1):
                t0 = time.perf_counter()
                opt.spot_jacobian(s, cands[:P], **kw)
                if rep:
                    ms.append(1e3*(time.perf_counter() - t0))
            line = dict(what="spot_jacobian call, Double-Gauss System, 3 heights x 3 wavelengths",
                        P=P, nrays_per_bundle=int(nr), call_ms=med(ms),
                        call_ms_range=[min(ms), max(ms)], gpu=gpu)
            print(json.dumps(line), flush=True)
            out.append(line)
    return out


def optimize_iteration(eng, gpu):
    """one optimize_spot iteration of the Cooke triplet: host aiming
    (launch_bundles and the chief rays) against the whole iteration"""
    from rayopt_b200 import optimize as opt
    from rayopt_b200.surface_table import pack_system
    s = reference_system("cooke")
    t = pack_system(s, s.wavelengths[0], 1, None)[0]
    params = [(j, "curvature") for j in range(1, len(t) + 1) if t["c"][j - 1] != 0][:6]
    params.append((len(t), "distance"))
    kw = dict(heights=(0., .7, 1.), nrays=10000, engine=eng)
    opt.optimize_spot(s, params, iterations=1, **kw)           # warm-up
    aims, whole = [], []
    for _ in range(3):
        t0 = time.perf_counter()
        B = opt._Bundles(s, kw["heights"], list(s.wavelengths), kw["nrays"], "hexapolar", eng,
                         False)
        eng.sync()
        aims.append(1e3*(time.perf_counter() - t0))
        B.close()
        t0 = time.perf_counter()
        opt.optimize_spot(s, params, iterations=1, **kw)
        whole.append(1e3*(time.perf_counter() - t0))
    # an iteration aims twice: for its Jacobian and for the re-aimed merit after it
    line = dict(what="optimize_spot iteration, Cooke, P=7, 9 bundles x 1e4 rays",
                aim_ms=med(aims), iteration_ms=med(whole), gpu=gpu)
    print(json.dumps(line), flush=True)
    return line


if __name__ == "__main__":
    main()
