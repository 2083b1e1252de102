#!/usr/bin/env python
"""Times of the device MTF derivatives (rtx_otf_jacobian_sums) next to the
march that feeds them (rtx_trace_jacobian), and of one optimize_mtf
iteration.

    python scripts/mtf_jacobian_timing.py [--params 4 20 40] [--freqs 8 64]
                                          [--nrays 1e4 1e6] [--reps 5] [--out FILE]

Workload: the Double-Gauss lens (tests/golden/systems.json), 3 field heights
(0, 0.7, 1) x 3 wavelengths, P parameters (curvatures, distances and conics
of its curved surfaces, then other distances and aspherics), clip on, FP64
fast mode, F frequencies spread over 0 .. 100 cycles per length unit, about
each bundle's first ray.  The launch rays are generated on the host
(aim_infinite of a disc).  For each P, F and bundle size it prints one JSON
line: the median kernel ms (CUDA events) of each call summed over the 9
bundles, the terms (rays x 2F x P) per second of the sums, the share of the
data-sheet FP64 rate that 2 FMA per term and one sincospi per ray, unit and
block of 8 parameters would need (sincospi counted as 40 FP64 operations,
a rough figure of its polynomial and reduction), and the card's name and
power limit read in the same run.  With the reference staged, one
optimize_mtf iteration of the Cooke triplet (six curvatures and the image
distance, 1e4 rays per bundle, F = 8) is split into host aiming and the rest.
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

FP64_PEAK = 67e12        # H100 SXM data sheet, FP64 vector FLOP/s at 700 W
SINCOSPI_FLOP = 40       # assumed cost of one FP64 sincospi in FLOP
PB = 8                   # parameters per sincospi (OTF_JAC_PB in rtx_device.cuh)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--params", type=int, nargs="+", default=[4, 20, 40])
    ap.add_argument("--freqs", type=int, nargs="+", default=[8, 64])
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
    cands = ([(j, k) for k in ("curvature", "distance", "conic") for j in curved]
             + [(j, "distance") for j in range(1, S) if j not in curved]
             + [(j, x) for x in ("asph0", "asph1") for j in curved])
    lines = []
    for nr in a.nrays:
        n = int(nr)
        bundles = []
        for li in range(W):
            for h in range(3):
                aim = ent["aim"][li][h]
                y0, u0 = aim_infinite(aim["field"], disc(n, 10*li + h)*.95, aim["z"], aim["p"],
                                      ent["object_angle"])
                bundles.append((li, eng.to_device(y0), eng.to_device(u0)))
        for P in a.params:
            moves = record_tangents(nominal, cands[:P])
            for F in a.freqs:
                nu = np.linspace(0., 100., F)
                t = {k: [] for k in ("trace_jacobian", "otf_jacobian_sums")}
                n_in = 0
                for rep in range(a.reps + 1):                 # rep 0 warms up
                    acc = dict.fromkeys(t, 0.)
                    n_in = 0
                    for li, y0, u0 in bundles:
                        mv = [[(r, rec[li]) for r, rec in m] for m in moves]
                        q, J = eng.trace_jacobian(nominal[li], y0, u0, mv, clip=True)
                        eng.sync()
                        acc["trace_jacobian"] += eng.last_kernel_ms()
                        c = q.rows(0, 1).download()[0]
                        s = eng.otf_jacobian_sums(q, J, nu, c if np.isfinite(c).all() else None)
                        acc["otf_jacobian_sums"] += eng.last_kernel_ms()
                        n_in += s["n"]
                        q.free(), J.free()
                    if rep:
                        for k in t:
                            t[k].append(acc[k])
                ms = statistics.median(t["otf_jacobian_sums"])
                terms = n_in*2*F*P
                flop = terms*4 + n_in*2*F*-(-P//PB)*SINCOSPI_FLOP
                line = dict(P=P, F=F, nrays_per_bundle=n, bundles=len(bundles),
                            rays_entering=int(n_in),
                            **{k + "_kernel_ms": statistics.median(v) for k, v in t.items()},
                            terms_per_s=terms/(ms*1e-3),
                            fp64_share=flop/(ms*1e-3)/FP64_PEAK, gpu=gpu)
                print(json.dumps(line), flush=True)
                lines.append(line)
        for _, y, u in bundles:
            y.free(), u.free()
    import ref_shim
    if ref_shim.available():
        lines.append(optimize_iteration(eng, gpu))
    if a.out:
        with open(a.out, "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")
    eng.close()


def optimize_iteration(eng, gpu):
    """one optimize_mtf iteration of the Cooke triplet: host aiming
    (launch_bundles and the chief rays) against the whole iteration"""
    from rayopt_b200 import optimize as opt
    from rayopt_b200.mtf import default_dnu
    from rayopt_b200.surface_table import pack_system
    s = reference_system("cooke")
    t = pack_system(s, s.wavelengths[0], 1, None)[0]
    params = [(j, "curvature") for j in range(1, len(t) + 1) if t["c"][j - 1] != 0][:6]
    params.append((len(t), "distance"))
    nu = np.arange(1, 9)*default_dnu(s, 16)
    kw = dict(heights=(0., .7, 1.), nrays=10000, engine=eng)
    opt.optimize_mtf(s, params, nu, iterations=1, **kw)           # warm-up
    aims, whole = [], []
    for _ in range(3):
        t0 = time.perf_counter()
        B = opt._Bundles(s, kw["heights"], list(s.wavelengths), kw["nrays"], "hexapolar", eng,
                         False)
        eng.sync()
        aims.append(1e3*(time.perf_counter() - t0))
        B.close()
        t0 = time.perf_counter()
        opt.optimize_mtf(s, params, nu, iterations=1, **kw)
        whole.append(1e3*(time.perf_counter() - t0))
    # an iteration aims twice: for its Jacobian and for the re-aimed merit after it
    line = dict(what="optimize_mtf iteration, Cooke, P=7, F=8, 9 bundles x 1e4 rays",
                aim_ms=statistics.median(aims), iteration_ms=statistics.median(whole), gpu=gpu)
    print(json.dumps(line), flush=True)
    return line


if __name__ == "__main__":
    main()
