#!/usr/bin/env python
"""Kernel and host times of the device tolerance analysis
(rtx_trace_reduce_many) in one run.

    python scripts/tolerance_timing.py [--variants 1 64 1024 4096] [--nrays 1e3 1e4]
                                       [--reps 5] [--out FILE]

Workload: the Double-Gauss lens (tests/golden/systems.json), V perturbed
variants (curvature, spacing, conic and tilt deltas), 3 field heights (0,
0.7, 1) x 3 wavelengths, one bundle of launch rays per height and
wavelength shared by all variants, clip=True, FP64 fast mode.  For each V and
bundle size it prints one JSON line with the median and range of the kernel
time (CUDA events around both kernels), the ray-surfaces per second, the
host setup time (perturbed tables and items) and, as the reference arm, the
numpy trace (oracle/np_oracle.py) of 8 variants in ms per variant, with the
card's name and power limit read in the same run.
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
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)

PARAMS = [(1, "curvature"), (2, "distance"), (4, "conic"), (6, "tilt_x")]
TOL = [1e-4, 1e-2, 1e-2, 1e-3]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--variants", type=int, nargs="+", default=[1, 64, 1024, 4096])
    ap.add_argument("--nrays", type=float, nargs="+", default=[1e3, 1e4])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out")
    a = ap.parse_args()
    np.seterr(all="ignore")
    from conftest import load_systems
    from rayopt_b200.engine import Engine
    from rayopt_b200.rays import aim_infinite, disc
    from rayopt_b200.tolerance import monte_carlo_deltas, perturbed_tables
    import np_oracle
    eng = Engine(0)
    gpu = card()
    ent = load_systems()["double_gauss"]
    nominal = np.stack(ent["tables"][:3])
    W, S = nominal.shape
    H = 3
    lines = []
    for nr in a.nrays:
        N = int(nr)
        host = []
        for h, fi in enumerate((0, 3, 5)):
            for w in range(W):
                aim = ent["aim"][w][fi]
                host.append(aim_infinite(aim["field"], disc(N, 3*h + w), aim["z"], aim["p"],
                                         ent["object_angle"]))
        bundles = [(eng.to_device(y), eng.to_device(u), N) for y, u in host]
        for V in a.variants:
            deltas = monte_carlo_deltas(TOL, V, seed=1)
            t0 = time.perf_counter()
            t = perturbed_tables(nominal, PARAMS, deltas).reshape(V*W, S)
            vv, hh, ww = np.meshgrid(np.arange(V), np.arange(H), np.arange(W), indexing="ij")
            items = np.stack([vv*W + ww, hh*W + ww], -1).reshape(-1, 2)
            setup = 1e3*(time.perf_counter() - t0)
            eng.trace_reduce_many(t, bundles, items, clip=True)            # warm-up
            ks, calls = [], []
            for _ in range(a.reps):
                c0 = time.perf_counter()
                eng.trace_reduce_many(t, bundles, items, clip=True)
                calls.append(1e3*(time.perf_counter() - c0))
                ks.append(eng.last_kernel_ms())
            km = statistics.median(ks)
            lines.append(dict(workload="double_gauss", variants=V, heights=H, wavelengths=W,
                              rays_per_bundle=N, surfaces=S, kernel_ms=km,
                              kernel_ms_range=[min(ks), max(ks)],
                              call_ms=statistics.median(calls),
                              ray_surfaces_per_s=V*H*W*N*S/(km*1e-3), host_setup_ms=setup,
                              gpu=gpu))
            print(json.dumps(lines[-1]), flush=True)
        # the reference arm: numpy traces of 8 variants, every bundle
        t8 = perturbed_tables(nominal, PARAMS, monte_carlo_deltas(TOL, 8, seed=1))
        c0 = time.perf_counter()
        for v in range(8):
            for b, (y, u) in enumerate(host):
                np_oracle.trace(t8[v, b % W], y, u, clip=True)
        lines.append(dict(workload="double_gauss", arm="numpy", rays_per_bundle=N,
                          ms_per_variant=1e3*(time.perf_counter() - c0)/8, gpu=gpu))
        print(json.dumps(lines[-1]), flush=True)
        for y, u, _ in bundles:
            y.free(), u.free()
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(json.dumps(x) for x in lines) + "\n")


if __name__ == "__main__":
    main()
