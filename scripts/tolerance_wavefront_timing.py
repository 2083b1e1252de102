#!/usr/bin/env python
"""Kernel and call times of the wavefront tolerance analysis
(rayopt_b200.tolerance_wavefront, rtx_trace_opd_many) against the per-variant
trial scorer of optimize_wavefront (optimize._wavefront_merits), in one run.

    python scripts/tolerance_wavefront_timing.py [--variants 64 1024] [--nrays 1e4]
                                                 [--reps 3] [--out FILE]

Workload: the reference's Cooke triplet and Double-Gauss lens (the staged
reference tree), V Monte Carlo variants of the curvatures of the first two
surfaces and the spacing of the second, 3 field heights x 3 wavelengths,
hexapolar bundles, clip=True, FP64 fast mode.  For each case it prints one
JSON line: the median and range over `reps` runs after a warm-up of the
whole tolerance_wavefront call (three launches per chunk, aiming included)
and of the kernel time of its full-bundle rtx_trace_opd_many launch (CUDA
events around both kernels); then _wavefront_merits on the same deltas (one
rtx_trace_reduce_many launch, then one rtx_trace_opd and one
rtx_wavefront_sums launch and host sync per variant and bundle), the ratio
of the two call times and the largest relative difference of the merit
sum_b rms_b^2.  The card's name and power limit are read in the same run.
"""
import argparse
import copy
import json
import os
import statistics
import subprocess
import sys
import time
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests"),
          os.path.join(ROOT, "tests", "golden")):
    sys.path.insert(0, p)

HEIGHTS = (0., .707, 1.)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def stats(x):
    return dict(median=statistics.median(x), min=min(x), max=max(x))


def lens(name):
    import yaml
    import ref_shim
    import systems_yaml
    R = ref_shim.load()
    s = R.System(**yaml.safe_load(systems_yaml.SYSTEMS[name]))
    s.update()
    s.paraxial.refocus()
    return s


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--variants", type=int, nargs="+", default=[64, 1024])
    ap.add_argument("--nrays", type=float, nargs="+", default=[1e4])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out")
    a = ap.parse_args()
    warnings.simplefilter("ignore")
    np.seterr(all="ignore")
    from rayopt_b200 import optimize as opt
    from rayopt_b200.engine import Engine
    from rayopt_b200.tolerance import monte_carlo_deltas, tolerance_wavefront
    eng = Engine(0)
    gpu = card()
    lines = []
    for name in ("cooke", "double_gauss"):
        s0 = lens(name)
        params = [(1, "curvature"), (2, "curvature"), (2, "distance")]
        tol = [1e-4, 1e-4, 1e-2]
        W = len(s0.wavelengths)
        for nr in a.nrays:
            N = int(nr)
            for V in a.variants:
                deltas = monte_carlo_deltas(tol, V, seed=V)
                call, kern = [], []
                for r in range(a.reps + 1):
                    s = copy.deepcopy(s0)
                    t0 = time.perf_counter()
                    res = tolerance_wavefront(s, params, deltas, HEIGHTS, nrays=N, engine=eng)
                    t1 = time.perf_counter()
                    if r:                                # the first run is the warm-up
                        call.append(1e3*(t1 - t0))
                        kern.append(eng.last_kernel_ms())
                merit = (res["rms"]**2).sum((1, 2))
                sb = copy.deepcopy(s0)
                B = opt._Bundles(sb, HEIGHTS, sb.wavelengths, N, "hexapolar", eng, False)
                st = opt._Wavefront(eng, sb, B, HEIGHTS, None, None, True, False)
                trial = []
                try:
                    for r in range(2):
                        t0 = time.perf_counter()
                        m = opt._wavefront_merits(eng, B, st, params, deltas, np.ones(3*W), True,
                                                  False)
                        if r:
                            trial.append(1e3*(time.perf_counter() - t0))
                finally:
                    st.close()
                    B.close()
                diff = float(np.nanmax(np.abs(merit - m)/m))
                rec = dict(card=gpu, lens=name, nrays=N, variants=V,
                           bundles=3*W, call_ms=stats(call), kernel_ms=stats(kern),
                           trial_call_ms=stats(trial),
                           speedup=statistics.median(trial)/statistics.median(call),
                           max_merit_rel_diff=diff,
                           median_rms_waves=float(np.nanmedian(res["rms"])),
                           median_rms_tilt_waves=float(np.nanmedian(res["rms_tilt"])))
                lines.append(json.dumps(rec))
                print(lines[-1], flush=True)
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")
    eng.close()


if __name__ == "__main__":
    main()
