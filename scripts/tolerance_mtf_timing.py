#!/usr/bin/env python
"""Kernel and host times of the MTF tolerance analysis (rtx_trace_otf_many)
against the per-variant path of the optimiser's trial scorer, in one run.

    python scripts/tolerance_mtf_timing.py [--variants 1 64 1024 4096] [--nrays 1e3 1e4]
                                           [--reps 5] [--out FILE]

Workload: the Double-Gauss lens (tests/golden/systems.json), V perturbed
variants (curvature, spacing, conic and tilt deltas), 3 field heights x 3
wavelengths, one bundle of launch rays per height and wavelength shared by
all variants, clip=True, FP64 fast mode, (K planes, F frequencies) in
{(1, 3), (5, 16)}.  For each case it prints one JSON line: the median and
range of the kernel time (CUDA events around both kernels) and of the whole
call over `reps` runs after a warm-up, and the host setup time (perturbed
tables and items).  At V = 64 and 1024 it also times optimize._trial_mtf
(keep-LAST batched marches, then one rtx_otf_jacobian_sums per bundle) on
the same bundles and deltas and checks that both polychromatic MTFs agree
within their bounds.  The card's name and power limit are read in the same
run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)

PARAMS = [(1, "curvature"), (2, "distance"), (4, "conic"), (6, "tilt_x")]
TOL = [1e-4, 1e-2, 1e-2, 1e-3]
CASES = [(1, 3), (5, 16)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def stats(x):
    return dict(median=statistics.median(x), min=min(x), max=max(x))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--variants", type=int, nargs="+", default=[1, 64, 1024, 4096])
    ap.add_argument("--nrays", type=float, nargs="+", default=[1e3, 1e4])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out")
    a = ap.parse_args()
    np.seterr(all="ignore")
    from conftest import load_systems
    from rayopt_b200 import optimize as opt
    from rayopt_b200.engine import Engine
    from rayopt_b200.mtf import poly_otf
    from rayopt_b200.rays import aim_infinite, disc
    from rayopt_b200.tolerance import monte_carlo_deltas, perturbed_tables
    eng = Engine(0)
    gpu = card()
    ent = load_systems()["double_gauss"]
    nominal = np.stack(ent["tables"][:3])
    W, S = nominal.shape
    H = 3
    sw = np.ones(W)
    lines = []
    for nr in a.nrays:
        N = int(nr)
        rays = []
        for h in range(H):
            for w in range(W):
                aim = ent["aim"][w][(0, 3, 5)[h]]
                y, u = aim_infinite(aim["field"], disc(N, 3*h + w), aim["z"], aim["p"],
                                    ent["object_angle"])
                rays.append((eng.to_device(y), eng.to_device(u)))
        centers = np.zeros((H*W, 4))
        for h in range(H):                              # the height's first ray at wavelength 0
            y, u = rays[h*W]
            Y = eng.trace(nominal[0], y.download()[:1], u.download()[:1], clip=True,
                          keep_last=True, want=("y",))[0]
            if np.isfinite(Y[0, 0, :2]).all():
                centers[h*W:(h + 1)*W, :2] = Y[0, 0, :2]
        B = types.SimpleNamespace(nominal=nominal, rot0=None, W=W, rays=rays, centers=centers)
        dev = [(y, u, None) for y, u in rays]
        for V in a.variants:
            deltas = monte_carlo_deltas(TOL, V, seed=V)
            for K, F in CASES:
                z = np.linspace(-1e-2, 1e-2, K) if K > 1 else np.zeros(1)
                nu = np.linspace(10., 50., F)
                setup, call, kern = [], [], []
                for r in range(a.reps + 1):
                    t0 = time.perf_counter()
                    t = perturbed_tables(nominal, PARAMS, deltas).reshape(V*W, S)
                    vv, hh, ww = np.meshgrid(np.arange(V), np.arange(H), np.arange(W),
                                             indexing="ij")
                    items = np.stack([vv*W + ww, hh*W + ww], -1).reshape(-1, 2)
                    c = centers[(hh*W).reshape(-1), :2]
                    t1 = time.perf_counter()
                    s, n = eng.trace_otf_many(t, dev, items, c, z, nu, clip=True)
                    t2 = time.perf_counter()
                    if r:                                # the first run is the warm-up
                        setup.append(1e3*(t1 - t0))
                        call.append(1e3*(t2 - t1))
                        kern.append(eng.last_kernel_ms())
                terms = float(n.sum())*2*F
                rec = dict(card=gpu, nrays=N, variants=V, K=K, F=F, kernel_ms=stats(kern),
                           call_ms=stats(call), setup_ms=stats(setup),
                           terms_per_s=terms/(statistics.median(kern)*1e-3))
                if V in (64, 1024) and K == 1:
                    with np.errstate(all="ignore"):
                        otf = s.reshape(V, H, W, K, 2, F)/n.reshape(V, H, W, K)[..., None, None]
                    poly = np.abs(poly_otf(otf.reshape(V*H, W, K, 2, F),
                                           n.reshape(V*H, W, K), sw)).reshape(V, H, 2, F)
                    trial = []
                    for r in range(4):
                        t0 = time.perf_counter()
                        M = opt._trial_mtf(eng, B, PARAMS, deltas, nu, sw, True, False)
                        if r:
                            trial.append(1e3*(time.perf_counter() - t0))
                    # both sums are within (D + 4 Phi + 3) eps n of the exact one
                    # (D <= 532, Phi < 1e3 here): 1e-11 of the MTF covers both
                    diff = float(np.nanmax(np.abs(poly - M)))
                    assert np.array_equal(np.isnan(poly), np.isnan(M)) and diff <= 1e-11, diff
                    rec.update(trial_call_ms=stats(trial), max_poly_mtf_diff=diff,
                               speedup=statistics.median(trial)/statistics.median(call))
                lines.append(json.dumps(rec))
                print(lines[-1], flush=True)
        for y, u in rays:
            y.free(), u.free()
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")
    eng.close()


if __name__ == "__main__":
    main()
