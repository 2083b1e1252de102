#!/usr/bin/env python
"""Kernel and call times of the Zernike decomposition on the device
(rayopt_b200.tolerance_zernike and zernike, rtx_trace_zernike_many), next to
the march alone (rtx_trace_opd_many through tolerance_wavefront on the same
lens, bundles and deltas) and a numpy least-squares fit of downloaded
per-ray values, in one run.

    python scripts/zernike_timing.py [--orders 1 4 6 8] [--variants 1 64 1024 4096]
                                     [--nrays 1e3 1e4] [--big 1e5 1e6] [--reps 3] [--out FILE]

Workload: the reference's Double-Gauss lens (the staged reference tree), V
Monte Carlo variants of the curvatures of the first two surfaces and the
spacing of the second, 3 field heights x 3 wavelengths, hexapolar bundles,
clip=True, FP64 fast mode.  Each JSON line has the median and range over
`reps` runs after a warm-up of the whole call (aiming, the chief-ray
launches and the nominal order-0 launch included) and of the two-kernel
time of its last rtx_trace_zernike_many launch (CUDA events; with more than
one chunk, the last chunk's), and the same two numbers of
tolerance_wavefront, whose last launch is rtx_trace_opd_many on the same
items: the difference of the kernel times is the Gram's cost over the
march.  Then zernike() of the nominal lens at `--big` rays per bundle, and
the host fit: the nominal lens's per-ray (a, x, y) of the 9 bundles
downloaded from rtx_trace_opd, the closed-form basis and
numpy.linalg.lstsq, timed per variant.  The card's name and power limit
are read in the same run.
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


def timed(eng, fn, reps):
    call, kern = [], []
    for r in range(reps + 1):
        t0 = time.perf_counter()
        res = fn()
        t1 = time.perf_counter()
        if r:                                                  # the first run is the warm-up
            call.append(1e3*(t1 - t0))
            kern.append(eng.last_kernel_ms())
    return res, stats(call), stats(kern)


def host_fit(eng, s0, N, order):
    """the nominal lens's per-ray values of the 9 bundles, fitted on the
    host: (seconds of basis + lstsq per variant, seconds of the downloads,
    largest |c_host - c_device| in waves)"""
    from rayopt_b200.tolerance import _nominal, _WavefrontRef, launch_bundles, perturbed_tables
    from rayopt_b200.zernike import nterms, tolerance_zernike, zernike_basis
    J = nterms(order)
    W = len(s0.wavelengths)
    s = copy.deepcopy(s0)
    dev = tolerance_zernike(copy.deepcopy(s0), [], np.zeros((1, 0)), HEIGHTS, nrays=N,
                            order=order, engine=eng)
    nominal, rot0 = _nominal(s, s.wavelengths)
    bundles, chiefs = launch_bundles(s, HEIGHTS, s.wavelengths, N, "hexapolar", eng)
    ref = _WavefrontRef(s, nominal, s.wavelengths, chiefs)
    fit_s, dl_s, worst = 0., 0., 0.
    try:
        ref.upload(eng)
        march, items, specs, a0, cen, ok = ref.chief(eng, perturbed_tables(nominal, [],
                                                                           np.zeros((1, 0))),
                                                     rot0, False)
        for b, (y, u) in enumerate(bundles):
            n = y.shape[0]
            A, P = eng.empty((n,)), eng.empty((n, 3))
            t0 = time.perf_counter()
            eng.trace_opd(march[b % W], y, u, specs[b], A, P, N=n, clip=True, rot0=rot0)
            eng.sync()
            a, p = A.download() - a0[b], P.download()
            dl_s += time.perf_counter() - t0
            A.free(), P.free()
            t0 = time.perf_counter()
            x, yy = p[:, 0] - cen[b, 0], p[:, 1] - cen[b, 1]
            m = np.isfinite(a) & np.isfinite(x) & np.isfinite(yy)
            rho = dev["radius"].reshape(-1)[b]
            Z = zernike_basis(J, x[m]/rho, yy[m]/rho)
            c = np.linalg.lstsq(Z, a[m], rcond=None)[0]
            fit_s += time.perf_counter() - t0
            lam = s.wavelengths[b % W]/s.scale
            worst = max(worst, float(np.abs(-c/lam - dev["coefficients"][0].reshape(-1, J)[b]).max()))
    finally:
        for y, u in bundles:
            y.free(), u.free()
        ref.free()
    return fit_s, dl_s, worst


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--orders", type=int, nargs="+", default=[1, 4, 6, 8])
    ap.add_argument("--variants", type=int, nargs="+", default=[1, 64, 1024, 4096])
    ap.add_argument("--nrays", type=float, nargs="+", default=[1e3, 1e4])
    ap.add_argument("--big", type=float, nargs="+", default=[1e5, 1e6])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out")
    a = ap.parse_args()
    warnings.simplefilter("ignore")
    np.seterr(all="ignore")
    from rayopt_b200.engine import Engine
    from rayopt_b200.tolerance import monte_carlo_deltas, tolerance_wavefront
    from rayopt_b200.zernike import tolerance_zernike, zernike
    eng = Engine(0)
    gpu = card()
    lines = []

    def emit(rec):
        rec = dict(card=gpu, lens="double_gauss", **rec)
        lines.append(json.dumps(rec))
        print(lines[-1], flush=True)
    s0 = lens("double_gauss")
    params = [(1, "curvature"), (2, "curvature"), (2, "distance")]
    tol = [1e-4, 1e-4, 1e-2]
    for nr in a.nrays:
        N = int(nr)
        for V in a.variants:
            deltas = monte_carlo_deltas(tol, V, seed=V)
            _, wc, wk = timed(eng, lambda: tolerance_wavefront(copy.deepcopy(s0), params, deltas,
                                                               HEIGHTS, nrays=N, engine=eng),
                              a.reps)
            for order in a.orders:
                _, zc, zk = timed(eng, lambda: tolerance_zernike(
                    copy.deepcopy(s0), params, deltas, HEIGHTS, nrays=N, order=order,
                    engine=eng), a.reps)
                emit(dict(nrays=N, variants=V, order=order, bundles=9, zernike_call_ms=zc,
                          zernike_kernel_ms=zk, wavefront_call_ms=wc, opd_many_kernel_ms=wk,
                          kernel_ratio=zk["median"]/wk["median"]))
    for nr in a.big:
        N = int(nr)
        for order in a.orders:
            _, zc, zk = timed(eng, lambda: zernike(copy.deepcopy(s0), HEIGHTS, nrays=N,
                                                   order=order, engine=eng), a.reps)
            emit(dict(nrays=N, variants="zernike()", order=order, bundles=9, call_ms=zc,
                      kernel_ms=zk))
    for nr in a.nrays:
        for order in a.orders:
            fit_s, dl_s, worst = host_fit(eng, s0, int(nr), order)
            emit(dict(nrays=int(nr), order=order, bundles=9,
                      host_fit_ms_per_variant=1e3*fit_s, download_ms_per_variant=1e3*dl_s,
                      max_coefficient_diff_waves=worst))
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")
    eng.close()


if __name__ == "__main__":
    main()
