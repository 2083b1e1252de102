#!/usr/bin/env python
"""Kernel times of the through-focus spot images (rtx_trace_spot) against the
march alone (rtx_trace_reduce) and the host path, in one run.

    python scripts/spot_timing.py [--nrays 1e7 1e8] [--reps 5] [--out FILE]

Workloads: Double-Gauss (the C2 lens of bench.py), hexapolar launch rays
generated in HBM, clip=True, K = 5 planes, 512 x 512 bins over the default
range (the symmetric range holding every finite point, taken by one
extent-only launch outside the timed calls):

* spread:  field 0.7, planes 0.1 mm apart -- rays over many bins;
* focused: on axis, planes 1 um apart about best focus -- most rays of a warp
  in the same few bins, the worst case for the counter atomics.

For each workload, size and arithmetic (FP64 fast, FP32) it prints the
median and range of the kernel time (CUDA events) of rtx_trace_spot and of
rtx_trace_reduce on the same rays.  At 1e7 rays FP64 it also times the host
path (keep-last trace of y and i, download, np.histogram2d per plane) and
checks that its counts equal the device's.
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


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nrays", type=float, nargs="+", default=[1e7, 1e8])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out")
    a = ap.parse_args()
    np.seterr(all="ignore")
    from conftest import load_systems
    from rayopt_b200.engine import Engine, spot_spec, spot_shape
    from rayopt_b200.spot import default_range
    import spot_oracle
    eng = Engine(0)
    print("card: %s (name, power limit)" % card())
    ent = load_systems()["double_gauss"]
    table = ent["tables"][0]
    K, bins = 5, (512, 512)
    work = {"spread": (3, (np.arange(K) - K//2)*0.1),
            "focused": (0, (np.arange(K) - K//2)*1e-3)}
    rows = []
    for n in [int(v) for v in a.nrays]:
        for wname, (fi, z) in work.items():
            aim = ent["aim"][0][fi]
            for dname, dtype in (("f64", np.float64), ("f32", np.float32)):
                y0, u0 = eng.aim_infinite_device(aim["field"], aim["z"], aim["p"],
                                                 ent["object_angle"], nrays=n, dtype=dtype)
                N = y0.shape[0]
                # the chief ray (ray 0 of the hexapolar grid) at the image
                Y = eng.trace(table, y0.rows(0).download(), u0.rows(0).download(), clip=True,
                              keep_last=True, dtype=dtype, want=("y",))[0]
                c = Y[0, 0, :2].astype(np.float64)
                probe = spot_spec(z, bins, ((-1., 1.), (-1., 1.)), c)
                _, ext = eng.trace_spot(table, y0, u0, probe, None, clip=True, extent=True)
                spec = spot_spec(z, bins, default_range(ext, bins), c)
                counts = eng.empty(spot_shape(spec), np.uint64)
                t_spot, t_red = [], []
                for r in range(a.reps + 1):          # the first of each is a warm-up
                    eng.memset(counts, 0)
                    tally, _ = eng.trace_spot(table, y0, u0, spec, counts, clip=True)
                    if r:
                        t_spot.append(eng.last_kernel_ms())
                    eng.trace_reduce(table, y0, u0, clip=True)
                    if r:
                        t_red.append(eng.last_kernel_ms())
                got = counts.download()
                row = dict(workload=wname, nrays=N, dtype=dname,
                           spot_ms=statistics.median(t_spot), spot_range=(min(t_spot), max(t_spot)),
                           reduce_ms=statistics.median(t_red), reduce_range=(min(t_red), max(t_red)),
                           binned=int(tally[:, 0].sum()), nonfinite=int(tally[:, 1].sum()),
                           peak_bin=int(got.max()))
                if n <= 10**7 and dtype == np.float64:
                    ld = (N + 63)//64*64
                    Yd, Id = eng.empty((1, ld, 3)), eng.empty((1, ld, 3))
                    eng.sync()
                    t0 = time.perf_counter()
                    eng.trace_device(table, y0, u0, Yd, None, Id, None, N=N, ld=ld, clip=True,
                                     keep_last=True)
                    y, inc = Yd.download()[0, :N], Id.download()[0, :N]
                    t1 = time.perf_counter()
                    q = spot_oracle.points(y, inc, c, z)
                    rng = spec[0]["range"]
                    host = np.stack([np.histogram2d(q[k, :, 0], q[k, :, 1], bins=bins,
                                                    range=rng)[0] for k in range(K)])
                    t2 = time.perf_counter()
                    row.update(host_trace_download_s=t1 - t0, host_histogram_s=t2 - t1,
                               host_counts_equal=bool(np.array_equal(host, got)))
                    Yd.free(), Id.free()
                rows.append(row)
                print(json.dumps(row), flush=True)
                for d in (y0, u0, counts):
                    d.free()
    print("%-8s %-10s %-4s %10s %10s %6s %10s %12s" % ("workload", "rays", "type", "spot ms",
                                                     "march ms", "ratio", "host s", "host equal"))
    for r in rows:
        print("%-8s %-10d %-4s %10.3f %10.3f %6.2f %10s %12s" % (
            r["workload"], r["nrays"], r["dtype"], r["spot_ms"], r["reduce_ms"],
            r["spot_ms"]/r["reduce_ms"],
            "%.2f" % (r["host_trace_download_s"] + r["host_histogram_s"])
            if "host_histogram_s" in r else "-", r.get("host_counts_equal", "-")))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(dict(card=card(), rows=rows), f, indent=1)
    eng.close()


if __name__ == "__main__":
    main()
