#!/usr/bin/env python
"""Times of the geometric MTF (rtx_otf_rows, rayopt_b200.geometric_mtf) and
of the march that feeds it, in one run.

    python scripts/mtf_timing.py [--nrays 1e7 1e8] [--reps 5] [--out FILE]

Workload: the Double-Gauss lens (the reference's System, staged under
oracle/_ref), field 0.7, the first wavelength, hexapolar launch rays
generated in HBM, clip=True, K = 5 planes (Analysis's through-focus planes,
(arange(5) - 2) * rayleigh_range), F in {64, 256} frequencies up to
1/airy_radius, FP64 and FP32 traces.  For each configuration it prints the
median and range over `reps` calls (after one warm-up) of

* march_ms: the keep-LAST march storing y and i (rtx_trace, CUDA events);
* otf_ms:   rtx_otf_rows on those rows (CUDA events, both kernels);
* mtf_s:    the whole geometric_mtf call (host clock; it ends synchronised),
            aiming, ray generation, march and OTF in chunks of 2^24 rays;

the terms (ray x plane x axis x frequency) per second of rtx_otf_rows and
the share of the data-sheet FP64 (non-tensor) rate of the H100 SXM, 34
TFLOP/s, that 8 flops per term would be.  It also times the long-double
oracle (oracle/otf_oracle.py) at 1e5 rays, K = 5, F = 64 on the host CPU for
scale, and prints the card's name and power limit.
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

FP64_DATASHEET = 34e12     # H100 SXM, FP64 without tensor cores, FLOP/s
FLOPS_PER_TERM = 8


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def stats(v):
    return statistics.median(v), (min(v), max(v))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nrays", type=float, nargs="+", default=[1e7, 1e8])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out")
    a = ap.parse_args()
    import yaml
    import ref_shim
    import systems_yaml
    import otf_oracle
    from rayopt_b200 import geometric_mtf
    from rayopt_b200.engine import Engine, otf_spec
    from rayopt_b200.rays import aim_record, grid_spec
    from rayopt_b200.surface_table import pack_system
    np.seterr(all="ignore")
    warnings.simplefilter("ignore")
    R = ref_shim.load()
    s = R.System(**yaml.safe_load(systems_yaml.SYSTEMS["double_gauss"]))
    s.update()
    s.paraxial.refocus()
    eng = Engine(0)
    print("card: %s (name, power limit)" % card(), flush=True)
    wl, yo, K = s.wavelengths[0], (0, .7), 5
    z = (np.arange(K) - K//2)*s.paraxial.rayleigh_range[1]
    zp, p = s.pupil(yo, l=wl)
    table, _, rot0 = pack_system(s, wl, 1, None, n0=s.refractive_index(wl, 0))
    rows = []
    for nr in [int(v) for v in a.nrays]:
        ref, grid = grid_spec("hexapolar", nr)
        rec = aim_record(s.object, yo, zp, p, grid, False, s[0])
        for dname, dtype in (("f64", np.float64), ("f32", np.float32)):
            y0, u0 = eng.aim_rays(rec, dtype=dtype)
            N = y0.shape[0]
            ld = (N + 63)//64*64
            Y, I = eng.empty((1, ld, 3), dtype), eng.empty((1, ld, 3), dtype)
            cy, cu = eng.aim_rays(rec, first=ref, count=1)      # the chief ray, as geometric_mtf
            c = eng.trace(table, cy.download(), cu.download(), clip=True, rot0=rot0,
                          keep_last=True, want=("y",))[0][0, 0, :2]
            cy.free(), cu.free()
            t_march = []
            for r in range(a.reps + 1):
                eng.trace_device(table, y0, u0, Y, None, I, None, N=N, ld=ld, clip=True,
                                 keep_last=True, rot0=rot0)
                eng.sync()
                if r:
                    t_march.append(eng.last_kernel_ms())
            for F in (64, 256):
                dnu = 1/s.paraxial.airy_radius[1]/(F - 1)
                spec = otf_spec(z, dnu, F, c)
                t_otf, t_mtf = [], []
                for r in range(a.reps + 1):
                    S, count = eng.otf_rows(Y.rows(0), I.rows(0), spec, N=N)
                    if r:
                        t_otf.append(eng.last_kernel_ms())
                for r in range(a.reps + 1):
                    t0 = time.perf_counter()
                    out = geometric_mtf(s, heights=(.7,), wavelengths=[wl], nrays=nr, defocus=z,
                                        nfreq=F, engine=eng, dtype=dtype)
                    if r:
                        t_mtf.append(time.perf_counter() - t0)
                same = bool(np.array_equal(out["count"][0, 0], count))
                m_otf, r_otf = stats(t_otf)
                terms = N*K*2*F
                row = dict(nrays=N, dtype=dname, K=K, F=F, counted=int(count[0]))
                row["march_ms"], row["march_range"] = stats(t_march)
                row["otf_ms"], row["otf_range"] = m_otf, r_otf
                row["mtf_s"], row["mtf_range"] = stats(t_mtf)
                row["terms_per_s"] = terms/(m_otf*1e-3)
                row["fp64_datasheet_share_at_8_flops_per_term"] = \
                    FLOPS_PER_TERM*row["terms_per_s"]/FP64_DATASHEET
                row["mtf_count_equals_rows"] = same
                rows.append(row)
                print(json.dumps(row), flush=True)
            for d in (y0, u0, Y, I):
                d.free()
    # the host oracle at 1e5 rays for scale
    rec = aim_record(s.object, yo, zp, p, grid_spec("hexapolar", 10**5)[1], False, s[0])
    y0, u0 = eng.aim_rays(rec)
    N = y0.shape[0]
    ld = (N + 63)//64*64
    Y, I = eng.empty((1, ld, 3)), eng.empty((1, ld, 3))
    eng.trace_device(table, y0, u0, Y, None, I, None, N=N, ld=ld, clip=True, keep_last=True,
                     rot0=rot0)
    y, inc = Y.download()[0, :N], I.download()[0, :N]
    c = y[0, :2]
    dnu = 1/s.paraxial.airy_radius[1]/63
    t0 = time.perf_counter()
    otf_oracle.otf(y, inc, c, z, dnu, 64)
    host = dict(host_oracle_rays=N, K=K, F=64, host_oracle_s=time.perf_counter() - t0)
    print(json.dumps(host), flush=True)
    print("%-10s %-4s %4s %10s %10s %10s %12s %8s" % ("rays", "type", "F", "march ms", "otf ms",
                                                     "mtf s", "terms/s", "fp64 %"))
    for r in rows:
        print("%-10d %-4s %4d %10.3f %10.3f %10.3f %12.3e %8.1f" % (
            r["nrays"], r["dtype"], r["F"], r["march_ms"], r["otf_ms"], r["mtf_s"],
            r["terms_per_s"], 100*r["fp64_datasheet_share_at_8_flops_per_term"]))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(dict(card=card(), rows=rows, host=host), f, indent=1)
    eng.close()


if __name__ == "__main__":
    main()
