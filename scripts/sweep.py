#!/usr/bin/env python
"""Tuning sweep of the trace kernel on the C2 workload (one wavelength bundle
per launch, 1e7 rays, S=12, FP64): env knobs RTX_RPT / RTX_WARPS / RTX_LOCK /
RTX_MAX_CTAS / RTX_TUNE / RTX_CLUSTER are read by rtx_init, so one Engine per
configuration.  RTX_MAX_CLUSTERS (resident clusters of the clustered kernel,
0: all that fit) is taken from the environment as set.
usage: python scripts/sweep.py [--rays N] [--exact 0|1] cfg1 cfg2 ...
       cfg = rpt,store,warps,nbuf,lock,maxctas[,tune[,cluster]]   e.g. 2,1,8,2,1,0
       (store 1: per-warp bulk stores, 2: per-CTA bulk stores; tune: RTX_TUNE,
       of which only bit 1 (value 2: no input L2 prefetch) is read -- the bulk
       stores always take the L2 evict_first policy; cluster: CTAs per
       thread-block cluster of the per-CTA store kernel, 1: none)
Build with RTX_TUNING_SPACE=1 for the full variant space."""
import argparse, os, statistics, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench
from rayopt_b200.engine import Engine

ap = argparse.ArgumentParser()
ap.add_argument("--rays", type=int, default=10_000_000)
ap.add_argument("--exact", type=int, default=0)
ap.add_argument("--system", default="double_gauss")
ap.add_argument("--dtype", default="f64")
ap.add_argument("--device-rays", type=int, default=0,
                help="1: hexapolar launch rays generated in HBM (large bundles)")
ap.add_argument("--keep-last", type=int, default=0, help="1: store the last surface only (compute-bound)")
ap.add_argument("--pad", type=int, default=0, help="extra rays of row pitch (ld = N rounded + pad)")
ap.add_argument("--gap", type=int, default=0, help="bytes of dummy allocation between the result arrays")
ap.add_argument("cfgs", nargs="*", default=["2,2,16,1,0,0,1"])
a = ap.parse_args()
ent = bench.load_system(a.system)
S, N = ent["S"], a.rays
dt = np.float64 if a.dtype == "f64" else np.float32
w = np.dtype(dt).itemsize
mem = Engine(0)
if a.device_rays:
    aim = ent["aim"][0][bench.FIELD_INDEX]
    d_y0, d_u0 = mem.aim_infinite_device(aim["field"], aim["z"], aim["p"], ent["object_angle"],
                                         nrays=N, dtype=dt)
    N = d_y0.shape[0]//128*128
else:
    y0, u0 = bench.make_rays(ent, 0, N, 0)
    d_y0, d_u0 = mem.to_device(y0, dt), mem.to_device(u0, dt)
ld = ((N + 127)//128)*128 + a.pad
gaps = []
def _arr(shape):
    if a.gap:
        gaps.append(mem.empty((a.gap,), np.uint8))
    return mem.empty(shape, dt)
Y, U, I = (_arr((S, ld, 3)) for _ in range(3))
T = _arr((S, ld))
print("ld %d pad %d gap %d  bases %s" % (ld, a.pad, a.gap, [hex(x.ptr) for x in (Y, U, I, T)]), flush=True)
alg = N*(6*w + 10*w*S)
peak_gbs, peak_src = bench.peaks()
print("frac: algorithmic GB/s over %.1f GB/s (%s)" % (peak_gbs, peak_src), flush=True)
for cfg in a.cfgs:
    if cfg == "default":          # the library's own heuristics (no RTX_* knob set)
        for k in ("RTX_RPT", "RTX_STORE", "RTX_WARPS", "RTX_NBUF", "RTX_LOCK", "RTX_MAX_CTAS", "RTX_TUNE",
                  "RTX_CLUSTER"):
            os.environ.pop(k, None)
        parts = [0, 0, 0, 0, 0, 0, -1, 0]
    else:
        parts = [int(x) for x in cfg.split(",")]
    rpt, store, warps, nbuf, lock, maxc = parts[:6]
    tune = parts[6] if len(parts) > 6 else 0
    cluster = parts[7] if len(parts) > 7 else 1
    if cfg != "default":
        os.environ["RTX_TUNE"] = str(tune)
        os.environ["RTX_CLUSTER"] = str(cluster)
        os.environ.update(RTX_RPT=str(rpt), RTX_STORE=str(store), RTX_WARPS=str(warps),
                      RTX_NBUF=str(nbuf), RTX_LOCK=str(lock), RTX_MAX_CTAS=str(maxc))
    e = Engine(0)
    ms = []
    try:
        e.trace_device(ent["tables"][0], d_y0, d_u0, Y, U, I, T, N=N, ld=ld, clip=True, exact=bool(a.exact), keep_last=bool(a.keep_last))
    except Exception as ex:
        print("cfg %s: %s" % (cfg, ex), flush=True)
        e.close()
        continue
    for i in range(12):
        e.trace_device(ent["tables"][0], d_y0, d_u0, Y, U, I, T, N=N, ld=ld, clip=True, exact=bool(a.exact), keep_last=bool(a.keep_last))
        t = e.last_kernel_ms()
        ctas = e.last_launch_ctas()
        if i >= 4:
            ms.append(t)
    m = statistics.median(ms)
    print("tune %d rpt %d store %d warps %2d nbuf %d lock %d maxctas %d cluster %d ctas %3d exact %d %s %s: %7.3f ms (min %.3f)  %7.1f GB/s  %.3e ray-surf/s  frac %.3f" % (
        tune, rpt, store, warps, nbuf, lock, maxc, cluster, ctas, a.exact, a.dtype, a.system, m, min(ms), alg/m/1e6, N*S/m*1e3, alg/m/1e6/peak_gbs), flush=True)
    e.close()
