#!/usr/bin/env python
"""North-star headline point: zoom fixture, 3e7 rays x 20 surfaces, FP64, full
trace device-resident on ONE 80 GB H100 (49.4 GB of algorithmic traffic per
launch, 48 GB of results in HBM).  The 3e7-ray bundle is three copies of a
1e7-ray aimed bundle (synthetic; distinct seeds per copy would only change
the host generation time)."""
import json, os, statistics, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "oracle"))
import bench, np_oracle
from rayopt_b200.engine import Engine
from rayopt_b200._lib import check, ptr

N1, COPIES = 10_000_000, int(os.environ.get("HEADLINE_COPIES", "3"))
exact = int(os.environ.get("HEADLINE_EXACT", "0"))
ent = bench.load_system("zoom")
S, N = ent["S"], N1*COPIES
eng = Engine(0)
y0, u0 = bench.make_rays(ent, 0, N1, 0)
ld = ((N + 63)//64)*64
print("free HBM %.1f GB, need %.1f GB" % (eng.free_bytes()/1e9, (N*48 + S*ld*80)/1e9), flush=True)
d_y0, d_u0 = eng.empty((N, 3)), eng.empty((N, 3))
for c in range(COPIES):
    for d, h in ((d_y0, y0), (d_u0, u0)):
        check(eng.lib.rtx_memcpy_h2d(eng.ctx, d.ptr + c*N1*24, ptr(h), h.nbytes))
eng.sync()
Y, U, I = (eng.empty((S, ld, 3)) for _ in range(3))
T = eng.empty((S, ld))
ms = []
for i in range(5):
    eng.trace_device(ent["tables"][0], d_y0, d_u0, Y, U, I, T, N=N, ld=ld, clip=True, exact=bool(exact))
    ms.append(eng.last_kernel_ms())
m = statistics.median(ms[1:])
alg = N*(48 + 80*S)
peak, src = bench.peaks()
idx = np.arange(0, N1, 5003)
want = np_oracle.trace(ent["tables"][0], y0[idx], u0[idx], clip=True)
got = np.stack([Y.rows(j).download()[0][(COPIES - 1)*N1 + idx] for j in range(S)])
err = float(np.nanmax(np.abs(got - want[0])/np.maximum(np.abs(want[0]), 1.0)))
print(json.dumps({"workload": "zoom S=20, N=%d rays, FP64, full trace resident (%.1f GB)" % (N, alg/1e9),
                  "kernel_ms": m, "all_ms": ms, "ray_surfaces_per_s": N*S/m*1e3,
                  "achieved_GBps": alg/m/1e6, "peak_GBps": peak, "frac": alg/m/1e6/peak,
                  "arithmetic": "exact" if exact else "fast",
                  "parity_sample": {"n": len(idx), "nan_mask_equal": bool(np.array_equal(np.isnan(got), np.isnan(want[0]))),
                                    "max_rel_err_y": err}}))
