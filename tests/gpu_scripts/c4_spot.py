#!/usr/bin/env python
"""BASELINE config C4: Double-Gauss, 1e9-ray spot-diagram bundle, FP64,
ray-sharded over the GPUs of one box, last-surface intercepts gathered on
every GPU.  Under torchrun, one rank per GPU:

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 \
        --master-port 29561 tests/gpu_scripts/c4_spot.py [rays_per_rank]

Every rank generates its shard in HBM (rtx_aim_rays, hexapolar pupil grid,
its own field point), marches it through the 12 surfaces and the SAME kernel
bulk-stores y[-1] into the gather buffers of all ranks over NVLink
(rtx_trace_gather) -- no NCCL in the data path.  A sample of a PEER's segment
is checked against the oracle on every rank."""
import json, os, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import torch, torch.distributed as dist
import np_oracle, bench
from rayopt_b200.engine import Engine
from rayopt_b200.rays import aim_infinite
from rayopt_b200.sharding import PeerGather

local = int(os.environ.get("LOCAL_RANK", "0"))
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
rank, world = dist.get_rank(), dist.get_world_size()
eng = Engine(local)
ent = bench.load_system("double_gauss")
S = ent["S"]
n_local = int(sys.argv[1]) if len(sys.argv) > 1 else 125_000_000
n_local = n_local//64*64
fields = [0, 3, 1, 2, 4, 3, 1, 2]                      # indices into the stored aim solutions
aim = ent["aim"][0][fields[rank % 8]]
y0, u0 = eng.aim_infinite_device(aim["field"], aim["z"], aim["p"], ent["object_angle"],
                                 nrays=int(n_local*1.001) + 64)
assert y0.shape[0] >= n_local
pg = PeerGather(eng, dist, n_local*world)
assert pg.b[rank + 1] - pg.b[rank] == n_local
table = ent["tables"][0]


def run():
    eng.trace_gather(table, y0, u0, pg.ptrs, pg.b[rank], N=n_local, clip=True)
    eng.sync()
    dist.barrier()


run()                                                   # warm-up: IPC mappings, peer access
t0 = time.perf_counter()
run()
wall = time.perf_counter() - t0
kms = eng.last_kernel_ms()
t = torch.tensor([kms, wall*1e3], device="cuda")
dist.all_reduce(t, op=dist.ReduceOp.MAX)
kms_max, wall_max = (float(x) for x in t)
# check a sample of the NEXT rank's segment as it arrived in THIS rank's buffer
peer = (rank + 1) % world
aim_p = ent["aim"][0][fields[peer % 8]]
rings = int(np.sqrt((int(n_local*1.001) + 64)/3. - 1/12.) - 1/2.)
idx = np.unique(np.r_[0, np.random.default_rng(rank).integers(1, min(n_local, 3*rings*(rings + 1)), 300)])
i_ring = np.floor((1 + np.sqrt(1 + 4*(idx - 1)/3.))/2).astype(np.int64)
i_ring = np.where(3*i_ring*(i_ring + 1) < idx, i_ring + 1, i_ring)
i_ring = np.where(3*i_ring*(i_ring - 1) >= idx, i_ring - 1, i_ring)
k = idx - 1 - 3*i_ring*(i_ring - 1)
with np.errstate(all="ignore"):
    a = k*(2*np.pi/(6*np.maximum(i_ring, 1)))
    xy = np.c_[np.sin(a)*i_ring/rings, np.cos(a)*i_ring/rings]
xy[idx == 0] = 0
hy, hu = aim_infinite(aim_p["field"], xy, aim_p["z"], aim_p["p"], ent["object_angle"])
want = np_oracle.trace(table, hy, hu, clip=True)[0][-1]
got = np.empty((len(idx), 3))
from rayopt_b200._lib import check, ptr          # 24-byte D2H per sampled ray
for j, ii in enumerate(idx):
    row = np.empty(3)
    check(eng.lib.rtx_memcpy_d2h(eng.ctx, ptr(row), pg.buf.ptr + (pg.b[peer] + int(ii))*24, 24))
    eng.sync()
    got[j] = row
ok = bool(np.array_equal(np.isnan(got), np.isnan(want)) and
          np.nanmax(np.abs(got - want)/np.maximum(np.abs(want), 1.0)) < 1e-10)
res = {"rank": rank, "world": world, "rays_per_rank": n_local, "surfaces": S,
       "kernel_ms_max_over_ranks": kms_max, "wall_ms_max_over_ranks": wall_max,
       "ray_surfaces_per_s_total": world*n_local*S/(kms_max*1e-3),
       "nvlink_bytes_sent_per_rank": (world - 1)*n_local*24,
       "nvlink_GBps_per_rank": (world - 1)*n_local*24/(kms_max*1e-3)/1e9,
       "peer_segment_parity_ok": ok}
print(json.dumps(res), flush=True)
assert ok
pg.close()
dist.barrier()
dist.destroy_process_group()
eng.close()
