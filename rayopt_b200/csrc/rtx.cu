// rtx.cu -- C ABI of the ray-trace engine (include/rtx.h): context, memory,
// the table conversion and the kernel launches.  Build:
//   nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -shared \
//        -Xcompiler -fPIC -o librtx.so rtx.cu
#include "../../include/rtx.h"
#include "rtx_device.cuh"
#include "rtx_psf.cuh"
#include "rtx_delaunay.cuh"
#include "rtx_pupil.cuh"

#include <cufft.h>  // types only: the library is opened at run time (rtx_psf)
#include <dlfcn.h>
#include <sched.h>
#include <sys/syscall.h>
#include <unistd.h>

#include <algorithm>
#include <cctype>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <vector>

using namespace rtx;

#define CK(call)                                \
    do {                                        \
        cudaError_t e_ = (call);                \
        if (e_ != cudaSuccess) return (int)e_;  \
    } while (0)

namespace {

constexpr int TABLE_SLOTS = 8;

struct TableSlot {
    void* host = nullptr;  // pinned
    void* dev = nullptr;
    cudaEvent_t done = nullptr;
    bool used = false;
    std::vector<unsigned char> key;  // the rtx_surface bytes + element size this slot holds
};

struct ChunkBuf {
    void* y0 = nullptr;
    void* u0 = nullptr;
    void* Y = nullptr;
    void* U = nullptr;
    void* I = nullptr;
    void* T = nullptr;
    size_t in_bytes = 0, out3_bytes = 0, out1_bytes = 0;
    cudaStream_t stream = nullptr;
};

// the RTX_* environment knobs (rtx_init): experiments that override the
// per-call choice of choose_trace_cfg
struct Tuning {
    bool tuned = false;       // RTX_RPT / RTX_STORE / RTX_WARPS / RTX_NBUF / RTX_CLUSTER was set
    int rpt = 2;              // rays per thread
    int store = STORE_CTA;    // STORE_WARP / STORE_CTA
    int warps = 16;           // warps per CTA
    int nbuf = 1;             // staging buffers per CTA
    int cluster = 1;          // CTAs per cluster of the per-CTA store kernel
    int lockstep = 1;         // CTA barrier per stored surface (STORE_WARP)
    int max_ctas_per_sm = 0;  // 0: whatever fits
    int max_clusters = -1;    // resident clusters of the clustered kernel (-1: MAX_STORE_CLUSTERS, 0: all that fit)
    bool prefetch = true;     // TraceParams::prefetch (RTX_TUNE bit 1 clears it)
};

// A device buffer of the context kept across calls: it grows (reserve) and
// never shrinks.
struct Workspace {
    void* p = nullptr;
    size_t cap = 0;
};

// the context's workspaces (rtx_ctx::ws)
enum {
    WS_MOMENTS,  // rtx_moments, rtx_focus_moments: the 8 sums
    WS_EPI,      // rtx_trace_reduce: the RTX_NMOMENTS sums
    WS_SPOT,     // rtx_trace_spot / rtx_spot_rows: tallies, extents
    WS_AIM,      // rtx_aim_plan: per-block counts, then the offsets of the kept rays
    WS_WINNER,   // rtx_grid_linear: claim grid when the caller wants no winner output
    WS_PSF_RED,  // rtx_psf: partial sums, the finite count and the stats
    WS_PROF,     // rtx_psf_profiles: per-block partial rows, their sum and the pixel flag
    WS_DT,       // rtx_delaunay: slots, adjacency and point-location workspace
    WS_OPD,      // rtx_opd_points: keep flags / ranks, block sums and max(|x|, |y|)
    WS_RANGE,    // rtx_grid_range: count, min key, max key
    WS_MANY,     // rtx_trace_reduce_many: tables, items, tile sums, moments
    WS_OTF,      // rtx_otf_rows: slot sums, then the call's sums and counts
    WS_JAC,      // rtx_trace_jacobian: tangent records, their index, block first rows
    WS_JSUM,     // rtx_jacobian_sums: slot sums, then the call's sums
    WS_OTFJ,     // rtx_otf_jacobian_sums: slot sums, the call's sums, the ray mask
    WS_PUPIL,    // rtx_pupil_sum: slot sums of U, counts and sum w
    WS_PUPIL_RED, // rtx_pupil_intensity: per-block sums, maxima and moments
    WS_COUNT
};

}  // namespace

struct rtx_ctx {
    int device = 0;
    int sm_count = 0;
    cudaStream_t stream = nullptr;
    cudaEvent_t t0 = nullptr, t1 = nullptr;    // rtx_timer_*
    cudaEvent_t k0 = nullptr, k1 = nullptr;    // around the last trace launch
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> chunk_events;
    bool kernel_timed = false;
    TableSlot slots[TABLE_SLOTS];
    int next_slot = 0;
    size_t slot_bytes = 0;
    ChunkBuf chunk[2];
    Workspace ws[WS_COUNT];
    // cached plan of the ray generator (rtx_aim_plan / rtx_aim_rays)
    std::vector<unsigned char> aim_key;
    std::vector<long long> aim_offsets;  // per block; empty: nothing is rejected
    long long aim_total = 0, aim_M = 0;
    // small-bundle latency path (ray aiming: hundreds of 1-3 ray traces)
    void* small_host = nullptr;  // pinned: [y0|u0] in, [Y|U|I|T] out
    void* small_dev = nullptr;
    size_t small_bytes = 0;
    int64_t launches = 0;
    int max_smem_optin = 0;
    Tuning tuning;
    int last_ctas = 0;  // CTAs of the last trace launch (rtx_last_launch_ctas)
    int last_cfg[5] = {0, 0, 0, 0, 0};  // rpt, store, warps, nbuf, cluster (rtx_last_launch_config)
    unsigned* mask = nullptr; // rtx_set_mask_output
    void* tsum = nullptr;     // rtx_set_path_sum_output
    int tsum_upto = 0;
    // rtx_numa_bind: what to restore
    bool numa_bound = false;
    cpu_set_t saved_affinity;
    // rtx_psf: the cuFFT plan of the last (nx, ny) and its work area
    cufftHandle fft_plan = 0;
    bool fft_planned = false;
    long long fft_nx = 0, fft_ny = 0;
    void* fft_work = nullptr;
    size_t fft_work_bytes = 0;
};

namespace {

template <typename T>
void convert_surface(const rtx_surface& s, DevSurf<T>& d) {
    memset(&d, 0, sizeof(d));
    for (int i = 0; i < 3; ++i) d.off[i] = (T)s.offset[i];
    for (int i = 0; i < 9; ++i) d.rot[i] = (T)s.rot[i];
    d.c = (T)s.c;
    d.k1 = (T)(1.0 + s.k);
    d.kc2 = (T)s.kc2;
    d.radius2 = (T)s.radius2;
    d.mu = (T)s.mu;
    d.muf = (T)s.muf;
    d.sgn = (T)s.sgn;
    d.mu2m1 = (T)s.mu2m1;
    d.n0 = (T)s.n0;
    d.inv_c = s.c != 0.0 ? (T)(1.0 / s.c) : (T)0;
    d.kc2k = (T)(s.k * s.c * s.c);
    for (int i = 0; i < RTX_MAX_ASPH; ++i) {
        d.asph[i] = (T)s.asph[i];
        d.dasph[i] = (T)s.dasph[i];
    }
    d.n_asph = s.n_asph;
    unsigned f = 0;
    if (s.flags & RTX_F_ROTATED) f |= DF_ROTATED;
    if (s.flags & RTX_F_ALT) f |= DF_ALT;
    if (s.c == 0.0 && s.n_asph < 0) f |= DF_FLATNORMAL;
    if (s.c != 0.0) f |= DF_CURVED;
    d.flags = f;
    // branch selection of Spheroid.intercept, elements.py:478-488
    if (s.n_asph >= 0)
        d.kind = KIND_NEWTON;
    else if (s.c == 0.0)
        d.kind = KIND_PLANE;
    else if (s.k == 0.0)
        d.kind = KIND_SPHERE;
    else
        d.kind = KIND_CONIC;
    // Interface.refract, elements.py:356,363
    if (s.mu == 1.0)
        d.refr = REFR_NONE;
    else if (s.mu == -1.0)
        d.refr = REFR_MIRROR;
    else
        d.refr = REFR_SNELL;
}

int ensure_slots(rtx_ctx* ctx, size_t bytes) {
    if (bytes <= ctx->slot_bytes) return 0;
    size_t nb = bytes < 16384 ? 16384 : bytes;
    for (auto& sl : ctx->slots) {
        if (sl.used) CK(cudaEventSynchronize(sl.done));
        if (sl.host) CK(cudaFreeHost(sl.host));
        if (sl.dev) CK(cudaFree(sl.dev));
        sl.host = sl.dev = nullptr;
        CK(cudaMallocHost(&sl.host, nb));
        CK(cudaMalloc(&sl.dev, nb));
        if (!sl.done) CK(cudaEventCreateWithFlags(&sl.done, cudaEventDisableTiming));
        sl.used = false;
        sl.key.clear();
    }
    ctx->slot_bytes = nb;
    return 0;
}

// CTAs per thread-block cluster of the per-CTA store kernel for large FP64
// analytic bundles (C2, the headline, C5).  scripts/sweep.py on C2 (one
// wavelength, 1e7 rays, S = 12), H100 80GB HBM3 SXM at 400 W, median kernel
// ms: 3.67-3.70 unclustered, 3.67 / 3.69 / 3.56-3.60 / 3.48-3.50 with
// 2 / 4 / 8 / 16 CTAs per cluster (16 is a non-portable size: 7 clusters, 112
// of the 132 SMs; the march alone takes 1.09 ms, so the idle SMs cost less
// than the longer runs gain).  DESIGN.md 3.7 has the whole record.
constexpr int DEFAULT_CLUSTER = 16;
// At most this many of those clusters run at once: fewer independent store
// fronts write faster, and the march of 96 SMs still hides behind the stores.
// C2 kernel on an H100 80GB HBM3 SXM at 700 W (scripts/sweep.py, medians of
// three runs alternated): 3.52-3.53 ms with all 7 clusters that fit, 3.35-3.39
// ms with 6 (96 CTAs).  RTX_MAX_CLUSTERS overrides it (0: all that fit).
constexpr int MAX_STORE_CLUSTERS = 6;

template <typename T, bool EXACT, int RPT, int STORE, int WARPS, int NBUF, int CLUSTER = 1>
int launch_one(rtx_ctx* ctx, const TraceParams<T>& p, cudaStream_t stream) {
    auto kern = trace_kernel<T, EXACT, RPT, STORE, WARPS, NBUF, CLUSTER>;
    constexpr int threads = WARPS * 32;
    size_t smem = trace_smem_bytes(sizeof(T), p.S, RPT, STORE, WARPS, NBUF);
    if ((int)smem > ctx->max_smem_optin) return RTX_E_UNSUPPORTED;
    if (smem > 48 * 1024)
        CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int occ = 0;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, threads, smem));
    if (occ < 1) occ = 1;
    const int max_ctas = ctx->tuning.max_ctas_per_sm;
    if (max_ctas > 0 && occ > max_ctas) occ = max_ctas;
    const long long per_cta = (long long)threads * RPT;
    TraceParams<T> q = p;  // launch-wide CTA-tile numbering over the bundles
    long long tiles = 0;
    for (int b = 0; b < q.nbatch; ++b) {
        q.item[b].tile0 = tiles;
        tiles += (q.item[b].N + per_cta - 1) / per_cta;
    }
    q.total_tiles = tiles;
    if constexpr (CLUSTER > 1) {
        // persistent: as many clusters as can be resident at once.  A cluster
        // lives inside one GPC, so with one CTA per SM this can leave SMs idle
        // (H100 SXM, 16 CTAs per cluster: 7 clusters = 112 of 132 SMs).
        cudaLaunchAttribute attr;
        attr.id = cudaLaunchAttributeClusterDimension;
        attr.val.clusterDim.x = CLUSTER;
        attr.val.clusterDim.y = 1;
        attr.val.clusterDim.z = 1;
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(CLUSTER);
        cfg.blockDim = dim3(threads);
        cfg.dynamicSmemBytes = smem;
        cfg.stream = stream;
        cfg.attrs = &attr;
        cfg.numAttrs = 1;
        if constexpr (CLUSTER > 8)
            CK(cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
        int ncl = 0;
        if (cudaOccupancyMaxActiveClusters(&ncl, kern, &cfg) != cudaSuccess || ncl < 1) {
            cudaGetLastError();  // (clear it) no cluster fits: the per-CTA kernel
            return launch_one<T, EXACT, RPT, STORE, WARPS, NBUF, 1>(ctx, p, stream);
        }
        const long long groups = (tiles + CLUSTER - 1) / CLUSTER;
        if (ncl > groups) ncl = (int)groups;
        const int cap = ctx->tuning.max_clusters < 0 ? MAX_STORE_CLUSTERS : ctx->tuning.max_clusters;
        if (cap > 0 && ncl > cap) ncl = cap;
        if (ncl < 1) ncl = 1;
        cfg.gridDim = dim3((unsigned)(ncl * CLUSTER));
        ctx->last_ctas = ncl * CLUSTER;
        CK(cudaLaunchKernelEx(&cfg, kern, q));
    } else {
        long long grid = (long long)ctx->sm_count * occ;  // persistent: one wave
        if (grid > tiles) grid = tiles;
        if (grid < 1) grid = 1;
        ctx->last_ctas = (int)grid;
        kern<<<(unsigned)grid, threads, smem, stream>>>(q);
    }
    const int cfg[5] = {RPT, STORE, WARPS, NBUF, CLUSTER};
    memcpy(ctx->last_cfg, cfg, sizeof(cfg));
    ctx->launches++;
    return (int)cudaGetLastError();
}

struct TraceCfg {
    int rpt, store, warps, nbuf, cluster, lockstep;
};

// One row of the instantiated tuning space.  ONLY: the element size of the
// one arithmetic type the kernel is built for (0: both); in the other type's
// table the row is empty.
template <typename T>
struct KernelRow {
    int rpt, store, warps, nbuf, cluster;
    int (*launch)(rtx_ctx*, const TraceParams<T>&, cudaStream_t);
};

template <typename T, bool EXACT, int RPT, int STORE, int WARPS, int NBUF, int CLUSTER = 1,
          int ONLY = 0>
constexpr KernelRow<T> row() {
    if constexpr (ONLY != 0 && ONLY != (int)sizeof(T))
        return {0, 0, 0, 0, 0, nullptr};
    else
        return {RPT, STORE, WARPS, NBUF, CLUSTER,
                &launch_one<T, EXACT, RPT, STORE, WARPS, NBUF, CLUSTER>};
}

constexpr int F32 = 4, F64 = 8;

template <typename T, bool EXACT>
constexpr KernelRow<T> KERNELS[] = {
    row<T, EXACT, 1, STORE_DIRECT, 8, 1>(),
    row<T, EXACT, 1, STORE_WARP, 8, 2>(),
    row<T, EXACT, 2, STORE_WARP, 8, 2>(),
    row<T, EXACT, 2, STORE_CTA, 16, 1>(),
    row<T, EXACT, 1, STORE_CTA, 16, 1>(),
    row<T, EXACT, 2, STORE_CTA, 32, 1>(),
    row<T, EXACT, 2, STORE_CTA, 8, 1>(),
    row<T, EXACT, 2, STORE_WARP, 16, 2>(),
    // FP32: four rays per thread (64 registers leave room)
    row<T, EXACT, 4, STORE_CTA, 16, 1, 1, F32>(),
    row<T, EXACT, 4, STORE_WARP, 16, 1, 1, F32>(),
    // FP64: clusters of per-CTA stores (FP32 clusters only in the tuning space)
    row<T, EXACT, 2, STORE_CTA, 16, 1, DEFAULT_CLUSTER, F64>(),
#ifdef RTX_TUNING_SPACE
    row<T, EXACT, 2, STORE_CTA, 16, 1, 2, F64>(),
    row<T, EXACT, 2, STORE_CTA, 16, 1, 4, F64>(),
    row<T, EXACT, 2, STORE_CTA, 16, 1, 8, F64>(),
    row<T, EXACT, 4, STORE_CTA, 16, 1, 2, F32>(),
    row<T, EXACT, 4, STORE_CTA, 16, 1, 4, F32>(),
    row<T, EXACT, 4, STORE_CTA, 16, 1, 8, F32>(),
    row<T, EXACT, 4, STORE_CTA, 16, 1, 16, F32>(),
    row<T, EXACT, 2, STORE_CTA, 8, 2>(),
    row<T, EXACT, 1, STORE_WARP, 16, 2>(),
    row<T, EXACT, 2, STORE_WARP, 8, 1>(),
    row<T, EXACT, 1, STORE_CTA, 8, 1>(),
    row<T, EXACT, 1, STORE_CTA, 8, 2>(),
    row<T, EXACT, 1, STORE_CTA, 16, 2>(),
    row<T, EXACT, 2, STORE_CTA, 16, 2>(),
    row<T, EXACT, 1, STORE_CTA, 32, 1>(),
    row<T, EXACT, 1, STORE_CTA, 32, 2>(),
    row<T, EXACT, 4, STORE_WARP, 8, 1, 1, F32>(),
    row<T, EXACT, 4, STORE_CTA, 8, 1, 1, F32>(),
    row<T, EXACT, 4, STORE_CTA, 32, 1, 1, F32>(),
    row<T, EXACT, 2, STORE_WARP, 16, 1>(),
    row<T, EXACT, 4, STORE_WARP, 16, 2, 1, F32>(),
    row<T, EXACT, 4, STORE_WARP, 8, 2, 1, F32>(),
#endif
};

template <typename T, bool EXACT>
int launch_kernel(rtx_ctx* ctx, const TraceParams<T>& p, const TraceCfg& c, cudaStream_t stream) {
    for (const KernelRow<T>& k : KERNELS<T, EXACT>)
        if (k.launch && k.rpt == c.rpt && k.store == c.store && k.warps == c.warps &&
            k.nbuf == c.nbuf && k.cluster == c.cluster)
            return k.launch(ctx, p, stream);
    return RTX_E_UNSUPPORTED;
}

// convert + upload the table; returns the device pointer.  The copy is
// ordered on `stream`; the pinned slot is recycled only after its copy ran.
template <typename T>
int upload_table(rtx_ctx* ctx, const rtx_surface* surf, int S, cudaStream_t stream,
                 const DevSurf<T>** out, const void* const* keep = nullptr, int nkeep = 0) {
    size_t bytes = (size_t)S * sizeof(DevSurf<T>);
    int rc = ensure_slots(ctx, bytes);
    if (rc) return rc;
    // a table that is already resident (same records, same arithmetic type) is
    // reused: repeated traces of the same lens / wavelength put no H2D copy
    // between their kernels
    const size_t raw = (size_t)S * sizeof(rtx_surface);
    const unsigned char* src = reinterpret_cast<const unsigned char*>(surf);
    for (auto& sl : ctx->slots) {
        if (sl.used && sl.key.size() == raw + 1 && sl.key[raw] == (unsigned char)sizeof(T) &&
            memcmp(sl.key.data(), src, raw) == 0) {
            *out = reinterpret_cast<const DevSurf<T>*>(sl.dev);
            return 0;
        }
    }
    // next slot in the ring that holds none of the tables the caller still
    // needs (the other bundles of a batched launch)
    int pick = ctx->next_slot;
    for (int tries = 0; tries < TABLE_SLOTS; ++tries) {
        bool busy = false;
        for (int k = 0; k < nkeep; ++k) busy = busy || keep[k] == ctx->slots[pick].dev;
        if (!busy) break;
        pick = (pick + 1) % TABLE_SLOTS;
    }
    TableSlot& sl = ctx->slots[pick];
    ctx->next_slot = (pick + 1) % TABLE_SLOTS;
    if (sl.used) CK(cudaEventSynchronize(sl.done));
    sl.used = false;
    DevSurf<T>* h = reinterpret_cast<DevSurf<T>*>(sl.host);
    for (int i = 0; i < S; ++i) convert_surface<T>(surf[i], h[i]);
    CK(cudaMemcpyAsync(sl.dev, sl.host, bytes, cudaMemcpyHostToDevice, stream));
    CK(cudaEventRecord(sl.done, stream));
    sl.key.assign(src, src + raw);
    sl.key.push_back((unsigned char)sizeof(T));
    sl.used = true;
    *out = reinterpret_cast<const DevSurf<T>*>(sl.dev);
    return 0;
}

int check_table(const rtx_surface* surf, int S) {
    if (!surf || S < 1 || S > RTX_MAX_SURFACES) return RTX_E_BADARG;
    for (int i = 0; i < S; ++i) {
        if (surf[i].n_asph > RTX_MAX_ASPH) return RTX_E_UNSUPPORTED;
        if (surf[i].n_asph < -1) return RTX_E_BADARG;
    }
    return 0;
}

// the table and the launch rays of a march
int check_march(const rtx_surface* surf, int S, long long N, const void* y0, const void* u0) {
    int rc = check_table(surf, S);
    if (rc) return rc;
    return N < 0 || !y0 || !u0 ? RTX_E_BADARG : 0;
}

bool valid_keep(int keep) { return keep == RTX_KEEP_ALL || keep == RTX_KEEP_LAST; }

// f(double()) or f(float()) by the element type code; RTX_E_BADARG for any other
template <typename F>
int dispatch(int dtype, F&& f) {
    if (dtype == RTX_F64) return f(double());
    if (dtype == RTX_F32) return f(float());
    return RTX_E_BADARG;
}

// the element type check of the calls that compute in FP64 only
int fp64_only(int dtype) {
    if (dtype == RTX_F64) return 0;
    return dtype == RTX_F32 ? RTX_E_UNSUPPORTED : RTX_E_BADARG;
}

// Runs `region` (the device work of one call) between the context's events k0
// and k1.  rtx_last_kernel_ms reports that span only when the region succeeded.
template <typename F>
int timed(rtx_ctx* ctx, F&& region) {
    ctx->kernel_timed = false;
    CK(cudaEventRecord(ctx->k0, ctx->stream));
    int rc = region();
    if (rc) return rc;
    CK(cudaEventRecord(ctx->k1, ctx->stream));
    ctx->kernel_timed = true;
    return 0;
}

// blocks of a grid-stride launch: at least one, at most per_sm per SM.  The
// reductions sum their block partials in an order that depends on the grid.
unsigned cap_grid(const rtx_ctx* ctx, long long nblocks, int per_sm) {
    return (unsigned)std::clamp(nblocks, 1ll, (long long)ctx->sm_count * per_sm);
}

// Makes `ws` hold at least `bytes`.  RTX_E_NOMEM, with the old buffer kept,
// when they do not fit in free device memory plus that buffer.
int reserve(Workspace& ws, size_t bytes) {
    if (bytes <= ws.cap) return 0;
    size_t free_b = 0, total_b = 0;
    CK(cudaMemGetInfo(&free_b, &total_b));
    if (bytes > free_b + ws.cap) return RTX_E_NOMEM;  // nothing freed
    if (ws.p) CK(cudaFree(ws.p));
    ws = Workspace();
    if (cudaMalloc(&ws.p, bytes) != cudaSuccess) {
        cudaGetLastError();  // (clear it)
        ws = Workspace();
        return RTX_E_NOMEM;
    }
    ws.cap = bytes;
    return 0;
}

// owner of one temporary cudaMalloc allocation, freed on every return path
class DeviceBuf {
  public:
    DeviceBuf() = default;
    DeviceBuf(DeviceBuf&& o) noexcept : p_(o.p_) { o.p_ = nullptr; }
    DeviceBuf(const DeviceBuf&) = delete;
    DeviceBuf& operator=(const DeviceBuf&) = delete;
    ~DeviceBuf() {
        if (p_) cudaFree(p_);
    }
    cudaError_t alloc(size_t bytes) {
        cudaError_t e = cudaMalloc(&p_, bytes);
        if (e != cudaSuccess) p_ = nullptr;
        return e;
    }
    void* get() const { return p_; }
    template <typename T>
    T* as() const {
        return static_cast<T*>(p_);
    }

  private:
    void* p_ = nullptr;
};

struct PeerDst {
    int n = 0;
    long long off = 0;
    void* ptr[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    void* ptr_i[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    bool has_i = false;
    bool xy = false;
};

// One trace launch as a front end describes it: the common part, 1 to
// RTX_MAX_BATCH bundles (each with its uploaded table) and, for a single
// bundle, the gather destinations and the per-ray side outputs.
template <typename T>
struct Launch {
    int S;
    int clip;
    bool keep_last;
    const double* rot0;
    long long ld;
    unsigned flags;  // RTX_EXACT, RTX_STORE_DIRECT, RTX_RPT1 / RTX_RPT2
    int newton = 0;  // Newton surfaces of the first bundle's table
    int n = 0;
    BatchItem<T> item[RTX_MAX_BATCH];
    const PeerDst* peers = nullptr;
    unsigned* mask = nullptr;
    T* tsum = nullptr;
    int tsum_upto = 0;

    Launch(const rtx_surface* surf, int S_, const double* rot0_, int clip_, int keep,
           long long ld_, unsigned flags_)
        : S(S_), clip(clip_ ? 1 : 0), keep_last(keep == RTX_KEEP_LAST), rot0(rot0_), ld(ld_),
          flags(flags_) {
        for (int i = 0; i < S; ++i) newton += surf[i].n_asph >= 0;
    }
    void add(const DevSurf<T>* table, long long N, const void* y0, const void* u0, void* Y,
             void* U, void* I, void* Tt) {
        item[n++] = {table, (const T*)y0, (const T*)u0, (T*)Y, (T*)U, (T*)I, (T*)Tt, N, 0};
    }
};

// what the kernel configuration depends on
struct TraceShape {
    size_t elem;     // sizeof(T)
    int S;
    int newton;      // Newton surfaces of the first bundle's table
    long long N;     // the largest bundle
    long long ld;
    bool keep_last;
    int nbatch;
    bool gather;
    bool aligned;    // every output and peer destination 16-byte aligned
    unsigned flags;  // RTX_STORE_DIRECT, RTX_RPT1 / RTX_RPT2
};

// The kernel configuration of a launch (DESIGN.md 3.2): the library's own
// choice by workload, or the RTX_* knobs of an experiment (tu.tuned).
TraceCfg choose_trace_cfg(const TraceShape& sh, const Tuning& tu, size_t smem_optin) {
    const bool explicit_rpt = (sh.flags & (RTX_RPT1 | RTX_RPT2)) != 0;
    const bool fp32 = sh.elem == 4;
    const bool own = !tu.tuned && !explicit_rpt;  // configurations by workload
    // Systems with >= 25 % Newton (aspheric) surfaces are bound by issue slots
    // / the FP64 pipe, not by HBM, and so is a keep-LAST trace (one stored
    // row: the stores are no limit): free-running CTAs with per-warp stores,
    // no lockstep barrier behind the long, divergent Newton chains.  (A fused
    // gather keeps the per-CTA 24 KB runs for its NVLink stores.)
    const bool heavy = own && (sh.newton * 4 >= sh.S || (sh.keep_last && !sh.gather));
    TraceCfg c = {tu.rpt, tu.store, tu.warps, tu.nbuf, tu.cluster, heavy ? 0 : tu.lockstep};
    auto set = [&c](int rpt, int store, int warps, int nbuf) {
        c.rpt = rpt;
        c.store = store;
        c.warps = warps;
        c.nbuf = nbuf;
    };
    if (sh.flags & RTX_RPT1) c.rpt = 1;
    if (sh.flags & RTX_RPT2) c.rpt = 2;
    //  FP64: 2 rays/thread x 16 warps, per-CTA bulk stores (24 KB runs)
    //  FP32: 4 rays/thread x 16 warps (2048-ray tiles, 24 KB runs again):
    //        half the per-thread overhead instructions of 2 rays/thread
    if (own && fp32) set(4, heavy ? STORE_WARP : STORE_CTA, 16, 1);
    else if (heavy) set(2, STORE_WARP, 16, 2);
    // (an explicit RPT request is honoured at every N; the pitch and alignment
    // step-downs below still apply to it)
    if (own && sh.N <= 150 * 1000) {
        set(1, STORE_WARP, 8, 2);  // small bundles: 256-ray warp tiles spread over all SMs
    } else if (own && !heavy && !fp32 && sh.N <= 1500 * 1000) {
        // mid-size FP64 bundles (what an analysis traces): 512-ray tiles, two
        // resident CTAs per SM -- twice the tiles to balance over the SMs
        set(1, STORE_CTA, 16, 1);
    } else if (own && !heavy && fp32 && sh.N > 500 * 1000 && sh.N <= 2500 * 1000) {
        set(2, STORE_CTA, 8, 1);  // mid-size FP32 bundles: 512-ray tiles, three CTAs per SM
    } else if (!explicit_rpt && sh.N <= 32 * 1024) {
        set(1, STORE_WARP, 8, 2);  // (tuned contexts keep the old small-bundle rule)
    } else if (explicit_rpt) {  // explicit RPT: its per-warp store kernel
        set(c.rpt, STORE_WARP, 8, 2);
    }
    // The staged paths write whole 32*rpt-ray groups: the pitch must be a
    // multiple of that, and so must the shard of a gather (into a gather buffer
    // a ragged tail would spill clamped copies of the last ray into the next
    // rank's range -- a race with that rank's own stores).
    const bool aligned = sh.aligned && !(sh.flags & RTX_STORE_DIRECT);
    auto fits = [&sh](int r) {
        return sh.ld % (32 * r) == 0 && (!sh.gather || sh.N % (32 * r) == 0);
    };
    if (aligned && !tu.tuned) {
        // step down to the kernel with fewer rays per thread that fits
        if (c.rpt == 4 && !fits(4)) {
            if (heavy)
                set(2, STORE_WARP, 8, 2);
            else
                set(2, STORE_CTA, 32, 1);
        }
        if (c.rpt == 2 && !fits(2) && fits(1)) set(1, STORE_WARP, 8, 2);
    }
    if (!(aligned && fits(c.rpt))) c.store = STORE_DIRECT;  // per-ray stores: exactly N rays
    // a long table leaves less shared memory for the staging buffers (256 FP64
    // surfaces take 92 KB): step down to the smallest staged kernel, then to
    // per-ray stores, rather than refuse a table the library accepts
    auto smem = [&sh](int rpt, int store, int warps, int nbuf) {
        return trace_smem_bytes(sh.elem, sh.S, rpt, store, warps, nbuf);
    };
    if (!tu.tuned && c.store != STORE_DIRECT &&
        smem(c.rpt, c.store, c.warps, c.nbuf) > smem_optin) {
        if (fits(1) && smem(1, STORE_WARP, 8, 2) <= smem_optin)
            set(1, STORE_WARP, 8, 2);
        else
            c.store = STORE_DIRECT;
    }
    // large FP64 analytic bundles: clusters of CTAs whose stores leave as one
    // run (DEFAULT_CLUSTER).  FP32 stays unclustered: 8-CTA clusters gained
    // only 3-4 % there (1.77-1.78 vs 1.84 ms, C2 in FP32).
    if (own && !heavy && !fp32 && sh.N > 1500 * 1000 && c.rpt == 2 && c.store == STORE_CTA &&
        c.warps == 16 && c.nbuf == 1)
        c.cluster = DEFAULT_CLUSTER;
    // clusters: single-bundle keep-ALL per-CTA stores only (batched launches,
    // fused gathers and keep-LAST traces keep the per-CTA kernel)
    if (sh.nbatch != 1 || sh.gather || sh.keep_last || c.store != STORE_CTA) c.cluster = 1;
    if (c.store == STORE_DIRECT) set(1, STORE_DIRECT, 8, 1);
    return c;
}

bool al16(const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15u) == 0; }

template <typename T>
TraceShape shape_of(const Launch<T>& L) {
    TraceShape sh = {sizeof(T), L.S, L.newton, 0, L.ld, L.keep_last, L.n, L.peers != nullptr,
                     true, L.flags};
    for (int b = 0; b < L.n; ++b) {
        const BatchItem<T>& it = L.item[b];
        sh.N = it.N > sh.N ? it.N : sh.N;
        sh.aligned = sh.aligned && al16(it.Y) && al16(it.U) && al16(it.I) && al16(it.Tt);
    }
    if (const PeerDst* pd = L.peers) {
        // bulk stores need 16-byte aligned runs in every destination
        sh.aligned = sh.aligned && (pd->off * (pd->xy ? 2 : 3) * (long long)sizeof(T)) % 16 == 0 &&
                     (!pd->has_i || (pd->off * 3 * (long long)sizeof(T)) % 16 == 0);
        for (int k = 0; k < pd->n; ++k)
            sh.aligned = sh.aligned && al16(pd->ptr[k]) && al16(pd->ptr_i[k]);
    }
    return sh;
}

template <typename T>
int launch_trace(rtx_ctx* ctx, const Launch<T>& L, cudaStream_t stream) {
    const TraceCfg c = choose_trace_cfg(shape_of(L), ctx->tuning, (size_t)ctx->max_smem_optin);
    TraceParams<T> p;
    memset(&p, 0, sizeof(p));
    p.S = L.S;
    p.clip = L.clip;
    p.keep_last = L.keep_last;
    p.has_rot0 = L.rot0 != nullptr;
    if (L.rot0)
        for (int i = 0; i < 9; ++i) p.rot0[i] = (T)L.rot0[i];
    p.ld = L.ld;
    p.lockstep = c.lockstep;
    p.prefetch = ctx->tuning.prefetch;
    if (const PeerDst* pd = L.peers) {
        p.npeer = pd->n;
        p.peer_off = pd->off;
        p.peer_has_i = pd->has_i ? 1 : 0;
        p.peer_xy = pd->xy ? 1 : 0;
        for (int k = 0; k < pd->n; ++k) {
            p.peer[k] = (T*)pd->ptr[k];
            p.peer_i[k] = (T*)pd->ptr_i[k];
        }
    }
    p.mask = L.mask;
    p.tsum = L.tsum;
    p.tsum_upto = L.tsum_upto < 0 ? L.S - 1 : L.tsum_upto;
    p.nbatch = L.n;
    for (int b = 0; b < L.n; ++b) p.item[b] = L.item[b];
    if (L.flags & RTX_EXACT) {
        if constexpr (sizeof(T) == 8) return launch_kernel<T, true>(ctx, p, c, stream);
        return RTX_E_UNSUPPORTED;  // RTX_EXACT is FP64 only
    }
    return launch_kernel<T, false>(ctx, p, c, stream);
}

// upload the table of a new bundle of `L` (on the context stream, keeping the
// tables of the bundles before it) and add the bundle
template <typename T>
int add_bundle(rtx_ctx* ctx, Launch<T>& L, const rtx_surface* surf, long long N, const void* y0,
               const void* u0, void* Y, void* U, void* I, void* Tt) {
    const void* keep[RTX_MAX_BATCH];
    for (int b = 0; b < L.n; ++b) keep[b] = L.item[b].table;
    const DevSurf<T>* table = nullptr;
    int rc = upload_table<T>(ctx, surf, L.S, ctx->stream, &table, keep, L.n);
    if (rc) return rc;
    L.add(table, N, y0, u0, Y, U, I, Tt);
    return 0;
}

// rtx_trace, rtx_trace_gather: one bundle with the registered side outputs
template <typename T>
int trace_registered(rtx_ctx* ctx, Launch<T>& L, const rtx_surface* surf, long long N,
                     const void* y0, const void* u0, void* Y, void* U, void* I, void* Tt) {
    L.mask = ctx->mask;
    L.tsum = (T*)ctx->tsum;
    L.tsum_upto = ctx->tsum_upto;
    int rc = add_bundle<T>(ctx, L, surf, N, y0, u0, Y, U, I, Tt);
    return rc ? rc : launch_trace<T>(ctx, L, ctx->stream);
}

int ensure_chunk(rtx_ctx* ctx, ChunkBuf& cb, size_t in_bytes, size_t out3, size_t out1) {
    if (!cb.stream) CK(cudaStreamCreateWithFlags(&cb.stream, cudaStreamNonBlocking));
    if (in_bytes > cb.in_bytes) {
        if (cb.y0) CK(cudaFree(cb.y0));
        if (cb.u0) CK(cudaFree(cb.u0));
        cb.y0 = cb.u0 = nullptr;
        cb.in_bytes = 0;
        CK(cudaMalloc(&cb.y0, in_bytes));
        CK(cudaMalloc(&cb.u0, in_bytes));
        cb.in_bytes = in_bytes;
    }
    if (out3 > cb.out3_bytes) {
        if (cb.Y) CK(cudaFree(cb.Y));
        if (cb.U) CK(cudaFree(cb.U));
        if (cb.I) CK(cudaFree(cb.I));
        cb.Y = cb.U = cb.I = nullptr;
        cb.out3_bytes = 0;
        CK(cudaMalloc(&cb.Y, out3));
        CK(cudaMalloc(&cb.U, out3));
        CK(cudaMalloc(&cb.I, out3));
        cb.out3_bytes = out3;
    }
    if (out1 > cb.out1_bytes) {
        if (cb.T) CK(cudaFree(cb.T));
        cb.T = nullptr;
        cb.out1_bytes = 0;
        CK(cudaMalloc(&cb.T, out1));
        cb.out1_bytes = out1;
    }
    return 0;
}

void free_chunk(ChunkBuf& cb) {
    if (cb.y0) cudaFree(cb.y0);
    if (cb.u0) cudaFree(cb.u0);
    if (cb.Y) cudaFree(cb.Y);
    if (cb.U) cudaFree(cb.U);
    if (cb.I) cudaFree(cb.I);
    if (cb.T) cudaFree(cb.T);
    if (cb.stream) cudaStreamDestroy(cb.stream);
    cb = ChunkBuf();
}

void clear_chunk_events(rtx_ctx* ctx) {
    for (auto& pr : ctx->chunk_events) {
        cudaEventDestroy(pr.first);
        cudaEventDestroy(pr.second);
    }
    ctx->chunk_events.clear();
}

// cuFFT is opened at run time, so that librtx.so loads and traces on a machine
// without it (the Python side preloads the toolkit's or the pip wheel's copy
// with RTLD_GLOBAL; the soname lookup then finds that one)
struct CufftApi {
    bool ok = false;
    cufftResult (*create)(cufftHandle*) = nullptr;
    cufftResult (*set_auto_allocation)(cufftHandle, int) = nullptr;
    cufftResult (*get_size_many64)(cufftHandle, int, long long*, long long*, long long, long long,
                                   long long*, long long, long long, cufftType, long long,
                                   size_t*) = nullptr;
    cufftResult (*make_plan_many64)(cufftHandle, int, long long*, long long*, long long, long long,
                                    long long*, long long, long long, cufftType, long long,
                                    size_t*) = nullptr;
    cufftResult (*set_work_area)(cufftHandle, void*) = nullptr;
    cufftResult (*set_stream)(cufftHandle, cudaStream_t) = nullptr;
    cufftResult (*exec_z2z)(cufftHandle, cufftDoubleComplex*, cufftDoubleComplex*, int) = nullptr;
    cufftResult (*destroy)(cufftHandle) = nullptr;
};

const CufftApi& cufft_api() {
    static const CufftApi api = [] {
        CufftApi a;
        void* h = dlopen("libcufft.so.11", RTLD_NOW | RTLD_GLOBAL);
        if (!h) h = dlopen("libcufft.so", RTLD_NOW | RTLD_GLOBAL);
        if (!h) return a;
        bool all = true;
        auto sym = [&](auto& fn, const char* name) {
            fn = reinterpret_cast<std::remove_reference_t<decltype(fn)>>(dlsym(h, name));
            all = all && fn != nullptr;
        };
        sym(a.create, "cufftCreate");
        sym(a.set_auto_allocation, "cufftSetAutoAllocation");
        sym(a.get_size_many64, "cufftGetSizeMany64");
        sym(a.make_plan_many64, "cufftMakePlanMany64");
        sym(a.set_work_area, "cufftSetWorkArea");
        sym(a.set_stream, "cufftSetStream");
        sym(a.exec_z2z, "cufftExecZ2Z");
        sym(a.destroy, "cufftDestroy");
        a.ok = all;
        return a;
    }();
    return api;
}

void release_fft_plan(rtx_ctx* ctx) {
    if (ctx->fft_planned) cufft_api().destroy(ctx->fft_plan);
    if (ctx->fft_work) cudaFree(ctx->fft_work);
    ctx->fft_planned = false;
    ctx->fft_work = nullptr;
    ctx->fft_work_bytes = 0;
    ctx->fft_nx = ctx->fft_ny = 0;
}

constexpr size_t SMALL_PATH_BYTES = 4u << 20;
constexpr size_t ZERO_COPY_BYTES = 16u << 10;  // rays + results of a zero-copy small trace

// grow the pinned bounce buffer of the small paths (and its device twin) to `need` bytes
int ensure_small(rtx_ctx* ctx, size_t need) {
    if (need <= ctx->small_bytes) return 0;
    if (ctx->small_host) CK(cudaFreeHost(ctx->small_host));
    if (ctx->small_dev) CK(cudaFree(ctx->small_dev));
    ctx->small_host = ctx->small_dev = nullptr;
    ctx->small_bytes = 0;
    const size_t nb = need < (256u << 10) ? (256u << 10) : need;
    CK(cudaMallocHost(&ctx->small_host, nb));
    CK(cudaMalloc(&ctx->small_dev, nb));
    ctx->small_bytes = nb;
    return 0;
}

// Latency path for small bundles (aim_chief / aim_marginal issue hundreds of
// 1-3 ray traces, rayopt/system.py:507-555): one pinned bounce buffer, ONE
// H2D of [y0|u0], the kernel with ld = N (per-thread stores, reference
// layout on the device), ONE D2H of [Y|U|I|T], one synchronisation.
template <typename T>
int trace_host_small(rtx_ctx* ctx, const rtx_surface* surf, int S, const double* rot0,
                     long long N, const void* y0, const void* u0, int clip, int keep, void* Y,
                     void* U, void* I, void* Tt, unsigned flags, size_t in_bytes,
                     size_t out_bytes) {
    const int rows = keep == RTX_KEEP_LAST ? 1 : S;
    const size_t need = in_bytes + out_bytes;
    int rc = ensure_small(ctx, need);
    if (rc) return rc;
    char* h = (char*)ctx->small_host;
    const size_t v3 = (size_t)N * 3 * sizeof(T), r3 = (size_t)rows * v3, r1 = r3 / 3;
    memcpy(h, y0, v3);
    memcpy(h + v3, u0, v3);
    // A handful of rays (ray aiming: 1-3): ZERO-COPY.  Page-locked memory is
    // mapped into the device's address space (UVA), so the kernel reads the
    // launch rays and writes its results straight over PCIe -- launch + one
    // synchronisation, no copy-engine round trips (2 x ~8 us).  Beyond
    // ZERO_COPY_BYTES the DMA engines win: one H2D, the kernel, one D2H.
    const bool zero_copy = need <= ZERO_COPY_BYTES && !getenv("RTX_NO_ZERO_COPY");
    char* d = zero_copy ? h : (char*)ctx->small_dev;
    if (!zero_copy) CK(cudaMemcpyAsync(d, h, in_bytes, cudaMemcpyHostToDevice, ctx->stream));
    char* dY = d + in_bytes;
    char *dU = dY + r3, *dI = dU + r3, *dT = dI + r3;
    Launch<T> L(surf, S, rot0, clip, keep, N, flags | RTX_STORE_DIRECT);
    rc = add_bundle<T>(ctx, L, surf, N, d, d + v3, Y ? dY : nullptr, U ? dU : nullptr,
                       I ? dI : nullptr, Tt ? dT : nullptr);
    if (!rc) rc = launch_trace<T>(ctx, L, ctx->stream);
    if (rc) return rc;
    if (!zero_copy)
        CK(cudaMemcpyAsync(h + in_bytes, dY, out_bytes, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    const char* o = h + in_bytes;
    if (Y) memcpy(Y, o, r3);
    if (U) memcpy(U, o + r3, r3);
    if (I) memcpy(I, o + 2 * r3, r3);
    if (Tt) memcpy(Tt, o + 3 * r3, r1);
    clear_chunk_events(ctx);
    ctx->kernel_timed = false;
    return 0;
}

template <typename T>
int trace_host(rtx_ctx* ctx, const rtx_surface* surf, int S, const double* rot0, long long N,
               const void* y0, const void* u0, int clip, int keep, void* Y, void* U, void* I,
               void* Tt, unsigned flags) {
    const int rows = keep == RTX_KEEP_LAST ? 1 : S;
    {
        const size_t in_b = (size_t)N * 6 * sizeof(T);
        const size_t out_b = (size_t)rows * N * 10 * sizeof(T);
        // (an explicit store-path / RPT request goes through the general path)
        if (in_b + out_b <= SMALL_PATH_BYTES && !(flags & (RTX_RPT1 | RTX_RPT2 | RTX_STORE_DIRECT)))
            return trace_host_small<T>(ctx, surf, S, rot0, N, y0, u0, clip, keep, Y, U, I, Tt,
                                       flags, in_b, out_b);
    }
    // chunk: ~256 MB of results, whole 128-ray groups
    long long per_ray = (long long)rows * 10 * sizeof(T) + 6 * sizeof(T);
    long long C = (256ll << 20) / per_ray;
    C = (C / 128) * 128;  // whole 128-ray groups: every staged kernel applies
    if (C < 4096) C = 4096;
    if (C > N) C = ((N + 127) / 128) * 128;
    const size_t in_bytes = (size_t)C * 3 * sizeof(T);
    const size_t out3 = (size_t)rows * C * 3 * sizeof(T);
    const size_t out1 = (size_t)rows * C * sizeof(T);
    for (int b = 0; b < 2; ++b) {
        int rc = ensure_chunk(ctx, ctx->chunk[b], in_bytes, out3, out1);
        if (rc) return rc;
    }
    // the table is uploaded once on the main stream; chunk streams wait for it
    const DevSurf<T>* table = nullptr;
    int rc = upload_table<T>(ctx, surf, S, ctx->stream, &table);
    if (rc) return rc;
    struct EventGuard {  // destroyed on every return path
        cudaEvent_t e = nullptr;
        ~EventGuard() {
            if (e) cudaEventDestroy(e);
        }
    } guard;
    CK(cudaEventCreateWithFlags(&guard.e, cudaEventDisableTiming));
    cudaEvent_t table_ready = guard.e;
    CK(cudaEventRecord(table_ready, ctx->stream));
    clear_chunk_events(ctx);
    int nchunk = 0;
    for (long long c0 = 0; c0 < N; c0 += C, ++nchunk) {
        ChunkBuf& cb = ctx->chunk[nchunk & 1];
        const long long n = (N - c0 < C) ? (N - c0) : C;
        if (nchunk < 2) CK(cudaStreamWaitEvent(cb.stream, table_ready, 0));
        CK(cudaMemcpyAsync(cb.y0, (const T*)y0 + c0 * 3, (size_t)n * 3 * sizeof(T),
                           cudaMemcpyHostToDevice, cb.stream));
        CK(cudaMemcpyAsync(cb.u0, (const T*)u0 + c0 * 3, (size_t)n * 3 * sizeof(T),
                           cudaMemcpyHostToDevice, cb.stream));
        cudaEvent_t e0 = nullptr, e1 = nullptr;
        CK(cudaEventCreate(&e0));
        if (cudaError_t er = cudaEventCreate(&e1)) {
            cudaEventDestroy(e0);
            return (int)er;
        }
        ctx->chunk_events.emplace_back(e0, e1);  // owned by ctx from here on
        CK(cudaEventRecord(e0, cb.stream));
        Launch<T> L(surf, S, rot0, clip, keep, C, flags);
        L.add(table, n, cb.y0, cb.u0, Y ? cb.Y : nullptr, U ? cb.U : nullptr, I ? cb.I : nullptr,
              Tt ? cb.T : nullptr);
        rc = launch_trace<T>(ctx, L, cb.stream);
        if (rc) {
            for (int b = 0; b < 2; ++b) cudaStreamSynchronize(ctx->chunk[b].stream);
            return rc;
        }
        CK(cudaEventRecord(e1, cb.stream));
        const size_t w3 = (size_t)n * 3 * sizeof(T), w1 = (size_t)n * sizeof(T);
        const size_t sp3 = (size_t)C * 3 * sizeof(T), sp1 = (size_t)C * sizeof(T);
        const size_t dp3 = (size_t)N * 3 * sizeof(T), dp1 = (size_t)N * sizeof(T);
        if (Y)
            CK(cudaMemcpy2DAsync((T*)Y + c0 * 3, dp3, cb.Y, sp3, w3, rows, cudaMemcpyDeviceToHost,
                                 cb.stream));
        if (U)
            CK(cudaMemcpy2DAsync((T*)U + c0 * 3, dp3, cb.U, sp3, w3, rows, cudaMemcpyDeviceToHost,
                                 cb.stream));
        if (I)
            CK(cudaMemcpy2DAsync((T*)I + c0 * 3, dp3, cb.I, sp3, w3, rows, cudaMemcpyDeviceToHost,
                                 cb.stream));
        if (Tt)
            CK(cudaMemcpy2DAsync((T*)Tt + c0, dp1, cb.T, sp1, w1, rows, cudaMemcpyDeviceToHost,
                                 cb.stream));
    }
    for (int b = 0; b < 2; ++b) CK(cudaStreamSynchronize(ctx->chunk[b].stream));
    ctx->kernel_timed = false;
    return 0;
}

}  // namespace

// =========================================================================
extern "C" {

int rtx_abi_version(void) { return RTX_ABI_VERSION; }

size_t rtx_sizeof_surface(void) { return sizeof(rtx_surface); }
size_t rtx_sizeof_aim(void) { return sizeof(rtx_aim); }
size_t rtx_sizeof_opd(void) { return sizeof(rtx_opd); }
size_t rtx_sizeof_spot(void) { return sizeof(rtx_spot); }
size_t rtx_sizeof_otf(void) { return sizeof(rtx_otf); }
size_t rtx_sizeof_pupil(void) { return sizeof(rtx_pupil); }

int rtx_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
    return n;
}

const char* rtx_strerror(int code) {
    switch (code) {
        case RTX_OK: return "ok";
        case RTX_E_BADARG: return "rtx: bad argument";
        case RTX_E_UNSUPPORTED:
            return "rtx: unsupported (too many aspheric coefficients / surfaces, RTX_EXACT with FP32, "
                   "FP32 in the PSF calls, or rtx_psf without a loadable cuFFT: libcufft.so.11 "
                   "was not found by dlopen)";
        case RTX_E_NOMEM: return "rtx: out of memory";
        default: break;
    }
    if (code > 0) return cudaGetErrorString((cudaError_t)code);
    return "rtx: unknown error";
}

int rtx_surface_finalize(rtx_surface* surf, int n, const double* radius) {
    if (!surf || n < 0) return RTX_E_BADARG;
    for (int i = 0; i < n; ++i) {
        rtx_surface& s = surf[i];
        s.kc2 = (1.0 + s.k) * (s.c * s.c);
        if (radius) s.radius2 = radius[i] * radius[i];
        s.muf = fabs(s.mu);
        s.sgn = s.mu > 0 ? 1.0 : (s.mu < 0 ? -1.0 : 0.0);
        s.mu2m1 = s.mu * s.mu - 1.0;
        for (int j = 0; j < RTX_MAX_ASPH; ++j)
            s.dasph[j] = (j < s.n_asph) ? (double)(2 * (j + 1)) * s.asph[j] : 0.0;
    }
    return 0;
}

int rtx_init(int device, rtx_ctx** out) {
    if (!out) return RTX_E_BADARG;
    int n = 0;
    CK(cudaGetDeviceCount(&n));
    if (device < 0 || device >= n) return RTX_E_BADARG;
    CK(cudaSetDevice(device));
    rtx_ctx* ctx = new (std::nothrow) rtx_ctx();
    if (!ctx) return RTX_E_NOMEM;
    ctx->device = device;
    auto setup = [&]() -> int {
        cudaDeviceProp prop;
        CK(cudaGetDeviceProperties(&prop, device));
        ctx->sm_count = prop.multiProcessorCount;
        ctx->max_smem_optin = (int)prop.sharedMemPerBlockOptin;
        CK(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
        CK(cudaEventCreate(&ctx->t0));
        CK(cudaEventCreate(&ctx->t1));
        CK(cudaEventCreate(&ctx->k0));
        CK(cudaEventCreate(&ctx->k1));
        return 0;
    };
    if (int rc = setup()) {
        rtx_free(ctx);
        return rc;
    }
    // tuning knobs (experiments; they override choose_trace_cfg's choice)
    Tuning& tu = ctx->tuning;
    if (const char* e = getenv("RTX_RPT")) {
        int v = atoi(e);
        if (v == 1 || v == 2 || v == 4) tu.rpt = v;
        tu.tuned = true;
    }
    if (const char* e = getenv("RTX_WARPS")) {
        int v = atoi(e);
        if (v == 8 || v == 16 || v == 32) tu.warps = v;
    }
    if (const char* e = getenv("RTX_STORE")) {
        int v = atoi(e);
        if (v == 1 || v == 2) tu.store = v;
    }
    if (const char* e = getenv("RTX_NBUF")) {
        int v = atoi(e);
        if (v == 1 || v == 2) tu.nbuf = v;
    }
    if (const char* e = getenv("RTX_CLUSTER")) {
        int v = atoi(e);
        if (v == 1 || v == 2 || v == 4 || v == 8 || v == 16) tu.cluster = v;
    }
    if (getenv("RTX_WARPS") || getenv("RTX_STORE") || getenv("RTX_NBUF") || getenv("RTX_CLUSTER"))
        tu.tuned = true;
    if (const char* e = getenv("RTX_LOCK")) tu.lockstep = atoi(e) != 0;
    if (const char* e = getenv("RTX_MAX_CTAS")) tu.max_ctas_per_sm = atoi(e);
    if (const char* e = getenv("RTX_MAX_CLUSTERS")) tu.max_clusters = atoi(e);
    if (const char* e = getenv("RTX_TUNE")) tu.prefetch = !(atoi(e) & 2);
    *out = ctx;
    return 0;
}

int rtx_free(rtx_ctx* ctx) {
    if (!ctx) return 0;
    cudaSetDevice(ctx->device);
    cudaDeviceSynchronize();
    clear_chunk_events(ctx);
    for (auto& sl : ctx->slots) {
        if (sl.host) cudaFreeHost(sl.host);
        if (sl.dev) cudaFree(sl.dev);
        if (sl.done) cudaEventDestroy(sl.done);
    }
    free_chunk(ctx->chunk[0]);
    free_chunk(ctx->chunk[1]);
    for (Workspace& w : ctx->ws)
        if (w.p) cudaFree(w.p);
    release_fft_plan(ctx);
    if (ctx->small_host) cudaFreeHost(ctx->small_host);
    if (ctx->small_dev) cudaFree(ctx->small_dev);
    if (ctx->t0) cudaEventDestroy(ctx->t0);
    if (ctx->t1) cudaEventDestroy(ctx->t1);
    if (ctx->k0) cudaEventDestroy(ctx->k0);
    if (ctx->k1) cudaEventDestroy(ctx->k1);
    if (ctx->stream) cudaStreamDestroy(ctx->stream);
    delete ctx;
    return 0;
}

int rtx_sync(rtx_ctx* ctx) {
    if (!ctx) return RTX_E_BADARG;
    CK(cudaStreamSynchronize(ctx->stream));
    return 0;
}

int rtx_device_info(rtx_ctx* ctx, int* sm_count, size_t* free_bytes, size_t* total_bytes,
                    char* name, int name_len) {
    if (!ctx) return RTX_E_BADARG;
    CK(cudaSetDevice(ctx->device));
    if (sm_count) *sm_count = ctx->sm_count;
    size_t f = 0, t = 0;
    CK(cudaMemGetInfo(&f, &t));
    if (free_bytes) *free_bytes = f;
    if (total_bytes) *total_bytes = t;
    if (name && name_len > 0) {
        cudaDeviceProp prop;
        CK(cudaGetDeviceProperties(&prop, ctx->device));
        snprintf(name, (size_t)name_len, "%s", prop.name);
    }
    return 0;
}

int rtx_malloc(rtx_ctx* ctx, size_t bytes, void** dptr) {
    if (!ctx || !dptr) return RTX_E_BADARG;
    CK(cudaSetDevice(ctx->device));
    CK(cudaMalloc(dptr, bytes ? bytes : 16));
    return 0;
}
int rtx_free_device(rtx_ctx* ctx, void* dptr) {
    if (!ctx) return RTX_E_BADARG;
    CK(cudaSetDevice(ctx->device));
    CK(cudaFree(dptr));
    return 0;
}
int rtx_host_alloc(rtx_ctx* ctx, size_t bytes, void** hptr) {
    if (!ctx || !hptr) return RTX_E_BADARG;
    CK(cudaSetDevice(ctx->device));
    CK(cudaMallocHost(hptr, bytes ? bytes : 16));
    return 0;
}
int rtx_host_free(rtx_ctx* ctx, void* hptr) {
    (void)ctx;  // page-locked memory may outlive the context that allocated it
    CK(cudaFreeHost(hptr));
    return 0;
}

int rtx_numa_bind(rtx_ctx* ctx, int enable, int* node_out) {
    if (!ctx) return RTX_E_BADARG;
    if (node_out) *node_out = -1;
    if (!enable) {
        if (ctx->numa_bound) {
            sched_setaffinity(0, sizeof(cpu_set_t), &ctx->saved_affinity);
            syscall(SYS_set_mempolicy, 0 /* MPOL_DEFAULT */, nullptr, 0);
            ctx->numa_bound = false;
        }
        return 0;
    }
    char bus[32] = {0};
    CK(cudaDeviceGetPCIBusId(bus, (int)sizeof(bus), ctx->device));
    for (char* c = bus; *c; ++c) *c = (char)tolower((unsigned char)*c);
    char path[128];
    snprintf(path, sizeof(path), "/sys/bus/pci/devices/%s/numa_node", bus);
    int node = -1;
    if (FILE* f = fopen(path, "r")) {
        if (fscanf(f, "%d", &node) != 1) node = -1;
        fclose(f);
    }
    if (node < 0 || node >= 1024) return 0;  // not reported: leave everything alone
    snprintf(path, sizeof(path), "/sys/devices/system/node/node%d/cpulist", node);
    cpu_set_t set;
    CPU_ZERO(&set);
    int ncpu = 0;
    if (FILE* f = fopen(path, "r")) {  // "0-31,64-95"
        int a = 0, b = 0;
        while (fscanf(f, "%d", &a) == 1) {
            b = a;
            int ch = fgetc(f);
            if (ch == '-') {
                if (fscanf(f, "%d", &b) != 1) b = a;
                ch = fgetc(f);
            }
            for (int c = a; c <= b && c < CPU_SETSIZE; ++c) {
                CPU_SET(c, &set);
                ++ncpu;
            }
            if (ch != ',') break;
        }
        fclose(f);
    }
    if (ncpu == 0) return 0;
    if (!ctx->numa_bound) sched_getaffinity(0, sizeof(cpu_set_t), &ctx->saved_affinity);
    // only CPUs this process may use anyway (cgroup / taskset limits)
    cpu_set_t both;
    CPU_AND(&both, &set, &ctx->saved_affinity);
    if (CPU_COUNT(&both) > 0) sched_setaffinity(0, sizeof(cpu_set_t), &both);
    unsigned long mask[16] = {0};
    mask[node / (8 * sizeof(unsigned long))] |= 1ul << (node % (8 * sizeof(unsigned long)));
    syscall(SYS_set_mempolicy, 1 /* MPOL_PREFERRED */, mask, 8 * sizeof(mask));
    ctx->numa_bound = true;
    if (node_out) *node_out = node;
    return 0;
}
int rtx_memcpy_h2d(rtx_ctx* ctx, void* dst, const void* src, size_t bytes) {
    if (!ctx) return RTX_E_BADARG;
    CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, ctx->stream));
    return 0;
}
int rtx_memcpy_d2h(rtx_ctx* ctx, void* dst, const void* src, size_t bytes) {
    if (!ctx) return RTX_E_BADARG;
    CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    return 0;
}
int rtx_memcpy_d2d(rtx_ctx* ctx, void* dst, const void* src, size_t bytes) {
    if (!ctx) return RTX_E_BADARG;
    CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, ctx->stream));
    return 0;
}
int rtx_memcpy2d_d2h(rtx_ctx* ctx, void* dst, size_t dpitch, const void* src, size_t spitch,
                     size_t width, size_t height) {
    if (!ctx) return RTX_E_BADARG;
    CK(cudaMemcpy2DAsync(dst, dpitch, src, spitch, width, height, cudaMemcpyDeviceToHost,
                         ctx->stream));
    return 0;
}
int rtx_memset(rtx_ctx* ctx, void* dptr, int value, size_t bytes) {
    if (!ctx) return RTX_E_BADARG;
    CK(cudaMemsetAsync(dptr, value, bytes, ctx->stream));
    return 0;
}

int rtx_timer_start(rtx_ctx* ctx) {
    if (!ctx) return RTX_E_BADARG;
    CK(cudaEventRecord(ctx->t0, ctx->stream));
    return 0;
}
int rtx_timer_stop(rtx_ctx* ctx, float* ms) {
    if (!ctx || !ms) return RTX_E_BADARG;
    CK(cudaEventRecord(ctx->t1, ctx->stream));
    CK(cudaEventSynchronize(ctx->t1));
    CK(cudaEventElapsedTime(ms, ctx->t0, ctx->t1));
    return 0;
}
int rtx_last_kernel_ms(rtx_ctx* ctx, float* ms) {
    if (!ctx || !ms) return RTX_E_BADARG;
    if (ctx->kernel_timed) {
        CK(cudaEventSynchronize(ctx->k1));
        CK(cudaEventElapsedTime(ms, ctx->k0, ctx->k1));
        return 0;
    }
    float tot = 0.f;
    for (auto& pr : ctx->chunk_events) {
        float t = 0.f;
        CK(cudaEventSynchronize(pr.second));
        CK(cudaEventElapsedTime(&t, pr.first, pr.second));
        tot += t;
    }
    *ms = tot;
    return 0;
}
int64_t rtx_launch_count(rtx_ctx* ctx) { return ctx ? ctx->launches : 0; }
int rtx_last_launch_ctas(rtx_ctx* ctx, int* ctas) {
    if (!ctx || !ctas) return RTX_E_BADARG;
    *ctas = ctx->last_ctas;
    return 0;
}
int rtx_last_launch_config(rtx_ctx* ctx, int cfg[5]) {
    if (!ctx || !cfg) return RTX_E_BADARG;
    memcpy(cfg, ctx->last_cfg, sizeof(ctx->last_cfg));
    return 0;
}

int rtx_trace(rtx_ctx* ctx, const rtx_surface* surf, int S, const double* rot0, int dtype,
              int64_t N, const void* y0, const void* u0, int clip, int keep, int64_t ld, void* Y,
              void* U, void* I, void* T, unsigned flags) {
    if (!ctx) return RTX_E_BADARG;
    int rc = check_march(surf, S, N, y0, u0);
    if (rc) return rc;
    if (ld < N || !valid_keep(keep)) return RTX_E_BADARG;
    return dispatch(dtype, [&](auto t) -> int {
        if (N == 0) return 0;
        CK(cudaSetDevice(ctx->device));
        return timed(ctx, [&] {
            Launch<decltype(t)> L(surf, S, rot0, clip, keep, ld, flags);
            return trace_registered(ctx, L, surf, N, y0, u0, Y, U, I, T);
        });
    });
}

}  // extern "C"

namespace {
template <typename T>
int trace_batch(rtx_ctx* ctx, int nb, const rtx_surface* const* surf, int S, const double* rot0,
                const int64_t* N, const void* const* y0, const void* const* u0, int clip, int keep,
                long long ld, void* const* Y, void* const* U, void* const* I, void* const* Tt,
                unsigned flags) {
    Launch<T> L(surf[0], S, rot0, clip, keep, ld, flags);
    for (int b = 0; b < nb; ++b) {
        int rc = add_bundle<T>(ctx, L, surf[b], N[b], y0[b], u0[b], Y ? Y[b] : nullptr,
                               U ? U[b] : nullptr, I ? I[b] : nullptr, Tt ? Tt[b] : nullptr);
        if (rc) return rc;
    }
    return launch_trace<T>(ctx, L, ctx->stream);
}
}  // namespace

extern "C" {

int rtx_trace_batch(rtx_ctx* ctx, int nb, const rtx_surface* const* surf, int S,
                    const double* rot0, int dtype, const int64_t* N, const void* const* y0,
                    const void* const* u0, int clip, int keep, int64_t ld, void* const* Y,
                    void* const* U, void* const* I, void* const* T, unsigned flags) {
    if (!ctx || nb < 1 || nb > RTX_MAX_BATCH || !surf || !N || !y0 || !u0) return RTX_E_BADARG;
    if (!valid_keep(keep)) return RTX_E_BADARG;
    return dispatch(dtype, [&](auto t) -> int {
        for (int b = 0; b < nb; ++b) {
            int rc = check_table(surf[b], S);
            if (rc) return rc;
            if (N[b] < 1 || ld < N[b] || !y0[b] || !u0[b]) return RTX_E_BADARG;
        }
        CK(cudaSetDevice(ctx->device));
        return timed(ctx, [&] {
            return trace_batch<decltype(t)>(ctx, nb, surf, S, rot0, N, y0, u0, clip, keep, ld, Y,
                                            U, I, T, flags);
        });
    });
}

}  // extern "C"

namespace {
constexpr size_t BATCH_HOST_BYTES = 64u << 20;

template <typename T>
int trace_batch_host(rtx_ctx* ctx, int nb, const rtx_surface* const* surf, int S,
                     const double* rot0, const int64_t* N, const void* const* y0,
                     const void* const* u0, int clip, int keep, void* const* Y, void* const* U,
                     void* const* I, void* const* Tt, unsigned flags) {
    const int rows = keep == RTX_KEEP_LAST ? 1 : S;
    long long nmax = 0;
    for (int b = 0; b < nb; ++b) nmax = N[b] > nmax ? N[b] : nmax;
    const long long ld = (nmax + 31) / 32 * 32;  // one pitch for all bundles: whole 32-ray groups
    std::vector<size_t> in_off((size_t)nb);
    size_t o = 0;
    for (int b = 0; b < nb; ++b) {  // [y0|u0] of every bundle, 16-byte aligned
        in_off[(size_t)b] = o;
        o += ((size_t)N[b] * 6 * sizeof(T) + 15) & ~size_t(15);
    }
    const size_t per3 = (size_t)rows * ld * 3 * sizeof(T), per1 = (size_t)rows * ld * sizeof(T);
    const size_t per_bundle = (Y ? per3 : 0) + (U ? per3 : 0) + (I ? per3 : 0) + (Tt ? per1 : 0);
    const size_t in_pad = (o + 255) & ~size_t(255);
    const size_t need = in_pad + per_bundle * nb;
    if (need > BATCH_HOST_BYTES) {  // large bundles: one by one through the chunked pipeline
        for (int b = 0; b < nb; ++b) {
            if (N[b] == 0) continue;
            int rc = trace_host<T>(ctx, surf[b], S, rot0, N[b], y0[b], u0[b], clip, keep,
                                   Y ? Y[b] : nullptr, U ? U[b] : nullptr, I ? I[b] : nullptr,
                                   Tt ? Tt[b] : nullptr, flags);
            if (rc) return rc;
        }
        return 0;
    }
    if (int rc = ensure_small(ctx, need)) return rc;
    char* h = (char*)ctx->small_host;
    char* d = (char*)ctx->small_dev;
    for (int b = 0; b < nb; ++b) {
        const size_t v3 = (size_t)N[b] * 3 * sizeof(T);
        if (!v3) continue;
        memcpy(h + in_off[(size_t)b], y0[b], v3);
        memcpy(h + in_off[(size_t)b] + v3, u0[b], v3);
    }
    CK(cudaMemcpyAsync(d, h, o, cudaMemcpyHostToDevice, ctx->stream));
    for (int g0 = 0; g0 < nb; g0 += RTX_MAX_BATCH) {
        const int g = nb - g0 < RTX_MAX_BATCH ? nb - g0 : RTX_MAX_BATCH;
        const rtx_surface* gs[RTX_MAX_BATCH];
        int64_t gn[RTX_MAX_BATCH];
        const void *gy0[RTX_MAX_BATCH], *gu0[RTX_MAX_BATCH];
        void *gY[RTX_MAX_BATCH], *gU[RTX_MAX_BATCH], *gI[RTX_MAX_BATCH], *gT[RTX_MAX_BATCH];
        int m = 0;
        for (int k = 0; k < g; ++k) {
            const int b = g0 + k;
            if (N[b] == 0) continue;
            char* ob = d + in_pad + per_bundle * b;
            gs[m] = surf[b];
            gn[m] = N[b];
            gy0[m] = d + in_off[(size_t)b];
            gu0[m] = d + in_off[(size_t)b] + (size_t)N[b] * 3 * sizeof(T);
            gY[m] = Y ? ob : nullptr;
            ob += Y ? per3 : 0;
            gU[m] = U ? ob : nullptr;
            ob += U ? per3 : 0;
            gI[m] = I ? ob : nullptr;
            ob += I ? per3 : 0;
            gT[m] = Tt ? ob : nullptr;
            ++m;
        }
        if (m == 0) continue;
        int rc = trace_batch<T>(ctx, m, gs, S, rot0, gn, gy0, gu0, clip, keep, ld, Y ? gY : nullptr,
                                U ? gU : nullptr, I ? gI : nullptr, Tt ? gT : nullptr, flags);
        if (rc) return rc;
    }
    CK(cudaMemcpyAsync(h + in_pad, d + in_pad, per_bundle * nb, cudaMemcpyDeviceToHost,
                       ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    for (int b = 0; b < nb; ++b) {  // (rows, ld, k) on the device -> (rows, N, k) of the caller
        const char* ob = h + in_pad + per_bundle * b;
        auto unpack = [&](void* dst, int k) {
            if (!dst) return;
            const size_t w = (size_t)N[b] * k * sizeof(T), pitch = (size_t)ld * k * sizeof(T);
            for (int r = 0; r < rows; ++r) memcpy((char*)dst + r * w, ob + r * pitch, w);
            ob += (size_t)rows * pitch;
        };
        unpack(Y ? Y[b] : nullptr, 3);
        unpack(U ? U[b] : nullptr, 3);
        unpack(I ? I[b] : nullptr, 3);
        unpack(Tt ? Tt[b] : nullptr, 1);
    }
    clear_chunk_events(ctx);
    ctx->kernel_timed = false;
    return 0;
}
}  // namespace

extern "C" {

int rtx_trace_batch_host(rtx_ctx* ctx, int nb, const rtx_surface* const* surf, int S,
                         const double* rot0, int dtype, const int64_t* N, const void* const* y0,
                         const void* const* u0, int clip, int keep, void* const* Y,
                         void* const* U, void* const* I, void* const* T, unsigned flags) {
    if (!ctx || nb < 1 || !surf || !N || !y0 || !u0) return RTX_E_BADARG;
    if (!valid_keep(keep)) return RTX_E_BADARG;
    return dispatch(dtype, [&](auto t) -> int {
        for (int b = 0; b < nb; ++b) {
            int rc = check_table(surf[b], S);
            if (rc) return rc;
            if (N[b] < 0 || (N[b] > 0 && (!y0[b] || !u0[b]))) return RTX_E_BADARG;
        }
        CK(cudaSetDevice(ctx->device));
        return trace_batch_host<decltype(t)>(ctx, nb, surf, S, rot0, N, y0, u0, clip, keep, Y, U,
                                             I, T, flags);
    });
}

int rtx_trace_host(rtx_ctx* ctx, const rtx_surface* surf, int S, const double* rot0, int dtype,
                   int64_t N, const void* y0, const void* u0, int clip, int keep, void* Y, void* U,
                   void* I, void* T, unsigned flags) {
    if (!ctx) return RTX_E_BADARG;
    int rc = check_march(surf, S, N, y0, u0);
    if (rc) return rc;
    if (!valid_keep(keep)) return RTX_E_BADARG;
    return dispatch(dtype, [&](auto t) -> int {
        if (N == 0) return 0;
        CK(cudaSetDevice(ctx->device));
        return trace_host<decltype(t)>(ctx, surf, S, rot0, N, y0, u0, clip, keep, Y, U, I, T,
                                       flags);
    });
}

int rtx_set_mask_output(rtx_ctx* ctx, uint32_t* dmask) {
    if (!ctx) return RTX_E_BADARG;
    ctx->mask = dmask;
    return 0;
}

int rtx_set_path_sum_output(rtx_ctx* ctx, void* dsum, int upto) {
    if (!ctx) return RTX_E_BADARG;
    ctx->tsum = dsum;
    ctx->tsum_upto = upto;
    return 0;
}

int rtx_ipc_export(rtx_ctx* ctx, void* dptr, unsigned char* handle) {
    if (!ctx || !dptr || !handle) return RTX_E_BADARG;
    static_assert(sizeof(cudaIpcMemHandle_t) == RTX_IPC_HANDLE_BYTES, "ipc handle size");
    CK(cudaSetDevice(ctx->device));
    cudaIpcMemHandle_t h;
    CK(cudaIpcGetMemHandle(&h, dptr));
    memcpy(handle, &h, sizeof(h));
    return 0;
}
int rtx_ipc_open(rtx_ctx* ctx, const unsigned char* handle, void** dptr) {
    if (!ctx || !dptr || !handle) return RTX_E_BADARG;
    CK(cudaSetDevice(ctx->device));
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, sizeof(h));
    CK(cudaIpcOpenMemHandle(dptr, h, cudaIpcMemLazyEnablePeerAccess));
    return 0;
}
int rtx_ipc_close(rtx_ctx* ctx, void* dptr) {
    if (!ctx) return RTX_E_BADARG;
    CK(cudaSetDevice(ctx->device));
    CK(cudaIpcCloseMemHandle(dptr));
    return 0;
}

int rtx_trace_gather(rtx_ctx* ctx, const rtx_surface* surf, int S, const double* rot0, int dtype,
                     int64_t N, const void* y0, const void* u0, int clip, int npeers,
                     void* const* dst, void* const* dst_i, int64_t dst_offset, unsigned flags) {
    if (!ctx) return RTX_E_BADARG;
    int rc = check_march(surf, S, N, y0, u0);
    if (rc) return rc;
    if (npeers < 1 || npeers > 8 || !dst || dst_offset < 0) return RTX_E_BADARG;
    return dispatch(dtype, [&](auto t) -> int {
        if (N == 0) return 0;
        PeerDst pd;
        pd.n = npeers;
        pd.off = dst_offset;
        pd.has_i = dst_i != nullptr;
        pd.xy = (flags & RTX_GATHER_XY) != 0;
        for (int k = 0; k < npeers; ++k) {
            if (!dst[k] || (dst_i && !dst_i[k])) return RTX_E_BADARG;
            pd.ptr[k] = dst[k];
            if (dst_i) pd.ptr_i[k] = dst_i[k];
        }
        CK(cudaSetDevice(ctx->device));
        const long long ld = ((N + 127) / 128) * 128;  // only the gather destinations are written
        return timed(ctx, [&] {
            Launch<decltype(t)> L(surf, S, rot0, clip, RTX_KEEP_LAST, ld, flags);
            L.peers = &pd;
            return trace_registered(ctx, L, surf, N, y0, u0, nullptr, nullptr, nullptr, nullptr);
        });
    });
}

}  // extern "C"

namespace {
// rtx_selftest_*: uploads the K arrays `in` of in_bytes each, runs
// launch(grid, d) with d[0..K) the device inputs and d[K] the output of
// out_bytes over n items, and downloads that output to `out`
template <size_t K, typename F>
int selftest(rtx_ctx* ctx, long long n, const void* const (&in)[K], size_t in_bytes, void* out,
             size_t out_bytes, F&& launch) {
    CK(cudaSetDevice(ctx->device));
    DeviceBuf d[K + 1];
    for (size_t k = 0; k < K; ++k) CK(d[k].alloc(in_bytes));
    CK(d[K].alloc(out_bytes));
    for (size_t k = 0; k < K; ++k)
        CK(cudaMemcpyAsync(d[k].get(), in[k], in_bytes, cudaMemcpyHostToDevice, ctx->stream));
    launch((unsigned)((n + 255) / 256), d);
    ctx->launches++;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(out, d[K].get(), out_bytes, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return 0;
}

// rtx_moments, rtx_focus_moments: the 8 sums, zeroed, then added to by
// launch(grid, sums) when N > 0, copied to m
template <typename F>
int moments(rtx_ctx* ctx, long long N, double* m, F&& launch) {
    CK(cudaSetDevice(ctx->device));
    Workspace& acc = ctx->ws[WS_MOMENTS];
    int rc = reserve(acc, 8 * sizeof(double));
    if (rc) return rc;
    CK(cudaMemsetAsync(acc.p, 0, 8 * sizeof(double), ctx->stream));
    if (N > 0) {
        launch(cap_grid(ctx, (N + 255) / 256, 8), (double*)acc.p);
        ctx->launches++;
        CK(cudaGetLastError());
    }
    CK(cudaMemcpyAsync(m, acc.p, 8 * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return 0;
}
}  // namespace

extern "C" {

int rtx_selftest_math(rtx_ctx* ctx, int64_t n, const double* a, const double* b, double* out) {
    if (!ctx || n < 1 || !a || !b || !out) return RTX_E_BADARG;
    const size_t v = n * sizeof(double);
    return selftest(ctx, n, {a, b}, v, out, 6 * v, [&](unsigned grid, const DeviceBuf* d) {
        selftest_math_kernel<<<grid, 256, 0, ctx->stream>>>(d[0].as<double>(), d[1].as<double>(),
                                                            d[2].as<double>(), n);
    });
}

int rtx_selftest_math2(rtx_ctx* ctx, int64_t n, const double* a, const double* b,
                       const double* c, double* out) {
    if (!ctx || n < 1 || !a || !b || !c || !out) return RTX_E_BADARG;
    const size_t v = n * sizeof(double);
    return selftest(ctx, n, {a, b, c}, v, out, 7 * v, [&](unsigned grid, const DeviceBuf* d) {
        selftest_math2_kernel<<<grid, 256, 0, ctx->stream>>>(
            d[0].as<double>(), d[1].as<double>(), d[2].as<double>(), d[3].as<double>(), n);
    });
}

int rtx_moments(rtx_ctx* ctx, int dtype, int64_t N, const void* y, const void* w,
                const double* center, double* m) {
    if (!ctx || !y || !m || N < 0) return RTX_E_BADARG;
    const double cx = center ? center[0] : 0.0, cy = center ? center[1] : 0.0;
    return dispatch(dtype, [&](auto t) {
        using T = decltype(t);
        return moments(ctx, N, m, [&](unsigned grid, double* acc) {
            moments_kernel<T><<<grid, 256, 0, ctx->stream>>>((const T*)y, (const T*)w, N, cx, cy,
                                                             acc);
        });
    });
}

}  // extern "C"

namespace {
// one persistent wave of epi_kernel over `tiles` tiles of EPI_TILE rays, the
// staged table of p.S records in dynamic shared memory
template <typename T, int MODE>
int launch_epi_kernel(rtx_ctx* ctx, unsigned flags, long long tiles, const EpiParams<T>& p) {
    constexpr int RPT = 2, threads = 256;
    static_assert(threads * RPT == EPI_TILE, "epi_kernel's tile");
    // the table, its barrier and (EPI_OTF, EPI_ZRN) the tile's staged rays
    size_t smem = (((size_t)p.S * sizeof(DevSurf<T>) + 127) & ~size_t(127)) +
                  (MODE == EPI_OTF   ? 128 + 4 * EPI_TILE * sizeof(double)
                   : MODE == EPI_ZRN ? 128 + zrn_smem_doubles(p.zrn_order) * sizeof(double)
                                     : 16);
    if ((int)smem > ctx->max_smem_optin) return RTX_E_UNSUPPORTED;
    auto go = [&](auto kern) -> int {
        if (smem > 48 * 1024)
            CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        int occ = 0;
        CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, threads, smem));
        if (occ < 1) occ = 1;
        long long grid = (long long)ctx->sm_count * occ;
        if (grid > tiles) grid = tiles;
        if (grid < 1) grid = 1;
        kern<<<(unsigned)grid, threads, smem, ctx->stream>>>(p);
        ctx->launches++;
        return (int)cudaGetLastError();
    };
    if constexpr (sizeof(T) == 8) {
        if (flags & RTX_EXACT) return go(epi_kernel<T, true, RPT, MODE>);
    }
    return go(epi_kernel<T, false, RPT, MODE>);
}

template <typename T, int MODE>
int launch_epi(rtx_ctx* ctx, const rtx_surface* surf, int S, const double* rot0, long long N,
               const void* y0, const void* u0, int clip, unsigned flags, EpiParams<T>& p) {
    const DevSurf<T>* table = nullptr;
    int rc = upload_table<T>(ctx, surf, S, ctx->stream, &table);
    if (rc) return rc;
    p.table = table;
    p.S = S;
    p.clip = clip ? 1 : 0;
    p.has_rot0 = rot0 != nullptr;
    if (rot0)
        for (int i = 0; i < 9; ++i) p.rot0[i] = (T)rot0[i];
    p.N = N;
    p.y0 = (const T*)y0;
    p.u0 = (const T*)u0;
    if ((flags & RTX_EXACT) && sizeof(T) == 4) return RTX_E_UNSUPPORTED;
    return launch_epi_kernel<T, MODE>(ctx, flags, (N + EPI_TILE - 1) / EPI_TILE, p);
}

// rtx_trace_reduce, rtx_trace_opd, rtx_trace_spot: the timed fused march of
// N > 0 rays with the epilogue MODE, whose EpiParams members fill(p) sets
template <int MODE, typename T, typename F>
int trace_epi(rtx_ctx* ctx, T, const rtx_surface* surf, int S, const double* rot0, long long N,
              const void* y0, const void* u0, int clip, unsigned flags, F&& fill) {
    EpiParams<T> p;
    memset(&p, 0, sizeof(p));
    fill(p);
    return timed(ctx, [&] {
        return launch_epi<T, MODE>(ctx, surf, S, rot0, N, y0, u0, clip, flags, p);
    });
}
}  // namespace

extern "C" {

int rtx_trace_reduce(rtx_ctx* ctx, const rtx_surface* surf, int S, const double* rot0, int dtype,
                     int64_t N, const void* y0, const void* u0, int clip, const void* w,
                     const double* center, double* m, unsigned flags) {
    if (!ctx || !m) return RTX_E_BADARG;
    int rc = check_march(surf, S, N, y0, u0);
    if (rc) return rc;
    return dispatch(dtype, [&](auto t) -> int {
        using T = decltype(t);
        CK(cudaSetDevice(ctx->device));
        Workspace& acc = ctx->ws[WS_EPI];
        int rc = reserve(acc, RTX_NMOMENTS * sizeof(double));
        if (rc) return rc;
        CK(cudaMemsetAsync(acc.p, 0, RTX_NMOMENTS * sizeof(double), ctx->stream));
        if (N > 0) {
            rc = trace_epi<EPI_REDUCE>(ctx, t, surf, S, rot0, N, y0, u0, clip, flags, [&](auto& p) {
                p.w = (const T*)w;
                for (int k = 0; k < 2; ++k) {
                    p.cy[k] = center ? center[k] : 0.0;
                    p.cu[k] = center ? center[2 + k] : 0.0;
                }
                p.out = (double*)acc.p;
            });
            if (rc) return rc;
        }
        CK(cudaMemcpyAsync(m, acc.p, RTX_NMOMENTS * sizeof(double), cudaMemcpyDeviceToHost,
                           ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        return 0;
    });
}

}  // extern "C"

namespace {
// rtx_trace_reduce_many (MODE EPI_MANY, W = RTX_NMOMENTS, centres of 4
// doubles), rtx_trace_otf_many (EPI_OTF, W its row width, centres of 2) and
// rtx_trace_opd_many (EPI_WFE, W = RTX_NMOMENTS, no centres) and
// rtx_trace_zernike_many (EPI_ZRN, W = zrn_row, no centres): the launch-wide
// tile list, the epilogue kernel over it, then the second pass that adds
// each item's W-wide tile rows in tile order into out (host, (nitems, W)).
// `consts` go to the device after the items (EPI_OTF: z, nu; EPI_WFE: the
// WfeItem of every item; EPI_ZRN: those, then every item's rho).
template <typename T, int MODE>
int trace_many(rtx_ctx* ctx, int nt, const rtx_surface* tables, int S, const double* rot0,
               const int64_t* N, const void* const* y0, const void* const* u0, long long nitems,
               const int32_t* item_table, const int32_t* item_bundle, const double* centers,
               int cstride, int clip, int W, const std::vector<double>& consts, double* out,
               unsigned flags, EpiParams<T>& p) {
    // the launch-wide tile list: item i owns tiles tile0 .. tile0 + ceil(N/512) - 1
    std::vector<EpiItem> items((size_t)nitems);
    long long tiles = 0;
    for (long long i = 0; i < nitems; ++i) {
        EpiItem& it = items[(size_t)i];
        const int b = item_bundle[i];
        it.y0 = y0[b];
        it.u0 = u0[b];
        it.N = N[b];
        it.tile0 = tiles;
        it.table = item_table[i];
        for (int k = 0; k < 2; ++k) {
            it.cy[k] = centers ? centers[cstride * i + k] : 0.0;
            it.cu[k] = centers && cstride == 4 ? centers[cstride * i + 2 + k] : 0.0;
        }
        tiles += (N[b] + EPI_TILE - 1) / EPI_TILE;
    }
    // one workspace: tables | items | consts | tile rows | item rows
    auto up = [](size_t b) { return (b + 255) & ~size_t(255); };
    const size_t tb = up((size_t)nt * S * sizeof(DevSurf<T>)), ib = up(items.size() * sizeof(EpiItem));
    const size_t cb = up(consts.size() * sizeof(double));
    const size_t row = (size_t)W * sizeof(double);
    if ((unsigned long long)nitems > (SIZE_MAX - tb - ib - cb) / (2 * row)) return RTX_E_NOMEM;
    const size_t mb = (size_t)nitems * row;
    if ((unsigned long long)tiles > (SIZE_MAX - tb - ib - cb - mb) / (row + 1)) return RTX_E_NOMEM;
    const size_t pb = up((size_t)tiles * row);
    CK(cudaSetDevice(ctx->device));
    Workspace& ws = ctx->ws[WS_MANY];
    int rc = reserve(ws, tb + ib + cb + pb + mb);
    if (rc) return rc;
    unsigned char* base = (unsigned char*)ws.p;
    DevSurf<T>* dtab = (DevSurf<T>*)base;
    EpiItem* ditems = (EpiItem*)(base + tb);
    double* dconsts = (double*)(base + tb + ib);
    double* part = (double*)(base + tb + ib + cb);
    double* dm = (double*)(base + tb + ib + cb + pb);
    std::vector<DevSurf<T>> host((size_t)nt * S);
    for (size_t r = 0; r < host.size(); ++r) convert_surface<T>(tables[r], host[r]);
    CK(cudaMemcpyAsync(dtab, host.data(), host.size() * sizeof(DevSurf<T>), cudaMemcpyHostToDevice,
                       ctx->stream));
    CK(cudaMemcpyAsync(ditems, items.data(), items.size() * sizeof(EpiItem),
                       cudaMemcpyHostToDevice, ctx->stream));
    if (!consts.empty())
        CK(cudaMemcpyAsync(dconsts, consts.data(), consts.size() * sizeof(double),
                           cudaMemcpyHostToDevice, ctx->stream));
    p.table = dtab;
    p.S = S;
    p.clip = clip ? 1 : 0;
    p.has_rot0 = rot0 != nullptr;
    if (rot0)
        for (int i = 0; i < 9; ++i) p.rot0[i] = (T)rot0[i];
    p.items = ditems;
    p.nitems = nitems;
    p.tiles = tiles;
    p.part = part;
    p.otf_zf = dconsts;
    if constexpr (MODE == EPI_WFE || MODE == EPI_ZRN) p.wfe = reinterpret_cast<const WfeItem*>(dconsts);
    if constexpr (MODE == EPI_ZRN) p.zrn_rho = dconsts + (size_t)nitems * WFE_ITEM_DOUBLES;
    rc = timed(ctx, [&]() -> int {
        if (tiles > 0) {
            int rc = launch_epi_kernel<T, MODE>(ctx, flags, tiles, p);
            if (rc) return rc;
        }
        if constexpr (MODE == EPI_MANY || MODE == EPI_WFE)
            many_sum_kernel<<<cap_grid(ctx, (nitems * RTX_NMOMENTS + 255) / 256, 8), 256, 0,
                              ctx->stream>>>(ditems, nitems, part, dm);
        else
            many_rows_kernel<MODE == EPI_ZRN>
                <<<cap_grid(ctx, (nitems * W + 255) / 256, 8), 256, 0, ctx->stream>>>(
                    ditems, nitems, W, part, dm);
        ctx->launches++;
        return (int)cudaGetLastError();
    });
    if (rc) return rc;
    CK(cudaMemcpyAsync(out, dm, mb, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return 0;
}

// the refusals rtx_trace_reduce_many, rtx_trace_otf_many,
// rtx_trace_opd_many and rtx_trace_zernike_many share
int check_many(rtx_ctx* ctx, int nt, const rtx_surface* tables, int S, int nb, const int64_t* N,
               const void* const* y0, const void* const* u0, int64_t nitems,
               const int32_t* item_table, const int32_t* item_bundle) {
    if (!ctx || !tables || !N || !y0 || !u0 || !item_table || !item_bundle) return RTX_E_BADARG;
    if (nt < 1 || nb < 1 || nitems < 1 || S < 1 || S > RTX_MAX_SURFACES) return RTX_E_BADARG;
    for (int t = 0; t < nt; ++t) {
        int rc = check_table(tables + (size_t)t * S, S);
        if (rc) return rc;
    }
    for (int b = 0; b < nb; ++b)
        if (N[b] < 0 || (N[b] > 0 && (!y0[b] || !u0[b]))) return RTX_E_BADARG;
    for (long long i = 0; i < nitems; ++i)
        if (item_table[i] < 0 || item_table[i] >= nt || item_bundle[i] < 0 ||
            item_bundle[i] >= nb)
            return RTX_E_BADARG;
    return 0;
}
}  // namespace

extern "C" {

int rtx_trace_reduce_many(rtx_ctx* ctx, int nt, const rtx_surface* tables, int S,
                          const double* rot0, int dtype, int nb, const int64_t* N,
                          const void* const* y0, const void* const* u0, int64_t nitems,
                          const int32_t* item_table, const int32_t* item_bundle,
                          const double* centers, int clip, double* m, unsigned flags) {
    if (!m) return RTX_E_BADARG;
    int rc = check_many(ctx, nt, tables, S, nb, N, y0, u0, nitems, item_table, item_bundle);
    if (rc) return rc;
    return dispatch(dtype, [&](auto t) -> int {
        using T = decltype(t);
        if ((flags & RTX_EXACT) && sizeof(T) == 4) return RTX_E_UNSUPPORTED;
        EpiParams<T> p;
        memset(&p, 0, sizeof(p));
        return trace_many<T, EPI_MANY>(ctx, nt, tables, S, rot0, N, y0, u0, nitems, item_table,
                                       item_bundle, centers, 4, clip, RTX_NMOMENTS, {}, m, flags,
                                       p);
    });
}

int rtx_trace_otf_many(rtx_ctx* ctx, int nt, const rtx_surface* tables, int S, const double* rot0,
                       int dtype, int nb, const int64_t* N, const void* const* y0,
                       const void* const* u0, int64_t nitems, const int32_t* item_table,
                       const int32_t* item_bundle, const double* centers, int clip, int planes,
                       const double* z, int nfreq, const double* freqs, double* sums,
                       int64_t* count, unsigned flags) {
    if (!sums || !count || !z || !freqs) return RTX_E_BADARG;
    int rc = check_many(ctx, nt, tables, S, nb, N, y0, u0, nitems, item_table, item_bundle);
    if (rc) return rc;
    if (planes < 1 || planes > RTX_OTF_MAX_PLANES || nfreq < 1 || nfreq > RTX_OTF_MAX_FREQS)
        return RTX_E_BADARG;
    const int K = planes, F = nfreq, W = 4 * K * F + K;
    std::vector<double> consts(z, z + K);
    consts.insert(consts.end(), freqs, freqs + F);
    bool finite = true;
    for (double v : consts) finite = finite && std::isfinite(v);
    for (long long i = 0; centers && i < 2 * nitems; ++i) finite = finite && std::isfinite(centers[i]);
    if (!finite) return RTX_E_BADARG;
    return dispatch(dtype, [&](auto t) -> int {
        using T = decltype(t);
        if ((flags & RTX_EXACT) && sizeof(T) == 4) return RTX_E_UNSUPPORTED;
        EpiParams<T> p;
        memset(&p, 0, sizeof(p));
        p.otf_K = K;
        p.otf_F = F;
        p.otf_W = W;
        std::vector<double> rows((size_t)nitems * W);
        int rc = trace_many<T, EPI_OTF>(ctx, nt, tables, S, rot0, N, y0, u0, nitems, item_table,
                                        item_bundle, centers, 2, clip, W, consts, rows.data(),
                                        flags, p);
        if (rc) return rc;
        for (long long i = 0; i < nitems; ++i) {
            const double* r = rows.data() + (size_t)i * W;
            memcpy(sums + (size_t)i * 4 * K * F, r, (size_t)4 * K * F * sizeof(double));
            for (int k = 0; k < K; ++k) count[(size_t)i * K + k] = (int64_t)r[4 * K * F + k];
        }
        return 0;
    });
}

}  // extern "C"

namespace {
// every item's WfeItem (rtx_trace_opd_many's and rtx_trace_zernike_many's
// device constants) into consts, checked before any device work
int wfe_items(long long nitems, const rtx_opd* specs, const double* a0, const double* centers,
              std::vector<double>& consts) {
    consts.assign((size_t)nitems * WFE_ITEM_DOUBLES, 0.0);
    for (long long i = 0; i < nitems; ++i) {
        const rtx_opd& o = specs[i];
        WfeItem w;
        for (int k = 0; k < 3; ++k) {
            w.y0r[k] = o.y0_ref[k];
            w.u0r[k] = o.u0_ref[k];
            w.d[k] = o.d[k];
        }
        for (int k = 0; k < 9; ++k) w.M[k] = o.M[k];
        w.n0 = o.n0;
        w.n_after = o.n_after;
        w.radius = o.radius;
        w.infinite = o.infinite ? 1.0 : 0.0;
        w.a0 = a0 ? a0[i] : 0.0;
        w.c[0] = centers ? centers[2 * i] : 0.0;
        w.c[1] = centers ? centers[2 * i + 1] : 0.0;
        const double* v = reinterpret_cast<const double*>(&w);
        for (int k = 0; k < WFE_ITEM_DOUBLES; ++k)
            if (!std::isfinite(v[k])) return RTX_E_BADARG;
        if (w.radius == 0.0) return RTX_E_BADARG;
        memcpy(consts.data() + (size_t)i * WFE_ITEM_DOUBLES, &w, sizeof(w));
    }
    return 0;
}
}  // namespace

extern "C" {

int rtx_trace_opd_many(rtx_ctx* ctx, int nt, const rtx_surface* tables, int S, const double* rot0,
                       int dtype, int nb, const int64_t* N, const void* const* y0,
                       const void* const* u0, int64_t nitems, const int32_t* item_table,
                       const int32_t* item_bundle, const rtx_opd* specs, const double* a0,
                       const double* centers, int clip, double* sums, unsigned flags) {
    static_assert(RTX_WFE_NSUMS == WFE_NSUMS && WFE_NSUMS <= RTX_NMOMENTS, "rtx_trace_opd_many's row");
    if (!sums || !specs) return RTX_E_BADARG;
    int rc = check_many(ctx, nt, tables, S, nb, N, y0, u0, nitems, item_table, item_bundle);
    if (rc) return rc;
    std::vector<double> consts;
    rc = wfe_items(nitems, specs, a0, centers, consts);
    if (rc) return rc;
    return dispatch(dtype, [&](auto t) -> int {
        using T = decltype(t);
        if constexpr (sizeof(T) != 8) {
            return RTX_E_UNSUPPORTED;  // an FP32 path sum of a long track is worth ~0.02 waves
        } else {
            EpiParams<T> p;
            memset(&p, 0, sizeof(p));
            std::vector<double> rows((size_t)nitems * RTX_NMOMENTS);
            int rc = trace_many<T, EPI_WFE>(ctx, nt, tables, S, rot0, N, y0, u0, nitems,
                                            item_table, item_bundle, nullptr, 2, clip,
                                            RTX_NMOMENTS, consts, rows.data(), flags, p);
            if (rc) return rc;
            for (long long i = 0; i < nitems; ++i)
                memcpy(sums + (size_t)i * RTX_WFE_NSUMS, rows.data() + (size_t)i * RTX_NMOMENTS,
                       RTX_WFE_NSUMS * sizeof(double));
            return 0;
        }
    });
}

int rtx_trace_zernike_many(rtx_ctx* ctx, int nt, const rtx_surface* tables, int S,
                           const double* rot0, int dtype, int nb, const int64_t* N,
                           const void* const* y0, const void* const* u0, int64_t nitems,
                           const int32_t* item_table, const int32_t* item_bundle,
                           const rtx_opd* specs, const double* a0, const double* centers, int clip,
                           int order, const double* rho, double* sums, double* r2max,
                           unsigned flags) {
    static_assert(RTX_ZRN_MAX_ORDER == ZRN_MAX_ORDER, "rtx_trace_zernike_many's orders");
    if (!sums || !specs || !rho || !r2max) return RTX_E_BADARG;
    int rc = check_many(ctx, nt, tables, S, nb, N, y0, u0, nitems, item_table, item_bundle);
    if (rc) return rc;
    if (order < 0 || order > RTX_ZRN_MAX_ORDER) return RTX_E_BADARG;
    std::vector<double> consts;
    rc = wfe_items(nitems, specs, a0, centers, consts);
    if (rc) return rc;
    for (long long i = 0; i < nitems; ++i)
        if (!(std::isfinite(rho[i]) && rho[i] > 0.0)) return RTX_E_BADARG;
    consts.insert(consts.end(), rho, rho + nitems);
    return dispatch(dtype, [&](auto t) -> int {
        using T = decltype(t);
        if constexpr (sizeof(T) != 8) {
            return RTX_E_UNSUPPORTED;  // as rtx_trace_opd_many
        } else {
            EpiParams<T> p;
            memset(&p, 0, sizeof(p));
            p.zrn_order = order;
            const int W = zrn_row(order), E = W - 1;
            std::vector<double> rows((size_t)nitems * W);
            int rc = trace_many<T, EPI_ZRN>(ctx, nt, tables, S, rot0, N, y0, u0, nitems, item_table,
                                            item_bundle, nullptr, 2, clip, W, consts, rows.data(),
                                            flags, p);
            if (rc) return rc;
            for (long long i = 0; i < nitems; ++i) {
                const double* r = rows.data() + (size_t)i * W;
                memcpy(sums + (size_t)i * E, r, (size_t)E * sizeof(double));
                r2max[i] = r[E];
            }
            return 0;
        }
    });
}

int rtx_trace_opd(rtx_ctx* ctx, const rtx_surface* surf, int S, const double* rot0, int dtype,
                  int64_t N, const void* y0, const void* u0, int clip, const rtx_opd* opd, void* A,
                  void* P, unsigned flags) {
    if (!ctx || !opd || !A || !P) return RTX_E_BADARG;
    int rc = check_march(surf, S, N, y0, u0);
    if (rc) return rc;
    if (opd->radius == 0.0) return RTX_E_BADARG;
    return dispatch(dtype, [&](auto t) -> int {
        using T = decltype(t);
        if (N == 0) return 0;
        CK(cudaSetDevice(ctx->device));
        return trace_epi<EPI_OPD>(ctx, t, surf, S, rot0, N, y0, u0, clip, flags, [&](auto& p) {
            p.infinite = opd->infinite;
            for (int k = 0; k < 3; ++k) {
                p.y0r[k] = opd->y0_ref[k];
                p.u0r[k] = opd->u0_ref[k];
                p.d[k] = opd->d[k];
            }
            for (int k = 0; k < 9; ++k) p.M[k] = opd->M[k];
            p.n0 = opd->n0;
            p.n_after = opd->n_after;
            p.radius = opd->radius;
            p.A = (T*)A;
            p.P = (T*)P;
        });
    });
}

}  // extern "C"

namespace {
// rtx_spot -> SpotDev with every check include/rtx.h lists (host only: no
// device work before a refusal)
int spot_to_dev(const rtx_spot* s, const uint64_t* counts, const double* extent, SpotDev& d) {
    if (!s || (!counts && !extent)) return RTX_E_BADARG;
    if (s->planes < 1 || s->planes > RTX_SPOT_MAX_PLANES) return RTX_E_BADARG;
    if (s->radial != 0 && s->radial != 1) return RTX_E_BADARG;
    if (s->nx < 1 || s->ny < 1 || (s->radial && s->ny != 1)) return RTX_E_BADARG;
    const long long lim = 1LL << 31;
    if (s->nx >= lim || s->ny >= lim) return RTX_E_BADARG;
    const long long kn = (long long)s->planes * s->nx;
    if (kn >= lim || kn * s->ny >= lim) return RTX_E_BADARG;
    memset(&d, 0, sizeof(d));
    d.K = s->planes;
    d.radial = s->radial;
    d.nx = (int)s->nx;
    d.ny = (int)s->ny;
    for (int a = 0; a < (s->radial ? 1 : 2); ++a) {
        const double lo = s->range[a][0], hi = s->range[a][1];
        if (!std::isfinite(lo) || !std::isfinite(hi) || !(lo < hi)) return RTX_E_BADARG;
        const double n = (double)(a == 0 ? s->nx : s->ny);
        const double step = (hi - lo) / n;  // np.linspace's step
        if (!std::isnormal(step)) return RTX_E_BADARG;
        d.lo[a] = lo;
        d.hi[a] = hi;
        d.step[a] = step;
        d.inv[a] = n / (hi - lo);
    }
    for (int k = 0; k < s->planes; ++k) {
        if (!std::isfinite(s->z[k]) || !std::isfinite(s->o[k][0]) || !std::isfinite(s->o[k][1]))
            return RTX_E_BADARG;
        d.z[k] = s->z[k];
        d.o[k][0] = s->o[k][0];
        d.o[k][1] = s->o[k][1];
    }
    d.c[0] = s->c[0];  // a NaN centre (a vignetted chief ray) is allowed: nothing is counted
    d.c[1] = s->c[1];
    d.counts = (unsigned long long*)counts;
    return 0;
}

// the context's tally / extent accumulator, zeroed on the stream
int spot_acc(rtx_ctx* ctx, SpotDev& d) {
    Workspace& acc = ctx->ws[WS_SPOT];
    int rc = reserve(acc, 5 * RTX_SPOT_MAX_PLANES * sizeof(unsigned long long));
    if (rc) return rc;
    CK(cudaMemsetAsync(acc.p, 0, 5 * d.K * sizeof(unsigned long long), ctx->stream));
    d.acc = (unsigned long long*)acc.p;
    return 0;
}

int spot_finish(rtx_ctx* ctx, const SpotDev& d, uint64_t* tally, double* extent) {
    const int K = d.K;
    unsigned long long h[5 * RTX_SPOT_MAX_PLANES];
    CK(cudaMemcpyAsync(h, d.acc, 5 * K * sizeof(unsigned long long), cudaMemcpyDeviceToHost,
                       ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    if (tally)
        for (int t = 0; t < 2 * K; ++t) tally[t] = h[t];
    if (extent)
        for (int t = 0; t < 3 * K; ++t) {
            memcpy(extent + t, h + 2 * K + t, sizeof(double));
            if (t % 3 == 2 && !d.radial) extent[t] = std::sqrt(extent[t]);  // the kernel kept r^2
        }
    return 0;
}
}  // namespace

extern "C" {

int rtx_trace_spot(rtx_ctx* ctx, const rtx_surface* surf, int S, const double* rot0, int dtype,
                   int64_t N, const void* y0, const void* u0, int clip, const rtx_spot* spot,
                   uint64_t* counts, uint64_t* tally, double* extent, unsigned flags) {
    SpotDev sd;
    int rc = spot_to_dev(spot, counts, extent, sd);
    if (rc) return rc;
    if (!ctx) return RTX_E_BADARG;
    rc = check_march(surf, S, N, y0, u0);
    if (rc) return rc;
    return dispatch(dtype, [&](auto t) -> int {
        CK(cudaSetDevice(ctx->device));
        int rc = spot_acc(ctx, sd);
        if (rc) return rc;
        if (N > 0) {
            rc = trace_epi<EPI_SPOT>(ctx, t, surf, S, rot0, N, y0, u0, clip, flags,
                                     [&](auto& p) { p.spot = sd; });
            if (rc) return rc;
        }
        return spot_finish(ctx, sd, tally, extent);
    });
}

int rtx_spot_rows(rtx_ctx* ctx, int dtype, int64_t N, const void* y, const void* inc,
                  const rtx_spot* spot, uint64_t* counts, uint64_t* tally, double* extent) {
    SpotDev sd;
    int rc = spot_to_dev(spot, counts, extent, sd);
    if (rc) return rc;
    if (!ctx || N < 0 || !y || !inc) return RTX_E_BADARG;
    return dispatch(dtype, [&](auto t) -> int {
        using T = decltype(t);
        CK(cudaSetDevice(ctx->device));
        int rc = spot_acc(ctx, sd);
        if (rc) return rc;
        if (N > 0) {
            const unsigned grid = cap_grid(ctx, (N + 255) / 256, 8);
            rc = timed(ctx, [&] {
                spot_rows_kernel<T><<<grid, 256, 0, ctx->stream>>>(sd, (const T*)y, (const T*)inc,
                                                                   N);
                ctx->launches++;
                return (int)cudaGetLastError();
            });
            if (rc) return rc;
        }
        return spot_finish(ctx, sd, tally, extent);
    });
}

int rtx_otf_rows(rtx_ctx* ctx, int dtype, int64_t N, const void* y, const void* inc,
                 const rtx_otf* spec, double* sums, int64_t* count) {
    if (!ctx || !spec || !sums || !count || N < 0 || (N > 0 && (!y || !inc)))
        return RTX_E_BADARG;
    if (dtype != RTX_F64 && dtype != RTX_F32) return RTX_E_BADARG;
    const int K = spec->planes, F = spec->nfreq;
    if (K < 1 || K > RTX_OTF_MAX_PLANES || F < 1 || F > RTX_OTF_MAX_FREQS) return RTX_E_BADARG;
    bool finite = std::isfinite(spec->dnu) && std::isfinite(spec->c[0]) &&
                  std::isfinite(spec->c[1]);
    for (int k = 0; k < K; ++k)
        finite = finite && std::isfinite(spec->z[k]) && std::isfinite(spec->o[k][0]) &&
                 std::isfinite(spec->o[k][1]);
    if (!finite) return RTX_E_BADARG;
    const int row = K * 2 * F * 2 + K;  // a slot's sums, then its counts
    const long long slots = (N + RTX_OTF_SLOT - 1) / RTX_OTF_SLOT;
    if (slots == 0) {
        memset(sums, 0, (size_t)(row - K) * sizeof(double));
        memset(count, 0, (size_t)K * sizeof(int64_t));
        return 0;
    }
    OtfDev d;
    memset(&d, 0, sizeof(d));
    d.K = K;
    d.F = F;
    d.units = K * 2 * ((F + OTF_B - 1) / OTF_B);
    d.groups = (d.units + 31) / 32;
    d.dnu = spec->dnu;
    d.c[0] = spec->c[0];
    d.c[1] = spec->c[1];
    for (int k = 0; k < K; ++k) {
        d.z[k] = spec->z[k];
        d.o[k][0] = spec->o[k][0];
        d.o[k][1] = spec->o[k][1];
    }
    return dispatch(dtype, [&](auto t) -> int {
        using T = decltype(t);
        CK(cudaSetDevice(ctx->device));
        Workspace& ws = ctx->ws[WS_OTF];
        const size_t per = (size_t)row * sizeof(double);
        if ((unsigned long long)slots >= SIZE_MAX / per - 1) return RTX_E_NOMEM;
        int rc = reserve(ws, (size_t)(slots + 1) * per);
        if (rc) return rc;
        d.part = (double*)ws.p;
        double* out = d.part + slots * row;
        const long long items = slots * d.groups;
        rc = timed(ctx, [&] {
            otf_rows_kernel<T><<<cap_grid(ctx, items, 2), 256, 0, ctx->stream>>>(
                d, (const T*)y, (const T*)inc, N, items);
            ctx->launches++;
            int rc = (int)cudaGetLastError();
            if (rc) return rc;
            otf_sum_kernel<<<(row + 255) / 256, 256, 0, ctx->stream>>>(d.part, row, slots, out);
            ctx->launches++;
            return (int)cudaGetLastError();
        });
        if (rc) return rc;
        std::vector<double> h((size_t)row);
        CK(cudaMemcpyAsync(h.data(), out, per, cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        memcpy(sums, h.data(), (size_t)(row - K) * sizeof(double));
        for (int k = 0; k < K; ++k) count[k] = (int64_t)h[(size_t)(row - K + k)];
        return 0;
    });
}

}  // extern "C"

namespace {
// a move record as the derivative of the DevSurf<double> members jac_kernel
// reads, added to `d` (several moves of one parameter may share a row)
void add_tangent(const rtx_surface& s, JacTan& d) {
    for (int i = 0; i < 3; ++i) d.off[i] += s.offset[i];
    for (int i = 0; i < 9; ++i) {
        d.rot[i] += s.rot[i];
        if (d.rot[i] != 0.0) d.has_rot = 1;
    }
    d.c += s.c;
    d.k1 += s.k;
    d.kc2 += s.kc2;
    d.n0 += s.n0;
    d.muf += s.muf;
    d.mu2m1 += s.mu2m1;
    for (int i = 0; i < RTX_MAX_ASPH; ++i) {
        d.asph[i] += s.asph[i];
        d.dasph[i] += s.dasph[i];
        if (d.asph[i] != 0.0 || d.dasph[i] != 0.0) d.n_asph = std::max(d.n_asph, i + 1);
    }
}

// rtx_trace_jacobian (dopd NULL: jp holds q, J) and rtx_trace_opd_jacobian
// (jp holds the rtx_opd members, A, dA): the refusals they share, the
// tangent records and the launch
int jacobian_march(rtx_ctx* ctx, const rtx_surface* surf, int S, const double* rot0, int dtype,
                   int64_t N, const void* y0, const void* u0, int clip, int P,
                   const int32_t* param_first, const int32_t* move_row, const rtx_surface* moves,
                   const double* dopd, int64_t ld, unsigned flags, JacParams& jp) {
    if (!ctx || !param_first || !move_row || !moves) return RTX_E_BADARG;
    if (!surf || S < 1 || S > RTX_MAX_SURFACES || N < 0 || !y0 || !u0) return RTX_E_BADARG;
    if (dtype != RTX_F64 || P < 1 || P > RTX_MAX_PARAMS || ld < N) return RTX_E_BADARG;
    if (param_first[0] != 0) return RTX_E_BADARG;
    for (int p = 0; p < P; ++p)
        if (param_first[p + 1] <= param_first[p]) return RTX_E_BADARG;
    for (int m = 0; m < param_first[P]; ++m) {
        if (move_row[m] < 0 || move_row[m] >= S) return RTX_E_BADARG;
        // a row with mu == 1 does not refract (elements.py:356): there is no
        // refraction to differentiate with respect to mu, muf or mu2m1
        const rtx_surface& mv = moves[m];
        if (surf[move_row[m]].mu == 1.0 && (mv.mu != 0.0 || mv.muf != 0.0 || mv.mu2m1 != 0.0))
            return RTX_E_BADARG;
    }
    const bool opd = dopd != nullptr;
    if (opd) {  // rtx_trace_opd_jacobian: P, param_first and move_row are checked above
        for (int i = 0; i < 4 * P; ++i)
            if (!std::isfinite(dopd[i])) return RTX_E_BADARG;
        // the frame change M to the image surface is held fixed: no tilt of
        // surface S-1 (`after`)
        for (int m = 0; m < param_first[P]; ++m)
            if (move_row[m] == S - 1)
                for (int i = 0; i < 9; ++i)
                    if (moves[m].rot[i] != 0.0) return RTX_E_BADARG;
    }
    int rc = check_table(surf, S);
    if (rc) return rc;
    if (N == 0) return 0;
    const int PB = opd ? JAC_OPD_PB : JAC_PB;
    // the tangent records: one per (parameter, moved row), their (P, S) index
    // and the first moved row of each block of PB parameters
    const int nblk = (P + PB - 1) / PB;
    std::vector<int> idx((size_t)P * S, -1), first(nblk, S);
    std::vector<JacTan> tan;
    for (int p = 0; p < P; ++p)
        for (int m = param_first[p]; m < param_first[p + 1]; ++m) {
            int& k = idx[(size_t)p * S + move_row[m]];
            if (k < 0) {
                k = (int)tan.size();
                tan.emplace_back();
                memset(&tan.back(), 0, sizeof(JacTan));
            }
            add_tangent(moves[m], tan[(size_t)k]);
            first[p / PB] = std::min(first[p / PB], (int)move_row[m]);
        }
    auto up = [](size_t b) { return (b + 255) & ~size_t(255); };
    const size_t tb = up(tan.size() * sizeof(JacTan)), xb = up(idx.size() * sizeof(int));
    const size_t fb = up(first.size() * sizeof(int)), db = opd ? (size_t)P * 4 * sizeof(double) : 0;
    CK(cudaSetDevice(ctx->device));
    Workspace& ws = ctx->ws[WS_JAC];
    rc = reserve(ws, tb + xb + fb + db);
    if (rc) return rc;
    unsigned char* base = (unsigned char*)ws.p;
    jp.tan = (const JacTan*)base;
    jp.idx = (const int*)(base + tb);
    jp.first = (const int*)(base + tb + xb);
    // pageable sources: each copy has left the host vector when it returns
    CK(cudaMemcpyAsync(base, tan.data(), tan.size() * sizeof(JacTan), cudaMemcpyHostToDevice,
                       ctx->stream));
    CK(cudaMemcpyAsync(base + tb, idx.data(), idx.size() * sizeof(int), cudaMemcpyHostToDevice,
                       ctx->stream));
    CK(cudaMemcpyAsync(base + tb + xb, first.data(), first.size() * sizeof(int),
                       cudaMemcpyHostToDevice, ctx->stream));
    if (opd) {
        jp.dopd = (const double*)(base + tb + xb + fb);
        CK(cudaMemcpyAsync(base + tb + xb + fb, dopd, db, cudaMemcpyHostToDevice, ctx->stream));
    }
    const DevSurf<double>* table = nullptr;
    rc = upload_table<double>(ctx, surf, S, ctx->stream, &table);
    if (rc) return rc;
    jp.table = table;
    jp.S = S;
    jp.clip = clip ? 1 : 0;
    jp.has_rot0 = rot0 != nullptr;
    if (rot0)
        for (int i = 0; i < 9; ++i) jp.rot0[i] = rot0[i];
    jp.P = P;
    jp.N = N;
    jp.ld = ld;
    jp.y0 = (const double*)y0;
    jp.u0 = (const double*)u0;
    const size_t smem = (((size_t)S * sizeof(DevSurf<double>) + 127) & ~size_t(127)) + 16;
    if ((int)smem > ctx->max_smem_optin) return RTX_E_UNSUPPORTED;
    const bool exact = flags & RTX_EXACT;
    auto kern = opd ? (exact ? jac_kernel<true, JAC_OPD_PB, true> : jac_kernel<false, JAC_OPD_PB, true>)
                    : (exact ? jac_kernel<true, JAC_PB, false> : jac_kernel<false, JAC_PB, false>);
    if (smem > 48 * 1024)
        CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const dim3 grid((unsigned)((N + JAC_THREADS - 1) / JAC_THREADS), (unsigned)nblk);
    return timed(ctx, [&] {
        kern<<<grid, JAC_THREADS, smem, ctx->stream>>>(jp);
        ctx->launches++;
        return (int)cudaGetLastError();
    });
}

// rtx_jacobian_sums (NC = 2) and rtx_wavefront_sums (NC = 1): W outputs of
// the slot sums, then the slots in slot order
template <int NC>
int gauss_newton_sums(rtx_ctx* ctx, int64_t N, int P, const void* q, const void* J, int64_t ld,
                      double c0, double c1, int W, double* out) {
    const long long slots = (N + RTX_JAC_SLOT - 1) / RTX_JAC_SLOT;
    if (slots == 0) {
        memset(out, 0, (size_t)W * sizeof(double));
        return 0;
    }
    CK(cudaSetDevice(ctx->device));
    Workspace& ws = ctx->ws[WS_JSUM];
    const size_t per = (size_t)W * sizeof(double);
    if ((unsigned long long)slots >= SIZE_MAX / per - 1) return RTX_E_NOMEM;
    int rc = reserve(ws, (size_t)(slots + 1) * per);
    if (rc) return rc;
    double* part = (double*)ws.p;
    double* sums = part + slots * W;
    rc = timed(ctx, [&] {
        const dim3 grid((unsigned)slots, (unsigned)((W + JSUM_OUT * 256 - 1) / (JSUM_OUT * 256)));
        jac_sums_kernel<NC><<<grid, 256, 0, ctx->stream>>>((const double*)q, (const double*)J, N,
                                                            ld, P, c0, c1, W, part);
        ctx->launches++;
        int rc = (int)cudaGetLastError();
        if (rc) return rc;
        // the slots in slot order: the same second pass as the OTF sums
        otf_sum_kernel<<<(W + 255) / 256, 256, 0, ctx->stream>>>(part, W, slots, sums);
        ctx->launches++;
        return (int)cudaGetLastError();
    });
    if (rc) return rc;
    CK(cudaMemcpyAsync(out, sums, per, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return 0;
}
}  // namespace

extern "C" {

int rtx_trace_jacobian(rtx_ctx* ctx, const rtx_surface* surf, int S, const double* rot0,
                       int dtype, int64_t N, const void* y0, const void* u0, int clip, int P,
                       const int32_t* param_first, const int32_t* move_row,
                       const rtx_surface* moves, void* q, void* J, int64_t ld, unsigned flags) {
    if (!q || !J) return RTX_E_BADARG;
    JacParams jp;
    memset(&jp, 0, sizeof(jp));
    jp.q = (double*)q;
    jp.J = (double*)J;
    return jacobian_march(ctx, surf, S, rot0, dtype, N, y0, u0, clip, P, param_first, move_row,
                          moves, nullptr, ld, flags, jp);
}

int rtx_trace_opd_jacobian(rtx_ctx* ctx, const rtx_surface* surf, int S, const double* rot0,
                           int dtype, int64_t N, const void* y0, const void* u0, int clip,
                           const rtx_opd* opd, int P, const int32_t* param_first,
                           const int32_t* move_row, const rtx_surface* moves, const double* dopd,
                           void* A, void* dA, int64_t ld, unsigned flags) {
    if (!opd || !A || !dA || (P > 0 && !dopd)) return RTX_E_BADARG;
    if (opd->radius == 0.0 || !std::isfinite(opd->radius)) return RTX_E_BADARG;
    JacParams jp;
    memset(&jp, 0, sizeof(jp));
    jp.infinite = opd->infinite;
    for (int k = 0; k < 3; ++k) {
        jp.y0r[k] = opd->y0_ref[k];
        jp.u0r[k] = opd->u0_ref[k];
        jp.d[k] = opd->d[k];
    }
    for (int k = 0; k < 9; ++k) jp.M[k] = opd->M[k];
    jp.n0 = opd->n0;
    jp.n_after = opd->n_after;
    jp.radius = opd->radius;
    jp.A = (double*)A;
    jp.dA = (double*)dA;
    return jacobian_march(ctx, surf, S, rot0, dtype, N, y0, u0, clip, P, param_first, move_row,
                          moves, dopd, ld, flags, jp);
}

int rtx_jacobian_sums(rtx_ctx* ctx, int64_t N, int P, const void* q, const void* J, int64_t ld,
                      const double* center, double* out) {
    if (!ctx || !out || N < 0 || (N > 0 && (!q || !J))) return RTX_E_BADARG;
    if (P < 1 || P > RTX_MAX_PARAMS || ld < N) return RTX_E_BADARG;
    return gauss_newton_sums<2>(ctx, N, P, q, J, ld, center ? center[0] : 0.0,
                                center ? center[1] : 0.0, 5 + 3 * P + P * (P + 1) / 2, out);
}

int rtx_wavefront_sums(rtx_ctx* ctx, int64_t N, int P, const void* A, const void* dA, int64_t ld,
                       double a0, double* out) {
    if (!ctx || !out || N < 0 || (N > 0 && (!A || (P > 0 && !dA)))) return RTX_E_BADARG;
    if (P < 0 || P > RTX_MAX_PARAMS || ld < N) return RTX_E_BADARG;
    return gauss_newton_sums<1>(ctx, N, P, A, dA, ld, a0, 0.0, 4 + 2 * P + P * (P + 1) / 2, out);
}

int rtx_otf_jacobian_sums(rtx_ctx* ctx, int64_t N, int P, const void* q, int qstride,
                          const void* J, int64_t ld, const double* center, int nfreq,
                          const double* freqs, double* out) {
    if (!ctx || !out || N < 0 || (N > 0 && (!q || (P > 0 && !J)))) return RTX_E_BADARG;
    if (P < 0 || P > RTX_MAX_PARAMS || (qstride != 2 && qstride != 3) || (P > 0 && ld < N))
        return RTX_E_BADARG;
    if (nfreq < 1 || nfreq > RTX_OTF_MAX_FREQS || !freqs) return RTX_E_BADARG;
    bool finite = !center || (std::isfinite(center[0]) && std::isfinite(center[1]));
    for (int j = 0; j < nfreq; ++j) finite = finite && std::isfinite(freqs[j]);
    if (!finite) return RTX_E_BADARG;
    const int F = nfreq, W = RTX_OTF_JAC_WIDTH(P, F);
    const long long slots = (N + RTX_OTF_JAC_SLOT - 1) / RTX_OTF_JAC_SLOT;
    if (slots == 0) {
        memset(out, 0, (size_t)W * sizeof(double));
        return 0;
    }
    OtfJacDev d;
    memset(&d, 0, sizeof(d));
    d.P = P;
    d.F = F;
    d.qstride = qstride;
    d.groups = (2 * F + 31) / 32;
    d.blocks = P > 0 ? (P + OTF_JAC_PB - 1) / OTF_JAC_PB : 1;
    d.ld = P > 0 ? ld : 0;
    d.c[0] = center ? center[0] : 0.0;
    d.c[1] = center ? center[1] : 0.0;
    for (int j = 0; j < F; ++j) d.nu[j] = freqs[j];
    CK(cudaSetDevice(ctx->device));
    Workspace& ws = ctx->ws[WS_OTFJ];
    // slot rows | the call's row | the mask (one bit per ray of every slot)
    const size_t per = (size_t)W * sizeof(double);
    const size_t mask_bytes = (size_t)slots * (RTX_OTF_JAC_SLOT / 8);
    if ((unsigned long long)slots >= (SIZE_MAX - mask_bytes) / per - 1) return RTX_E_NOMEM;
    int rc = reserve(ws, (size_t)(slots + 1) * per + mask_bytes);
    if (rc) return rc;
    d.part = (double*)ws.p;
    double* sums = d.part + slots * W;
    unsigned* mask = (unsigned*)(sums + W);
    d.mask = mask;
    const long long items = slots * d.groups * d.blocks;
    rc = timed(ctx, [&] {
        otf_jac_mask_kernel<<<(unsigned)slots, 256, 0, ctx->stream>>>(
            d, (const double*)q, (const double*)J, N, W, mask);
        ctx->launches++;
        int rc = (int)cudaGetLastError();
        if (rc) return rc;
        otf_jac_kernel<<<cap_grid(ctx, items, 2), 256, 0, ctx->stream>>>(
            d, (const double*)q, (const double*)J, N, W, items);
        ctx->launches++;
        rc = (int)cudaGetLastError();
        if (rc) return rc;
        otf_sum_kernel<<<(W + 255) / 256, 256, 0, ctx->stream>>>(d.part, W, slots, sums);
        ctx->launches++;
        return (int)cudaGetLastError();
    });
    if (rc) return rc;
    CK(cudaMemcpyAsync(out, sums, per, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    // dS = -2 pi i nu T: (re, im) = (2 pi nu T_im, -2 pi nu T_re)
    for (int p = 0; p < P; ++p)
        for (int j = 0; j < 2 * F; ++j) {
            const double k = (2.0 * M_PI) * freqs[j % F];
            double* t = out + 1 + 4 * F + 2 * (p * 2 * F + j);
            const double re = t[0], im = t[1];
            t[0] = k * im;
            t[1] = -(k * re);
        }
    return 0;
}

}  // extern "C"

namespace {
int aim_to_dev(const rtx_aim* a, long long n_given, AimDev& d) {
    memset(&d, 0, sizeof(d));
    d.conjugate = a->conjugate;
    d.grid = a->grid;
    d.filter = a->filter;
    d.curved = a->curved && a->conjugate == 0;
    d.n = a->n;
    d.seed = a->seed;
    memcpy(d.seg, a->seg, sizeof(d.seg));
    d.seg_m[0] = a->seg_m[0];
    d.seg_m[1] = a->seg_m[1];
    memcpy(d.frame, a->frame, sizeof(d.frame));
    d.pmax = a->pmax;
    d.z = a->z;
    for (int k = 0; k < 2; ++k) {
        d.fc[k] = a->fc[k];
        d.fd2[k] = a->fd2[k];
    }
    if (d.curved) {
        if (a->surface.n_asph > RTX_MAX_ASPH) return RTX_E_UNSUPPORTED;
        convert_surface<double>(a->surface, d.surf);
    }
    switch (a->grid) {
        case GRID_GIVEN: d.M = n_given; break;
        case GRID_HEXAPOLAR: d.M = 1 + 3 * a->n * (a->n + 1); break;
        case GRID_SQUARE:
        case GRID_TRIANGULAR:
            if (a->n < 2) return RTX_E_BADARG;
            d.M = 1 + a->n * a->n;
            break;
        case GRID_RANDOM: d.M = 1 + a->n; break;
        case GRID_LINES: d.M = a->seg_m[0] + a->seg_m[1]; break;
        default: return RTX_E_BADARG;
    }
    if (a->n < 0 || d.M < 0 || a->seg_m[0] < 0 || a->seg_m[1] < 0) return RTX_E_BADARG;
    if (a->conjugate != 0 && a->conjugate != 1) return RTX_E_BADARG;
    return 0;
}

// counting pass + prefix sum, cached per (spec, n_given, yp)
int aim_plan(rtx_ctx* ctx, const rtx_aim* spec, long long n_given, const void* yp, AimDev& d) {
    int rc = aim_to_dev(spec, n_given, d);
    if (rc) return rc;
    if (spec->grid == GRID_GIVEN && n_given > 0 && !yp) return RTX_E_BADARG;
    std::vector<unsigned char> key(sizeof(rtx_aim) + sizeof(long long) + sizeof(void*));
    memcpy(key.data(), spec, sizeof(rtx_aim));
    memcpy(key.data() + sizeof(rtx_aim), &n_given, sizeof(long long));
    memcpy(key.data() + sizeof(rtx_aim) + sizeof(long long), &yp, sizeof(void*));
    const bool rejects = spec->filter || spec->grid == GRID_SQUARE || spec->grid == GRID_TRIANGULAR;
    // (a GIVEN grid may have changed behind the same pointer: always recount it)
    if (key == ctx->aim_key && !(rejects && spec->grid == GRID_GIVEN)) return 0;
    ctx->aim_key.clear();
    ctx->aim_offsets.clear();
    ctx->aim_M = d.M;
    ctx->aim_total = d.M;
    if (rejects && d.M > 0) {
        const long long nb = (d.M + AIM_BLOCK - 1) / AIM_BLOCK;
        Workspace& ws = ctx->ws[WS_AIM];
        rc = reserve(ws, (size_t)(nb + 1) * sizeof(long long));
        if (rc) return rc;
        int* d_counts = reinterpret_cast<int*>(ws.p);  // reused before the offsets
        aim_count_kernel<<<cap_grid(ctx, nb, 8), 256, 0, ctx->stream>>>(d, (const double*)yp,
                                                                        d_counts, nb);
        ctx->launches++;
        CK(cudaGetLastError());
        std::vector<int> counts((size_t)nb);
        CK(cudaMemcpyAsync(counts.data(), d_counts, (size_t)nb * sizeof(int), cudaMemcpyDeviceToHost,
                           ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        ctx->aim_offsets.resize((size_t)nb + 1);
        long long acc = 0;
        for (long long b = 0; b < nb; ++b) {
            ctx->aim_offsets[(size_t)b] = acc;
            acc += counts[(size_t)b];
        }
        ctx->aim_offsets[(size_t)nb] = acc;
        ctx->aim_total = acc;
        CK(cudaMemcpyAsync(ws.p, ctx->aim_offsets.data(),
                           (size_t)(nb + 1) * sizeof(long long), cudaMemcpyHostToDevice, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
    }
    ctx->aim_key = key;
    return 0;
}
}  // namespace

extern "C" {

int rtx_aim_plan(rtx_ctx* ctx, const rtx_aim* spec, int64_t n_given, const void* yp,
                 int64_t* n_rays) {
    if (!ctx || !spec || !n_rays || n_given < 0) return RTX_E_BADARG;
    CK(cudaSetDevice(ctx->device));
    AimDev d;
    int rc = aim_plan(ctx, spec, n_given, yp, d);
    if (rc) return rc;
    *n_rays = ctx->aim_total;
    return 0;
}

int rtx_aim_rays(rtx_ctx* ctx, const rtx_aim* spec, int64_t n_given, const void* yp, int dtype,
                 int64_t first, int64_t count, void* y0, void* u0, void* yp_out) {
    if (!ctx || !spec || !y0 || !u0 || n_given < 0 || first < 0 || count < 0) return RTX_E_BADARG;
    return dispatch(dtype, [&](auto t) -> int {
        using T = decltype(t);
        CK(cudaSetDevice(ctx->device));
        AimDev d;
        int rc = aim_plan(ctx, spec, n_given, yp, d);
        if (rc) return rc;
        if (first + count > ctx->aim_total) return RTX_E_BADARG;
        if (count == 0) return 0;
        long long b0, b1;
        const long long* d_off = nullptr;
        if (ctx->aim_offsets.empty()) {
            b0 = first / AIM_BLOCK;
            b1 = (first + count + AIM_BLOCK - 1) / AIM_BLOCK;
        } else {
            const auto& off = ctx->aim_offsets;  // off[b] = rank of block b's first kept ray
            const long long nb = (long long)off.size() - 1;
            long long lo = 0, hi = nb;  // last block with off[b] <= first
            while (lo + 1 < hi) {
                const long long mid = (lo + hi) / 2;
                if (off[(size_t)mid] <= first) lo = mid; else hi = mid;
            }
            b0 = lo;
            b1 = b0;
            while (b1 < nb && off[(size_t)b1] < first + count) ++b1;
            d_off = (const long long*)ctx->ws[WS_AIM].p;
        }
        aim_rays_kernel<T><<<cap_grid(ctx, b1 - b0, 8), 256, 0, ctx->stream>>>(
            d, (const double*)yp, d_off, b0, b1, first, count, (T*)y0, (T*)u0, (double*)yp_out);
        ctx->launches++;
        return (int)cudaGetLastError();
    });
}

int rtx_focus_moments(rtx_ctx* ctx, int dtype, int64_t N, const void* y, const void* inc,
                      const void* w, const double* center, double* m) {
    if (!ctx || !y || !inc || !m || N < 0) return RTX_E_BADARG;
    double c[4] = {0, 0, 0, 0};
    if (center)
        for (int k = 0; k < 4; ++k) c[k] = center[k];
    return dispatch(dtype, [&](auto t) {
        using T = decltype(t);
        return moments(ctx, N, m, [&](unsigned grid, double* acc) {
            focus_moments_kernel<T><<<grid, 256, 0, ctx->stream>>>(
                (const T*)y, (const T*)inc, (const T*)w, N, c[0], c[1], c[2], c[3], acc);
        });
    });
}

}  // extern "C"

// ---- diffraction PSF (GeometricTrace.psf, rayopt/geometric_trace.py:133-169)
extern "C" {

int rtx_grid_linear(rtx_ctx* ctx, int dtype, int64_t M, const void* pts, const void* vals,
                    int64_t T, const int32_t* simplices, const void* transform, int n,
                    const void* gh, void* out, int32_t* winner) {
    // n <= 46340: node indices fit in int32
    if (!ctx || M < 0 || T < 0 || T >= INT_MAX || n < 2 || n > 46340 || !gh || !out)
        return RTX_E_BADARG;
    if ((M > 0 && (!pts || !vals)) || (T > 0 && (!simplices || !transform))) return RTX_E_BADARG;
    int rc = fp64_only(dtype);
    if (rc) return rc;
    CK(cudaSetDevice(ctx->device));
    const long long nn = (long long)n * n;
    int* claim = winner;
    if (!claim) {
        rc = reserve(ctx->ws[WS_WINNER], (size_t)nn * sizeof(int));
        if (rc) return rc;
        claim = (int*)ctx->ws[WS_WINNER].p;
    }
    const unsigned grid = cap_grid(ctx, (nn + 255) / 256, 16);
    return timed(ctx, [&] {
        fill_i32_kernel<<<grid, 256, 0, ctx->stream>>>(claim, nn, INT_MAX);
        ctx->launches++;
        CK(cudaGetLastError());
        if (T > 0) {
            grid_claim_kernel<<<(unsigned)((T + 255) / 256), 256, 0, ctx->stream>>>(
                (const double*)pts, M, simplices, (const double*)transform, T, (const double*)gh, n,
                claim);
            ctx->launches++;
            CK(cudaGetLastError());
        }
        grid_eval_kernel<<<grid, 256, 0, ctx->stream>>>(
            (const double*)vals, simplices, (const double*)transform, (const double*)gh, n, claim,
            (double*)out);
        ctx->launches++;
        return (int)cudaGetLastError();
    });
}

int rtx_psf_bytes(rtx_ctx* ctx, int n, int pad, size_t* bytes) {
    if (!ctx || !bytes || n < 1 || pad < 1) return RTX_E_BADARG;
    const long long nx = (long long)n * pad;
    size_t b = (size_t)(nx * nx) * sizeof(double2);  // the complex grid
    if (!(ctx->fft_planned && ctx->fft_nx == nx && ctx->fft_ny == nx)) {
        const CufftApi& fft = cufft_api();
        if (!fft.ok) return RTX_E_UNSUPPORTED;
        cufftHandle h;
        if (fft.create(&h) != CUFFT_SUCCESS) return RTX_E_UNSUPPORTED;
        long long dims[2] = {nx, nx};
        size_t ws = 0;
        cufftResult r = fft.set_auto_allocation(h, 0);
        if (r == CUFFT_SUCCESS)
            r = fft.get_size_many64(h, 2, dims, nullptr, 1, 0, nullptr, 1, 0, CUFFT_Z2Z, 1, &ws);
        fft.destroy(h);
        if (r != CUFFT_SUCCESS) return r == CUFFT_ALLOC_FAILED ? RTX_E_NOMEM : RTX_E_UNSUPPORTED;
        b += ws;
    }
    *bytes = b;
    return 0;
}

int rtx_psf(rtx_ctx* ctx, int dtype, int n, const void* o, int pad, void* psf, double* stats) {
    if (!ctx || n < 1 || pad < 1 || !o || !psf) return RTX_E_BADARG;
    int rc = fp64_only(dtype);
    if (rc) return rc;
    const CufftApi& fft = cufft_api();
    if (!fft.ok) return RTX_E_UNSUPPORTED;
    CK(cudaSetDevice(ctx->device));
    const long long nx = (long long)n * pad, ny = nx, tot = nx * ny;
    const size_t zbytes = (size_t)tot * sizeof(double2);
    const bool cached = ctx->fft_planned && ctx->fft_nx == nx && ctx->fft_ny == ny;
    size_t free_b = 0, total_b = 0;
    CK(cudaMemGetInfo(&free_b, &total_b));
    // what a new plan would give back
    const size_t avail = free_b + (cached ? 0 : ctx->fft_work_bytes);
    if (zbytes > avail) return RTX_E_NOMEM;  // nothing allocated, the cached plan kept
    if (!cached) {
        cufftHandle h;
        if (fft.create(&h) != CUFFT_SUCCESS) return RTX_E_UNSUPPORTED;
        long long dims[2] = {nx, ny};
        size_t ws = 0;
        cufftResult r = fft.set_auto_allocation(h, 0);
        if (r == CUFFT_SUCCESS)
            r = fft.get_size_many64(h, 2, dims, nullptr, 1, 0, nullptr, 1, 0, CUFFT_Z2Z, 1, &ws);
        if (r == CUFFT_SUCCESS && zbytes + ws > avail) {
            fft.destroy(h);
            return RTX_E_NOMEM;
        }
        release_fft_plan(ctx);
        if (r == CUFFT_SUCCESS)
            r = fft.make_plan_many64(h, 2, dims, nullptr, 1, 0, nullptr, 1, 0, CUFFT_Z2Z, 1, &ws);
        if (r != CUFFT_SUCCESS) {
            fft.destroy(h);
            return r == CUFFT_ALLOC_FAILED ? RTX_E_NOMEM : RTX_E_UNSUPPORTED;
        }
        if (ws && cudaMalloc(&ctx->fft_work, ws) != cudaSuccess) {
            cudaGetLastError();
            fft.destroy(h);
            ctx->fft_work = nullptr;
            return RTX_E_NOMEM;
        }
        if (fft.set_work_area(h, ctx->fft_work) != CUFFT_SUCCESS) {
            fft.destroy(h);
            release_fft_plan(ctx);
            return RTX_E_UNSUPPORTED;
        }
        ctx->fft_plan = h;
        ctx->fft_planned = true;
        ctx->fft_nx = nx;
        ctx->fft_ny = ny;
        ctx->fft_work_bytes = ws;
    }
    if (fft.set_stream(ctx->fft_plan, ctx->stream) != CUFFT_SUCCESS) return RTX_E_UNSUPPORTED;
    // partials (4 per block), the finite count, the 5 stats
    const size_t red_doubles = 4 * PSF_RED_BLOCKS + 1 + 5;
    rc = reserve(ctx->ws[WS_PSF_RED], red_doubles * sizeof(double));
    if (rc) return rc;
    double* part = (double*)ctx->ws[WS_PSF_RED].p;
    auto* count = reinterpret_cast<unsigned long long*>(part + 4 * PSF_RED_BLOCKS);
    double* d_stats = part + 4 * PSF_RED_BLOCKS + 1;
    DeviceBuf grid;  // the complex grid
    if (grid.alloc(zbytes) != cudaSuccess) {
        cudaGetLastError();
        return RTX_E_NOMEM;
    }
    double2* z = grid.as<double2>();
    const long long nn = (long long)n * n;
    CK(cudaMemsetAsync(count, 0, sizeof(unsigned long long), ctx->stream));
    rc = timed(ctx, [&] {
        count_finite_kernel<<<cap_grid(ctx, (nn + 255) / 256, 8), 256, 0, ctx->stream>>>(
            (const double*)o, nn, count);
        pupil_kernel<<<cap_grid(ctx, (tot + 255) / 256, 16), 256, 0, ctx->stream>>>(
            (const double*)o, n, nx, ny, count, z);
        ctx->launches += 2;
        CK(cudaGetLastError());
        if (fft.exec_z2z(ctx->fft_plan, (cufftDoubleComplex*)z, (cufftDoubleComplex*)z,
                         CUFFT_FORWARD) != CUFFT_SUCCESS)
            return RTX_E_UNSUPPORTED;
        intensity_kernel<<<PSF_RED_BLOCKS, 256, 0, ctx->stream>>>(z, nx, ny, (double*)psf, part);
        psf_stats_kernel<<<1, 1, 0, ctx->stream>>>(part, PSF_RED_BLOCKS, count, d_stats);
        ctx->launches += 2;
        return (int)cudaGetLastError();
    });
    if (rc) return rc;
    if (stats)
        CK(cudaMemcpyAsync(stats, d_stats, 5 * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return 0;
}

int rtx_psf_profiles(rtx_ctx* ctx, int dtype, int64_t nx, int64_t ny, const void* psf, double c0,
                     double c1, int64_t nbins, double* ee, double* lsf0, double* lsf1) {
    if (!ctx || !psf || nx < 1 || ny < 1 || !std::isfinite(c0) || !std::isfinite(c1))
        return RTX_E_BADARG;
    int rc = fp64_only(dtype);
    if (rc) return rc;
    if (nx > INT64_MAX / 8 / ny) return RTX_E_BADARG;
    // np.bincount's length: 1 + the largest bin, which sits at a corner
    long long last = 0;
    for (long long I : {0ll, (long long)nx - 1})
        for (long long J : {0ll, (long long)ny - 1}) {
            volatile double i = (double)I - c0, j = (double)J - c1;
            volatile double s = j * j + i * i;
            if (!(s < 0x1p100)) return RTX_E_NOMEM;  // radius >= 2^50: no such histogram fits
            last = std::max(last, profile_bin((double)I, (double)J, c0, c1));
        }
    if (nbins != last + 1) return RTX_E_BADARG;
    CK(cudaSetDevice(ctx->device));
    const long long stride = nbins + nx + ny;
    // PROF_BLOCKS partial rows, their sum, the flag
    const size_t need = ((size_t)(PROF_BLOCKS + 1) * stride + 1) * sizeof(double);
    rc = reserve(ctx->ws[WS_PROF], need);
    if (rc) return rc;
    double* part = (double*)ctx->ws[WS_PROF].p;
    double* out = part + (long long)PROF_BLOCKS * stride;
    int* flag = reinterpret_cast<int*>(out + stride);
    const unsigned grid = cap_grid(ctx, (stride + 255) / 256, 8);
    CK(cudaMemsetAsync(flag, 0, sizeof(int), ctx->stream));
    rc = timed(ctx, [&] {
        profile_tiles_kernel<<<PROF_BLOCKS, PROF_WARPS * 32, 0, ctx->stream>>>(
            (const double*)psf, nx, ny, c0, c1, nbins, part, stride, flag);
        profile_combine_kernel<<<grid, 256, 0, ctx->stream>>>(part, PROF_BLOCKS, stride, out);
        ctx->launches += 2;
        return (int)cudaGetLastError();
    });
    if (rc) return rc;
    int h_flag = 0;
    CK(cudaMemcpyAsync(&h_flag, flag, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    if (ee) CK(cudaMemcpyAsync(ee, out, nbins * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    if (lsf1)
        CK(cudaMemcpyAsync(lsf1, out + nbins, nx * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    if (lsf0)
        CK(cudaMemcpyAsync(lsf0, out + nbins + nx, ny * sizeof(double), cudaMemcpyDeviceToHost,
                           ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    if (h_flag & 1) return RTX_E_BADARG;        // a negative or non-finite pixel
    if (h_flag) return RTX_E_UNSUPPORTED;       // a tile over PROF_TILE_BINS bins: not reached below 2^50
    return 0;
}

}  // extern "C"

// ---- Delaunay triangulation of the exit pupil (rtx_delaunay.cuh) ----------
namespace {

constexpr long long DT_MAX_POINTS = (1ll << 30) - 1;  // 2M slots and the point index fit in int32

// the workspace of M points (slots for 2M triangles) carved from `base`;
// returns its size (base may be NULL to count only)
size_t dt_carve(void* base, long long M, const void* pts, dt::Work* w) {
    const long long S = 2 * M, nb = (S + dt::SCAN_THREADS - 1) / dt::SCAN_THREADS;
    size_t off = 0;
    auto take = [&](size_t bytes) {
        void* p = base ? (char*)base + off : nullptr;
        off += (bytes + 255) / 256 * 256;
        return p;
    };
    dt::Work x{};
    x.p = (const double2*)pts;
    x.M = M;
    x.pick = (unsigned long long*)take(S * 8);
    x.vote = (unsigned long long*)take(S * 8);
    x.ext = (int2*)take(S * 8);
    x.tv = (int*)take(S * 12);
    x.tn = (int*)take(S * 12);
    x.mod = (int*)take(S * 4);
    x.chk = (int*)take(S * 4);
    x.op = (int*)take(S * 4);
    x.flag = (int*)take(S * 4);
    x.rank = (int*)take(S * 4);
    x.bsum = (int*)take((nb + 1) * 4);
    x.loc = (int*)take(M * 4);
    x.cnt = (unsigned*)take(dt::C_N * 4);
    x.lex = (long long*)take((2 * dt::LEX_BLOCKS + 2) * 8);
    x.seed_key = (unsigned long long*)take(8);
    if (w) *w = x;
    return off;
}

}  // namespace

extern "C" {

int rtx_delaunay_bytes(rtx_ctx* ctx, int64_t M, size_t* bytes) {
    if (!ctx || !bytes || M < 3 || M > DT_MAX_POINTS) return RTX_E_BADARG;
    *bytes = dt_carve(nullptr, M, nullptr, nullptr);
    return 0;
}

int rtx_selftest_predicates(rtx_ctx* ctx, int64_t n, const double* pts, int* out) {
    if (!ctx || n < 1 || !pts || !out) return RTX_E_BADARG;
    return selftest(ctx, n, {pts}, 8 * n * sizeof(double), out, 2 * n * sizeof(int),
                    [&](unsigned grid, const DeviceBuf* d) {
                        dt::selftest_predicates_kernel<<<grid, 256, 0, ctx->stream>>>(
                            d[0].as<double>(), n, d[1].as<int>());
                    });
}

int rtx_delaunay(rtx_ctx* ctx, int dtype, int64_t M, const void* pts, int64_t* T, int32_t* simplices,
                 int32_t* neighbors, void* transform) {
    if (!ctx || !pts || !T || !simplices) return RTX_E_BADARG;
    int rc = fp64_only(dtype);
    if (rc) return rc;
    if (M < 3 || M > DT_MAX_POINTS) return RTX_E_BADARG;
    CK(cudaSetDevice(ctx->device));
    rc = reserve(ctx->ws[WS_DT], dt_carve(nullptr, M, nullptr, nullptr));
    if (rc) return rc;
    dt::Work w;
    dt_carve(ctx->ws[WS_DT].p, M, pts, &w);
    cudaStream_t st = ctx->stream;
    const unsigned grid_m = cap_grid(ctx, (M + 255) / 256, 16);  // one thread per point
    unsigned cnt[dt::C_N];
    auto counters = [&]() -> int {  // launches so far checked, counters read back
        CK(cudaGetLastError());
        CK(cudaMemcpyAsync(cnt, w.cnt, sizeof(cnt), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        return 0;
    };
    // exclusive prefix sum of w.flag[0, n) into w.rank; *total = the sum
    auto scan = [&](int n, int* total) -> int {
        const int nb = (n + dt::SCAN_THREADS - 1) / dt::SCAN_THREADS;
        dt::scan_block_kernel<<<nb, dt::SCAN_THREADS, 0, st>>>(w.flag, n, w.bsum);
        dt::scan_top_kernel<<<1, dt::SCAN_THREADS, 0, st>>>(w.bsum, nb);
        dt::scan_apply_kernel<<<nb, dt::SCAN_THREADS, 0, st>>>(w.flag, n, w.bsum, w.rank);
        ctx->launches += 3;
        CK(cudaGetLastError());
        CK(cudaMemcpyAsync(total, w.bsum + nb, sizeof(int), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        return 0;
    };
    auto relocate = [&]() -> int {
        CK(cudaMemsetAsync(w.cnt + dt::C_LEFT, 0, sizeof(unsigned), st));
        dt::relocate_kernel<<<grid_m, 256, 0, st>>>(w, 2 * M + 16);
        ctx->launches++;
        return counters();
    };
    int nfin = 0;
    rc = timed(ctx, [&]() -> int {
        // validation and the seed triangle
        CK(cudaMemsetAsync(w.cnt, 0, dt::C_N * sizeof(unsigned), st));
        CK(cudaMemsetAsync(w.seed_key, 0xff, 8, st));
        dt::lex_kernel<<<dt::LEX_BLOCKS, dt::LEX_THREADS, 0, st>>>(w);
        dt::lex_final_kernel<<<1, 1, 0, st>>>(w);
        CK(cudaGetLastError());
        if (int rc = counters()) return rc;
        if (cnt[dt::C_ERR]) return RTX_E_BADARG;  // non-finite or outside the predicates' domain
        unsigned long long seed = 0;
        dt::seed_kernel<<<grid_m, 256, 0, st>>>(w);
        CK(cudaGetLastError());
        CK(cudaMemcpyAsync(&seed, w.seed_key, 8, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        ctx->launches += 3;
        if (seed == dt::NONE) return RTX_E_BADARG;  // all points collinear
        fill_i32_kernel<<<grid_m, 256, 0, st>>>(w.loc, M, 0);
        dt::init_kernel<<<1, 1, 0, st>>>(w);
        ctx->launches += 2;
        int tcur = 4, stamp = 1;
        if (int rc = relocate()) return rc;
        while (cnt[dt::C_LEFT]) {
            CK(cudaMemsetAsync(w.pick, 0xff, (size_t)tcur * 8, st));
            CK(cudaMemsetAsync(w.vote, 0xff, (size_t)tcur * 8, st));
            unsigned grid = cap_grid(ctx, (tcur + 255) / 256, 16);  // one thread per slot
            dt::pick_kernel<<<grid_m, 256, 0, st>>>(w);
            dt::claim_kernel<<<grid, 256, 0, st>>>(w, tcur);
            dt::decide_kernel<<<grid, 256, 0, st>>>(w, tcur);
            ctx->launches += 3;
            int added = 0;
            if (int rc = scan(tcur, &added)) return rc;
            int m = stamp++, s = stamp++;
            dt::split_kernel<<<grid, 256, 0, st>>>(w, tcur, m, s);
            tcur += 2 * added;
            grid = cap_grid(ctx, (tcur + 255) / 256, 16);
            dt::fix_kernel<<<grid, 256, 0, st>>>(w, tcur, m);
            ctx->launches += 2;
            for (;;) {
                CK(cudaMemsetAsync(w.vote, 0xff, (size_t)tcur * 8, st));
                CK(cudaMemsetAsync(w.cnt + dt::C_FLIPS, 0, sizeof(unsigned), st));
                const int m2 = stamp++, s2 = stamp++;
                dt::detect_kernel<<<grid, 256, 0, st>>>(w, tcur, s);
                dt::flip_kernel<<<grid, 256, 0, st>>>(w, tcur, s, m2, s2);
                dt::fix_kernel<<<grid, 256, 0, st>>>(w, tcur, m2);
                ctx->launches += 3;
                s = s2;
                if (int rc = counters()) return rc;
                if (!cnt[dt::C_FLIPS]) break;
            }
            if (int rc = relocate()) return rc;
            if (cnt[dt::C_ERR]) return RTX_E_UNSUPPORTED;  // a broken invariant, never expected
        }
        // the finite triangles in slot order
        const unsigned grid = cap_grid(ctx, (tcur + 255) / 256, 16);
        dt::finite_kernel<<<grid, 256, 0, st>>>(w, tcur);
        ctx->launches++;
        if (int rc = scan(tcur, &nfin)) return rc;
        dt::output_kernel<<<grid, 256, 0, st>>>(w, tcur, simplices, neighbors, (double*)transform);
        ctx->launches++;
        return (int)cudaGetLastError();
    });
    if (rc) return rc;
    CK(cudaStreamSynchronize(st));
    *T = nfin;
    return 0;
}

}  // extern "C"

// ---- exit-pupil points and grid ranges of the OPD (rtx_psf.cuh) ------------
extern "C" {

int rtx_opd_points(rtx_ctx* ctx, int dtype, int64_t N, const void* A, const void* P, int64_t ref,
                   double k, double* pts, double* vals, int64_t* M, double* h) {
    // the prefix sum counts in int32
    if (!ctx || !A || !P || !pts || !vals || !M || !h || N < 1 || N >= (1ll << 31) || ref < 0 ||
        ref >= N || k == 0.0 || !std::isfinite(k))
        return RTX_E_BADARG;
    int rc = fp64_only(dtype);
    if (rc) return rc;
    CK(cudaSetDevice(ctx->device));
    const int n = (int)N, nb = (n + dt::SCAN_THREADS - 1) / dt::SCAN_THREADS;
    // [max bits | block sums and the total | keep flags, ranked in place]
    const size_t bsum_off = 256, flag_off = bsum_off + ((size_t)(nb + 1) * 4 + 255) / 256 * 256;
    rc = reserve(ctx->ws[WS_OPD], flag_off + (size_t)n * 4);
    if (rc) return rc;
    char* base = (char*)ctx->ws[WS_OPD].p;
    auto* hbits = (unsigned long long*)base;
    int* bsum = (int*)(base + bsum_off);
    int* flag = (int*)(base + flag_off);
    const double *a = (const double*)A, *p = (const double*)P;
    cudaStream_t st = ctx->stream;
    const unsigned grid = cap_grid(ctx, (N + 255) / 256, 16);
    CK(cudaMemsetAsync(hbits, 0, 8, st));
    rc = timed(ctx, [&] {
        opd_flag_kernel<<<grid, 256, 0, st>>>(a, p, N, ref, k, flag);
        dt::scan_block_kernel<<<nb, dt::SCAN_THREADS, 0, st>>>(flag, n, bsum);
        dt::scan_top_kernel<<<1, dt::SCAN_THREADS, 0, st>>>(bsum, nb);
        // in place: each thread reads its own flag before the block scan and
        // writes its rank after it
        dt::scan_apply_kernel<<<nb, dt::SCAN_THREADS, 0, st>>>(flag, n, bsum, flag);
        opd_scatter_kernel<<<grid, 256, 0, st>>>(a, p, N, ref, k, flag, pts, vals, hbits);
        ctx->launches += 5;
        return (int)cudaGetLastError();
    });
    if (rc) return rc;
    int count = 0;
    unsigned long long hb = 0;
    CK(cudaMemcpyAsync(&count, bsum + nb, sizeof(int), cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(&hb, hbits, 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    *M = count;
    memcpy(h, &hb, 8);
    return 0;
}

int rtx_grid_range(rtx_ctx* ctx, int dtype, int64_t n, const void* o, int64_t* count, double* lo,
                   double* hi) {
    if (!ctx || n < 1 || !o || !count || !lo || !hi) return RTX_E_BADARG;
    int rc = fp64_only(dtype);
    if (rc) return rc;
    CK(cudaSetDevice(ctx->device));
    rc = reserve(ctx->ws[WS_RANGE], 3 * sizeof(unsigned long long));
    if (rc) return rc;
    auto* d_acc = (unsigned long long*)ctx->ws[WS_RANGE].p;
    cudaStream_t st = ctx->stream;
    const unsigned grid = cap_grid(ctx, (n + 255) / 256, 8);
    CK(cudaMemsetAsync(d_acc, 0, 3 * sizeof(unsigned long long), st));
    CK(cudaMemsetAsync(d_acc + 1, 0xff, sizeof(unsigned long long), st));  // min key: ~0
    rc = timed(ctx, [&] {
        grid_range_kernel<<<grid, 256, 0, st>>>((const double*)o, n, d_acc);
        ctx->launches++;
        return (int)cudaGetLastError();
    });
    if (rc) return rc;
    unsigned long long acc[3];
    CK(cudaMemcpyAsync(acc, d_acc, sizeof(acc), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    auto value = [](unsigned long long key) {  // order_key's inverse
        const unsigned long long b = (key >> 63) ? key & ~0x8000000000000000ull : ~key;
        double v;
        memcpy(&v, &b, 8);
        return v;
    };
    *count = (int64_t)acc[0];
    *lo = acc[0] ? value(acc[1]) : NAN;
    *hi = acc[0] ? value(acc[2]) : NAN;
    return 0;
}

}  // extern "C"

namespace {
// rtx_pupil_sum's and rtx_pupil_intensity's record check (include/rtx.h)
bool pupil_ok(const rtx_pupil* s) {
    if (!s || s->planes < 1 || s->planes > RTX_PUPIL_MAX_PLANES || s->reserved != 0) return false;
    if (s->nx < 1 || s->nx > RTX_PUPIL_MAX_PIXELS || s->ny < 1 || s->ny > RTX_PUPIL_MAX_PIXELS)
        return false;
    if (!std::isfinite(s->wavelength) || s->wavelength == 0.0 || !std::isfinite(s->radius) ||
        s->radius == 0.0)
        return false;
    bool finite = std::isfinite(s->a0) && std::isfinite(s->kappa) && std::isfinite(s->p0) &&
                  std::isfinite(s->dp) && std::isfinite(s->q0) && std::isfinite(s->dq);
    for (int k = 0; k < s->planes; ++k) finite = finite && std::isfinite(s->z[k]);
    return finite;
}

template <int WR, int WC>
int launch_pupil_sum(rtx_ctx* ctx, PupilDev& d) {
    using SM = PupilSmem<WR, WC>;
    d.tiles_x = (int)((d.nx + SM::TA - 1) / SM::TA);
    d.tiles_y = (int)((d.ny + SM::TB - 1) / SM::TB);
    const long long items = d.slots * d.groups * d.tiles_x * d.tiles_y;
    const size_t smem = (size_t)SM::doubles * sizeof(double);
    auto kern = pupil_sum_kernel<WR, WC>;
    CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<(unsigned)items, PUP_THREADS, smem, ctx->stream>>>(d);
    ctx->launches++;
    return (int)cudaGetLastError();
}
}  // namespace

extern "C" {

int rtx_pupil_sum(rtx_ctx* ctx, int64_t N, const double* A, const double* P, const double* w,
                  const rtx_pupil* spec, double* U, int64_t* count, double* sumw) {
    if (!ctx || !spec || !U || !count || !sumw || N < 0 || (N > 0 && (!A || !P)))
        return RTX_E_BADARG;
    if (!pupil_ok(spec)) return RTX_E_BADARG;
    *count = 0;
    *sumw = 0.0;
    if (N == 0) return 0;
    PupilDev d;
    memset(&d, 0, sizeof(d));
    d.K = spec->planes;
    d.groups = (d.K + PUP_GROUP - 1) / PUP_GROUP;
    d.KG = (d.K + d.groups - 1) / d.groups;
    d.nx = spec->nx;
    d.ny = spec->ny;
    d.N = N;
    long long L = std::max<long long>(RTX_PUPIL_SLOT, (N + RTX_PUPIL_MAX_SLOTS - 1) / RTX_PUPIL_MAX_SLOTS);
    d.L = (L + PUP_CH - 1) / PUP_CH * PUP_CH;
    d.slots = (N + d.L - 1) / d.L;
    d.a0 = spec->a0;
    d.lambda = spec->wavelength;
    d.kappa = spec->kappa;
    d.radius = spec->radius;
    d.p0 = spec->p0;
    d.dp = spec->dp;
    d.q0 = spec->q0;
    d.dq = spec->dq;
    for (int k = 0; k < d.K; ++k) d.z[k] = spec->z[k];
    d.A = A;
    d.P = P;
    d.w = w;
    CK(cudaSetDevice(ctx->device));
    const long long n = 2LL * d.K * d.nx * d.ny, row = n + 2;
    int rc = reserve(ctx->ws[WS_PUPIL], (size_t)(d.slots * row) * sizeof(double));
    if (rc) return rc;
    d.part = (double*)ctx->ws[WS_PUPIL].p;
    rc = timed(ctx, [&] {
        int rc;
        if (d.KG == 1)
            rc = launch_pupil_sum<2, 4>(ctx, d);
        else if (d.KG == 2)
            rc = launch_pupil_sum<2, 2>(ctx, d);
        else if (d.KG <= 4)
            rc = launch_pupil_sum<1, 2>(ctx, d);
        else
            rc = launch_pupil_sum<1, 1>(ctx, d);
        if (rc) return rc;
        pupil_fold_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(d.part, row, n,
                                                                             d.slots, U);
        ctx->launches++;
        return (int)cudaGetLastError();
    });
    if (rc) return rc;
    std::vector<double> h((size_t)(2 * d.slots));
    CK(cudaMemcpy2DAsync(h.data(), 2 * sizeof(double), d.part + n, row * sizeof(double),
                         2 * sizeof(double), (size_t)d.slots, cudaMemcpyDeviceToHost,
                         ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    double c = 0.0, sw = 0.0;
    for (long long q = 0; q < d.slots; ++q) {
        c += h[(size_t)(2 * q)];
        sw += h[(size_t)(2 * q + 1)];
    }
    *count = (int64_t)c;
    *sumw = sw;
    return 0;
}

int rtx_pupil_intensity(rtx_ctx* ctx, const rtx_pupil* spec, const double* U, double scale,
                        double* psf, double* stats) {
    if (!ctx || !U || !psf || !pupil_ok(spec) || !std::isfinite(scale)) return RTX_E_BADARG;
    const int K = spec->planes;
    const long long npix = spec->nx * spec->ny;
    const long long nb = (npix + PUP_RED - 1) / PUP_RED;
    CK(cudaSetDevice(ctx->device));
    Workspace& ws = ctx->ws[WS_PUPIL_RED];
    const size_t bytes = (size_t)(K * nb * 5) * sizeof(double);
    int rc = reserve(ws, bytes);
    if (rc) return rc;
    double* part = (double*)ws.p;
    rc = timed(ctx, [&] {
        pupil_intensity_kernel<<<dim3((unsigned)nb, (unsigned)K), 256, 0, ctx->stream>>>(
            U, scale, psf, spec->nx, spec->ny, spec->p0, spec->dp, spec->q0, spec->dq, part);
        ctx->launches++;
        return (int)cudaGetLastError();
    });
    if (rc) return rc;
    std::vector<double> h((size_t)(K * nb * 5));
    CK(cudaMemcpyAsync(h.data(), part, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    if (stats)
        for (int k = 0; k < K; ++k) {
            double sum = 0.0, mx = -1.0, at = -1.0, sp = 0.0, sq = 0.0;
            for (long long b = 0; b < nb; ++b) {
                const double* r = &h[(size_t)((k * nb + b) * 5)];
                sum += r[0];
                sp += r[3];
                sq += r[4];
                if (r[1] > mx) {
                    mx = r[1];
                    at = r[2];
                }
            }
            double* o = stats + 5 * k;
            o[0] = sum;
            o[1] = mx;
            o[2] = at;
            o[3] = sp;
            o[4] = sq;
        }
    return 0;
}

}  // extern "C"
