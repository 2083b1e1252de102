// rtx.cu -- C ABI of the ray-trace engine (include/rtx.h): context, memory,
// the table conversion and the kernel launches.  Build:
//   nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -shared \
//        -Xcompiler -fPIC -o librtx.so rtx.cu
#include "../../include/rtx.h"
#include "rtx_device.cuh"
#include "rtx_psf.cuh"
#include "rtx_delaunay.cuh"

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
    int tune = 1;             // TraceParams::tune bits (RTX_TUNE); 1 = L2 evict_first stores
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
    double* d_moments = nullptr;
    double* d_epi = nullptr;  // rtx_trace_reduce
    // cached plan of the ray generator (rtx_aim_plan / rtx_aim_rays)
    std::vector<unsigned char> aim_key;
    std::vector<long long> aim_offsets;  // per block; empty: nothing is rejected
    long long* d_aim_offsets = nullptr;
    size_t d_aim_cap = 0;
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
    // rtx_grid_linear: claim grid when the caller wants no winner output
    int* d_winner = nullptr;
    size_t winner_cap = 0;
    // rtx_psf: the cuFFT plan of the last (nx, ny) and its work area
    cufftHandle fft_plan = 0;
    bool fft_planned = false;
    long long fft_nx = 0, fft_ny = 0;
    void* fft_work = nullptr;
    size_t fft_work_bytes = 0;
    double* d_psf_red = nullptr;  // partial sums, the finite count and the stats
    // rtx_psf_profiles: per-block partial rows, their sum and the pixel flag
    double* d_prof = nullptr;
    size_t prof_cap = 0;
    // rtx_delaunay: slots, adjacency and point-location workspace
    void* d_dt = nullptr;
    size_t dt_cap = 0;
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

bool valid_keep_dtype(int keep, int dtype) {
    return (keep == RTX_KEEP_ALL || keep == RTX_KEEP_LAST) &&
           (dtype == RTX_F64 || dtype == RTX_F32);
}

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
    p.tune = ctx->tuning.tune;
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
        CK(cudaMalloc((void**)&ctx->d_moments, 8 * sizeof(double)));
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
    if (const char* e = getenv("RTX_TUNE")) tu.tune = atoi(e);
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
    if (ctx->d_moments) cudaFree(ctx->d_moments);
    if (ctx->d_epi) cudaFree(ctx->d_epi);
    if (ctx->d_aim_offsets) cudaFree(ctx->d_aim_offsets);
    if (ctx->d_winner) cudaFree(ctx->d_winner);
    release_fft_plan(ctx);
    if (ctx->d_psf_red) cudaFree(ctx->d_psf_red);
    if (ctx->d_prof) cudaFree(ctx->d_prof);
    if (ctx->d_dt) cudaFree(ctx->d_dt);
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
    int rc = check_table(surf, S);
    if (rc) return rc;
    if (N < 0 || ld < N || !y0 || !u0) return RTX_E_BADARG;
    if (!valid_keep_dtype(keep, dtype)) return RTX_E_BADARG;
    if (N == 0) return 0;
    CK(cudaSetDevice(ctx->device));
    CK(cudaEventRecord(ctx->k0, ctx->stream));
    if (dtype == RTX_F64) {
        Launch<double> L(surf, S, rot0, clip, keep, ld, flags);
        rc = trace_registered(ctx, L, surf, N, y0, u0, Y, U, I, T);
    } else {
        Launch<float> L(surf, S, rot0, clip, keep, ld, flags);
        rc = trace_registered(ctx, L, surf, N, y0, u0, Y, U, I, T);
    }
    if (rc) return rc;
    CK(cudaEventRecord(ctx->k1, ctx->stream));
    ctx->kernel_timed = true;
    return 0;
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
    if (!valid_keep_dtype(keep, dtype)) return RTX_E_BADARG;
    for (int b = 0; b < nb; ++b) {
        int rc = check_table(surf[b], S);
        if (rc) return rc;
        if (N[b] < 1 || ld < N[b] || !y0[b] || !u0[b]) return RTX_E_BADARG;
    }
    CK(cudaSetDevice(ctx->device));
    CK(cudaEventRecord(ctx->k0, ctx->stream));
    int rc = dtype == RTX_F64
                 ? trace_batch<double>(ctx, nb, surf, S, rot0, N, y0, u0, clip, keep, ld, Y, U, I,
                                       T, flags)
                 : trace_batch<float>(ctx, nb, surf, S, rot0, N, y0, u0, clip, keep, ld, Y, U, I, T,
                                      flags);
    if (rc) return rc;
    CK(cudaEventRecord(ctx->k1, ctx->stream));
    ctx->kernel_timed = true;
    return 0;
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
    if (!valid_keep_dtype(keep, dtype)) return RTX_E_BADARG;
    for (int b = 0; b < nb; ++b) {
        int rc = check_table(surf[b], S);
        if (rc) return rc;
        if (N[b] < 0 || (N[b] > 0 && (!y0[b] || !u0[b]))) return RTX_E_BADARG;
    }
    CK(cudaSetDevice(ctx->device));
    return dtype == RTX_F64 ? trace_batch_host<double>(ctx, nb, surf, S, rot0, N, y0, u0, clip,
                                                       keep, Y, U, I, T, flags)
                            : trace_batch_host<float>(ctx, nb, surf, S, rot0, N, y0, u0, clip,
                                                      keep, Y, U, I, T, flags);
}

int rtx_trace_host(rtx_ctx* ctx, const rtx_surface* surf, int S, const double* rot0, int dtype,
                   int64_t N, const void* y0, const void* u0, int clip, int keep, void* Y, void* U,
                   void* I, void* T, unsigned flags) {
    if (!ctx) return RTX_E_BADARG;
    int rc = check_table(surf, S);
    if (rc) return rc;
    if (N < 0 || !y0 || !u0) return RTX_E_BADARG;
    if (!valid_keep_dtype(keep, dtype)) return RTX_E_BADARG;
    if (N == 0) return 0;
    CK(cudaSetDevice(ctx->device));
    if (dtype == RTX_F64)
        return trace_host<double>(ctx, surf, S, rot0, N, y0, u0, clip, keep, Y, U, I, T, flags);
    return trace_host<float>(ctx, surf, S, rot0, N, y0, u0, clip, keep, Y, U, I, T, flags);
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
    int rc = check_table(surf, S);
    if (rc) return rc;
    if (N < 0 || !y0 || !u0 || npeers < 1 || npeers > 8 || !dst || dst_offset < 0)
        return RTX_E_BADARG;
    if (!valid_keep_dtype(RTX_KEEP_LAST, dtype)) return RTX_E_BADARG;
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
    CK(cudaEventRecord(ctx->k0, ctx->stream));
    const long long ld = ((N + 127) / 128) * 128;  // only the gather destinations are written
    if (dtype == RTX_F64) {
        Launch<double> L(surf, S, rot0, clip, RTX_KEEP_LAST, ld, flags);
        L.peers = &pd;
        rc = trace_registered(ctx, L, surf, N, y0, u0, nullptr, nullptr, nullptr, nullptr);
    } else {
        Launch<float> L(surf, S, rot0, clip, RTX_KEEP_LAST, ld, flags);
        L.peers = &pd;
        rc = trace_registered(ctx, L, surf, N, y0, u0, nullptr, nullptr, nullptr, nullptr);
    }
    if (rc) return rc;
    CK(cudaEventRecord(ctx->k1, ctx->stream));
    ctx->kernel_timed = true;
    return 0;
}

int rtx_selftest_math(rtx_ctx* ctx, int64_t n, const double* a, const double* b, double* out) {
    if (!ctx || n < 1 || !a || !b || !out) return RTX_E_BADARG;
    CK(cudaSetDevice(ctx->device));
    struct Bufs {  // freed on every return path
        double *a = nullptr, *b = nullptr, *o = nullptr;
        ~Bufs() {
            cudaFree(a);
            cudaFree(b);
            cudaFree(o);
        }
    } d;
    CK(cudaMalloc((void**)&d.a, n * sizeof(double)));
    CK(cudaMalloc((void**)&d.b, n * sizeof(double)));
    CK(cudaMalloc((void**)&d.o, 6 * n * sizeof(double)));
    CK(cudaMemcpyAsync(d.a, a, n * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(d.b, b, n * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    selftest_math_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(d.a, d.b, d.o, n);
    ctx->launches++;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(out, d.o, 6 * n * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return 0;
}

int rtx_selftest_math2(rtx_ctx* ctx, int64_t n, const double* a, const double* b,
                       const double* c, double* out) {
    if (!ctx || n < 1 || !a || !b || !c || !out) return RTX_E_BADARG;
    CK(cudaSetDevice(ctx->device));
    struct Bufs {  // freed on every return path
        double *a = nullptr, *b = nullptr, *c = nullptr, *o = nullptr;
        ~Bufs() {
            cudaFree(a);
            cudaFree(b);
            cudaFree(c);
            cudaFree(o);
        }
    } d;
    CK(cudaMalloc((void**)&d.a, n * sizeof(double)));
    CK(cudaMalloc((void**)&d.b, n * sizeof(double)));
    CK(cudaMalloc((void**)&d.c, n * sizeof(double)));
    CK(cudaMalloc((void**)&d.o, 7 * n * sizeof(double)));
    CK(cudaMemcpyAsync(d.a, a, n * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(d.b, b, n * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(d.c, c, n * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    selftest_math2_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(d.a, d.b, d.c,
                                                                               d.o, n);
    ctx->launches++;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(out, d.o, 7 * n * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return 0;
}

int rtx_moments(rtx_ctx* ctx, int dtype, int64_t N, const void* y, const void* w,
                const double* center, double* m) {
    if (!ctx || !y || !m || N < 0) return RTX_E_BADARG;
    CK(cudaSetDevice(ctx->device));
    const double cx = center ? center[0] : 0.0, cy = center ? center[1] : 0.0;
    CK(cudaMemsetAsync(ctx->d_moments, 0, 8 * sizeof(double), ctx->stream));
    if (N > 0) {
        long long blocks = (N + 255) / 256;
        long long cap = (long long)ctx->sm_count * 8;
        if (blocks > cap) blocks = cap;
        if (dtype == RTX_F64)
            moments_kernel<double><<<(unsigned)blocks, 256, 0, ctx->stream>>>(
                (const double*)y, (const double*)w, N, cx, cy, ctx->d_moments);
        else if (dtype == RTX_F32)
            moments_kernel<float><<<(unsigned)blocks, 256, 0, ctx->stream>>>(
                (const float*)y, (const float*)w, N, cx, cy, ctx->d_moments);
        else
            return RTX_E_BADARG;
        ctx->launches++;
        CK(cudaGetLastError());
    }
    CK(cudaMemcpyAsync(m, ctx->d_moments, 8 * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return 0;
}

}  // extern "C"

namespace {
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
    const bool exact = (flags & RTX_EXACT) != 0;
    if (exact && sizeof(T) == 4) return RTX_E_UNSUPPORTED;
    constexpr int RPT = 2, threads = 256;
    size_t smem = (((size_t)S * sizeof(DevSurf<T>) + 127) & ~size_t(127)) + 16;
    if ((int)smem > ctx->max_smem_optin) return RTX_E_UNSUPPORTED;
    auto go = [&](auto kern) -> int {
        if (smem > 48 * 1024)
            CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        int occ = 0;
        CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, threads, smem));
        if (occ < 1) occ = 1;
        const long long tiles = (N + threads * RPT - 1) / (threads * RPT);
        long long grid = (long long)ctx->sm_count * occ;
        if (grid > tiles) grid = tiles;
        if (grid < 1) grid = 1;
        kern<<<(unsigned)grid, threads, smem, ctx->stream>>>(p);
        ctx->launches++;
        return (int)cudaGetLastError();
    };
    if constexpr (sizeof(T) == 8) {
        if (exact) return go(epi_kernel<T, true, RPT, MODE>);
    }
    return go(epi_kernel<T, false, RPT, MODE>);
}
}  // namespace

extern "C" {

int rtx_trace_reduce(rtx_ctx* ctx, const rtx_surface* surf, int S, const double* rot0, int dtype,
                     int64_t N, const void* y0, const void* u0, int clip, const void* w,
                     const double* center, double* m, unsigned flags) {
    if (!ctx || !m) return RTX_E_BADARG;
    int rc = check_table(surf, S);
    if (rc) return rc;
    if (N < 0 || !y0 || !u0) return RTX_E_BADARG;
    if (dtype != RTX_F64 && dtype != RTX_F32) return RTX_E_BADARG;
    CK(cudaSetDevice(ctx->device));
    if (!ctx->d_epi) CK(cudaMalloc((void**)&ctx->d_epi, RTX_NMOMENTS * sizeof(double)));
    CK(cudaMemsetAsync(ctx->d_epi, 0, RTX_NMOMENTS * sizeof(double), ctx->stream));
    if (N > 0) {
        CK(cudaEventRecord(ctx->k0, ctx->stream));
        if (dtype == RTX_F64) {
            EpiParams<double> p;
            memset(&p, 0, sizeof(p));
            p.w = (const double*)w;
            for (int k = 0; k < 2; ++k) {
                p.cy[k] = center ? center[k] : 0.0;
                p.cu[k] = center ? center[2 + k] : 0.0;
            }
            p.out = ctx->d_epi;
            rc = launch_epi<double, EPI_REDUCE>(ctx, surf, S, rot0, N, y0, u0, clip, flags, p);
        } else {
            EpiParams<float> p;
            memset(&p, 0, sizeof(p));
            p.w = (const float*)w;
            for (int k = 0; k < 2; ++k) {
                p.cy[k] = center ? center[k] : 0.0;
                p.cu[k] = center ? center[2 + k] : 0.0;
            }
            p.out = ctx->d_epi;
            rc = launch_epi<float, EPI_REDUCE>(ctx, surf, S, rot0, N, y0, u0, clip, flags, p);
        }
        if (rc) return rc;
        CK(cudaEventRecord(ctx->k1, ctx->stream));
        ctx->kernel_timed = true;
    }
    CK(cudaMemcpyAsync(m, ctx->d_epi, RTX_NMOMENTS * sizeof(double), cudaMemcpyDeviceToHost,
                       ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return 0;
}

int rtx_trace_opd(rtx_ctx* ctx, const rtx_surface* surf, int S, const double* rot0, int dtype,
                  int64_t N, const void* y0, const void* u0, int clip, const rtx_opd* opd, void* A,
                  void* P, unsigned flags) {
    if (!ctx || !opd || !A || !P) return RTX_E_BADARG;
    int rc = check_table(surf, S);
    if (rc) return rc;
    if (N < 0 || !y0 || !u0 || opd->radius == 0.0) return RTX_E_BADARG;
    if (dtype != RTX_F64 && dtype != RTX_F32) return RTX_E_BADARG;
    if (N == 0) return 0;
    CK(cudaSetDevice(ctx->device));
    auto fill = [&](auto& p) {
        memset(&p, 0, sizeof(p));
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
    };
    CK(cudaEventRecord(ctx->k0, ctx->stream));
    if (dtype == RTX_F64) {
        EpiParams<double> p;
        fill(p);
        p.A = (double*)A;
        p.P = (double*)P;
        rc = launch_epi<double, EPI_OPD>(ctx, surf, S, rot0, N, y0, u0, clip, flags, p);
    } else {
        EpiParams<float> p;
        fill(p);
        p.A = (float*)A;
        p.P = (float*)P;
        rc = launch_epi<float, EPI_OPD>(ctx, surf, S, rot0, N, y0, u0, clip, flags, p);
    }
    if (rc) return rc;
    CK(cudaEventRecord(ctx->k1, ctx->stream));
    ctx->kernel_timed = true;
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
        if ((size_t)(nb + 1) * sizeof(long long) > ctx->d_aim_cap) {
            if (ctx->d_aim_offsets) CK(cudaFree(ctx->d_aim_offsets));
            ctx->d_aim_offsets = nullptr;
            ctx->d_aim_cap = 0;
            CK(cudaMalloc((void**)&ctx->d_aim_offsets, (size_t)(nb + 1) * sizeof(long long)));
            ctx->d_aim_cap = (size_t)(nb + 1) * sizeof(long long);
        }
        int* d_counts = reinterpret_cast<int*>(ctx->d_aim_offsets);  // reused before the offsets
        long long grid = nb < (long long)ctx->sm_count * 8 ? nb : (long long)ctx->sm_count * 8;
        aim_count_kernel<<<(unsigned)grid, 256, 0, ctx->stream>>>(d, (const double*)yp, d_counts, nb);
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
        CK(cudaMemcpyAsync(ctx->d_aim_offsets, ctx->aim_offsets.data(),
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
    if (dtype != RTX_F64 && dtype != RTX_F32) return RTX_E_BADARG;
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
        d_off = ctx->d_aim_offsets;
    }
    long long grid = b1 - b0;
    const long long cap = (long long)ctx->sm_count * 8;
    if (grid > cap) grid = cap;
    if (grid < 1) grid = 1;
    if (dtype == RTX_F64)
        aim_rays_kernel<double><<<(unsigned)grid, 256, 0, ctx->stream>>>(
            d, (const double*)yp, d_off, b0, b1, first, count, (double*)y0, (double*)u0,
            (double*)yp_out);
    else
        aim_rays_kernel<float><<<(unsigned)grid, 256, 0, ctx->stream>>>(
            d, (const double*)yp, d_off, b0, b1, first, count, (float*)y0, (float*)u0,
            (double*)yp_out);
    ctx->launches++;
    return (int)cudaGetLastError();
}

int rtx_focus_moments(rtx_ctx* ctx, int dtype, int64_t N, const void* y, const void* inc,
                      const void* w, const double* center, double* m) {
    if (!ctx || !y || !inc || !m || N < 0) return RTX_E_BADARG;
    CK(cudaSetDevice(ctx->device));
    double c[4] = {0, 0, 0, 0};
    if (center)
        for (int k = 0; k < 4; ++k) c[k] = center[k];
    CK(cudaMemsetAsync(ctx->d_moments, 0, 8 * sizeof(double), ctx->stream));
    if (N > 0) {
        long long blocks = (N + 255) / 256;
        long long cap = (long long)ctx->sm_count * 8;
        if (blocks > cap) blocks = cap;
        if (dtype == RTX_F64)
            focus_moments_kernel<double><<<(unsigned)blocks, 256, 0, ctx->stream>>>(
                (const double*)y, (const double*)inc, (const double*)w, N, c[0], c[1], c[2], c[3],
                ctx->d_moments);
        else if (dtype == RTX_F32)
            focus_moments_kernel<float><<<(unsigned)blocks, 256, 0, ctx->stream>>>(
                (const float*)y, (const float*)inc, (const float*)w, N, c[0], c[1], c[2], c[3],
                ctx->d_moments);
        else
            return RTX_E_BADARG;
        ctx->launches++;
        CK(cudaGetLastError());
    }
    CK(cudaMemcpyAsync(m, ctx->d_moments, 8 * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return 0;
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
    if (dtype == RTX_F32) return RTX_E_UNSUPPORTED;
    if (dtype != RTX_F64) return RTX_E_BADARG;
    CK(cudaSetDevice(ctx->device));
    const long long nn = (long long)n * n;
    int* claim = winner;
    if (!claim) {
        if ((size_t)nn * sizeof(int) > ctx->winner_cap) {
            if (ctx->d_winner) CK(cudaFree(ctx->d_winner));
            ctx->d_winner = nullptr;
            ctx->winner_cap = 0;
            CK(cudaMalloc((void**)&ctx->d_winner, (size_t)nn * sizeof(int)));
            ctx->winner_cap = (size_t)nn * sizeof(int);
        }
        claim = ctx->d_winner;
    }
    long long grid = (nn + 255) / 256;
    const long long cap = (long long)ctx->sm_count * 16;
    if (grid > cap) grid = cap;
    CK(cudaEventRecord(ctx->k0, ctx->stream));
    fill_i32_kernel<<<(unsigned)grid, 256, 0, ctx->stream>>>(claim, nn, INT_MAX);
    ctx->launches++;
    CK(cudaGetLastError());
    if (T > 0) {
        grid_claim_kernel<<<(unsigned)((T + 255) / 256), 256, 0, ctx->stream>>>(
            (const double*)pts, M, simplices, (const double*)transform, T, (const double*)gh, n,
            claim);
        ctx->launches++;
        CK(cudaGetLastError());
    }
    grid_eval_kernel<<<(unsigned)grid, 256, 0, ctx->stream>>>(
        (const double*)vals, simplices, (const double*)transform, (const double*)gh, n, claim,
        (double*)out);
    ctx->launches++;
    CK(cudaGetLastError());
    CK(cudaEventRecord(ctx->k1, ctx->stream));
    ctx->kernel_timed = true;
    return 0;
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
    if (dtype == RTX_F32) return RTX_E_UNSUPPORTED;
    if (dtype != RTX_F64) return RTX_E_BADARG;
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
    if (!ctx->d_psf_red) CK(cudaMalloc((void**)&ctx->d_psf_red, red_doubles * sizeof(double)));
    double* part = ctx->d_psf_red;
    auto* count = reinterpret_cast<unsigned long long*>(part + 4 * PSF_RED_BLOCKS);
    double* d_stats = part + 4 * PSF_RED_BLOCKS + 1;
    struct Grid {  // the complex grid is freed on every return path
        double2* z = nullptr;
        ~Grid() { if (z) cudaFree(z); }
    } g;
    if (cudaMalloc((void**)&g.z, zbytes) != cudaSuccess) {
        cudaGetLastError();
        g.z = nullptr;
        return RTX_E_NOMEM;
    }
    const long long nn = (long long)n * n;
    auto blocks = [&](long long items, long long per_sm) {
        long long b = (items + 255) / 256, cap = (long long)ctx->sm_count * per_sm;
        return (unsigned)(b < 1 ? 1 : (b > cap ? cap : b));
    };
    CK(cudaMemsetAsync(count, 0, sizeof(unsigned long long), ctx->stream));
    CK(cudaEventRecord(ctx->k0, ctx->stream));
    count_finite_kernel<<<blocks(nn, 8), 256, 0, ctx->stream>>>((const double*)o, nn, count);
    pupil_kernel<<<blocks(tot, 16), 256, 0, ctx->stream>>>((const double*)o, n, nx, ny, count, g.z);
    ctx->launches += 2;
    CK(cudaGetLastError());
    if (fft.exec_z2z(ctx->fft_plan, (cufftDoubleComplex*)g.z, (cufftDoubleComplex*)g.z,
                     CUFFT_FORWARD) != CUFFT_SUCCESS)
        return RTX_E_UNSUPPORTED;
    intensity_kernel<<<PSF_RED_BLOCKS, 256, 0, ctx->stream>>>(g.z, nx, ny, (double*)psf, part);
    psf_stats_kernel<<<1, 1, 0, ctx->stream>>>(part, PSF_RED_BLOCKS, count, d_stats);
    ctx->launches += 2;
    CK(cudaGetLastError());
    CK(cudaEventRecord(ctx->k1, ctx->stream));
    ctx->kernel_timed = true;
    if (stats)
        CK(cudaMemcpyAsync(stats, d_stats, 5 * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return 0;
}

int rtx_psf_profiles(rtx_ctx* ctx, int dtype, int64_t nx, int64_t ny, const void* psf, double c0,
                     double c1, int64_t nbins, double* ee, double* lsf0, double* lsf1) {
    if (!ctx || !psf || nx < 1 || ny < 1 || !std::isfinite(c0) || !std::isfinite(c1))
        return RTX_E_BADARG;
    if (dtype == RTX_F32) return RTX_E_UNSUPPORTED;
    if (dtype != RTX_F64) return RTX_E_BADARG;
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
    if (need > ctx->prof_cap) {
        size_t free_b = 0, total_b = 0;
        CK(cudaMemGetInfo(&free_b, &total_b));
        if (need > free_b + ctx->prof_cap) return RTX_E_NOMEM;  // nothing allocated
        if (ctx->d_prof) CK(cudaFree(ctx->d_prof));
        ctx->d_prof = nullptr;
        ctx->prof_cap = 0;
        if (cudaMalloc((void**)&ctx->d_prof, need) != cudaSuccess) {
            cudaGetLastError();
            ctx->d_prof = nullptr;
            return RTX_E_NOMEM;
        }
        ctx->prof_cap = need;
    }
    double* part = ctx->d_prof;
    double* out = part + (long long)PROF_BLOCKS * stride;
    int* flag = reinterpret_cast<int*>(out + stride);
    long long grid = (stride + 255) / 256;
    const long long cap = (long long)ctx->sm_count * 8;
    if (grid > cap) grid = cap;
    CK(cudaMemsetAsync(flag, 0, sizeof(int), ctx->stream));
    CK(cudaEventRecord(ctx->k0, ctx->stream));
    profile_tiles_kernel<<<PROF_BLOCKS, PROF_WARPS * 32, 0, ctx->stream>>>(
        (const double*)psf, nx, ny, c0, c1, nbins, part, stride, flag);
    profile_combine_kernel<<<(unsigned)grid, 256, 0, ctx->stream>>>(part, PROF_BLOCKS, stride, out);
    ctx->launches += 2;
    CK(cudaGetLastError());
    CK(cudaEventRecord(ctx->k1, ctx->stream));
    ctx->kernel_timed = true;
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
    CK(cudaSetDevice(ctx->device));
    struct Bufs {  // freed on every return path
        double* q = nullptr;
        int* o = nullptr;
        ~Bufs() {
            cudaFree(q);
            cudaFree(o);
        }
    } d;
    CK(cudaMalloc((void**)&d.q, 8 * n * sizeof(double)));
    CK(cudaMalloc((void**)&d.o, 2 * n * sizeof(int)));
    CK(cudaMemcpyAsync(d.q, pts, 8 * n * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    dt::selftest_predicates_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(d.q, n, d.o);
    ctx->launches++;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(out, d.o, 2 * n * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return 0;
}

int rtx_delaunay(rtx_ctx* ctx, int dtype, int64_t M, const void* pts, int64_t* T, int32_t* simplices,
                 int32_t* neighbors, void* transform) {
    if (!ctx || !pts || !T || !simplices) return RTX_E_BADARG;
    if (dtype == RTX_F32) return RTX_E_UNSUPPORTED;
    if (dtype != RTX_F64 || M < 3 || M > DT_MAX_POINTS) return RTX_E_BADARG;
    CK(cudaSetDevice(ctx->device));
    ctx->kernel_timed = false;  // until the call completes
    const size_t need = dt_carve(nullptr, M, nullptr, nullptr);
    if (need > ctx->dt_cap) {
        size_t free_b = 0, total_b = 0;
        CK(cudaMemGetInfo(&free_b, &total_b));
        if (need > free_b + ctx->dt_cap) return RTX_E_NOMEM;  // nothing allocated
        if (ctx->d_dt) CK(cudaFree(ctx->d_dt));
        ctx->d_dt = nullptr;
        ctx->dt_cap = 0;
        if (cudaMalloc(&ctx->d_dt, need) != cudaSuccess) {
            cudaGetLastError();
            ctx->d_dt = nullptr;
            return RTX_E_NOMEM;
        }
        ctx->dt_cap = need;
    }
    dt::Work w;
    dt_carve(ctx->d_dt, M, pts, &w);
    cudaStream_t st = ctx->stream;
    auto grid = [&](long long items) {
        long long b = (items + 255) / 256, cap = (long long)ctx->sm_count * 16;
        return (unsigned)(b < 1 ? 1 : (b > cap ? cap : b));
    };
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
        dt::relocate_kernel<<<grid(M), 256, 0, st>>>(w, 2 * M + 16);
        ctx->launches++;
        return counters();
    };
    CK(cudaEventRecord(ctx->k0, st));
    // validation and the seed triangle
    CK(cudaMemsetAsync(w.cnt, 0, dt::C_N * sizeof(unsigned), st));
    CK(cudaMemsetAsync(w.seed_key, 0xff, 8, st));
    dt::lex_kernel<<<dt::LEX_BLOCKS, dt::LEX_THREADS, 0, st>>>(w);
    dt::lex_final_kernel<<<1, 1, 0, st>>>(w);
    CK(cudaGetLastError());
    if (int rc = counters()) return rc;
    if (cnt[dt::C_ERR]) return RTX_E_BADARG;  // non-finite or outside the predicates' domain
    unsigned long long seed = 0;
    dt::seed_kernel<<<grid(M), 256, 0, st>>>(w);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(&seed, w.seed_key, 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    ctx->launches += 3;
    if (seed == dt::NONE) return RTX_E_BADARG;  // all points collinear
    fill_i32_kernel<<<grid(M), 256, 0, st>>>(w.loc, M, 0);
    dt::init_kernel<<<1, 1, 0, st>>>(w);
    ctx->launches += 2;
    int tcur = 4, stamp = 1;
    if (int rc = relocate()) return rc;
    while (cnt[dt::C_LEFT]) {
        CK(cudaMemsetAsync(w.pick, 0xff, (size_t)tcur * 8, st));
        CK(cudaMemsetAsync(w.vote, 0xff, (size_t)tcur * 8, st));
        dt::pick_kernel<<<grid(M), 256, 0, st>>>(w);
        dt::claim_kernel<<<grid(tcur), 256, 0, st>>>(w, tcur);
        dt::decide_kernel<<<grid(tcur), 256, 0, st>>>(w, tcur);
        ctx->launches += 3;
        int added = 0;
        if (int rc = scan(tcur, &added)) return rc;
        int m = stamp++, s = stamp++;
        dt::split_kernel<<<grid(tcur), 256, 0, st>>>(w, tcur, m, s);
        tcur += 2 * added;
        dt::fix_kernel<<<grid(tcur), 256, 0, st>>>(w, tcur, m);
        ctx->launches += 2;
        for (;;) {
            CK(cudaMemsetAsync(w.vote, 0xff, (size_t)tcur * 8, st));
            CK(cudaMemsetAsync(w.cnt + dt::C_FLIPS, 0, sizeof(unsigned), st));
            const int m2 = stamp++, s2 = stamp++;
            dt::detect_kernel<<<grid(tcur), 256, 0, st>>>(w, tcur, s);
            dt::flip_kernel<<<grid(tcur), 256, 0, st>>>(w, tcur, s, m2, s2);
            dt::fix_kernel<<<grid(tcur), 256, 0, st>>>(w, tcur, m2);
            ctx->launches += 3;
            s = s2;
            if (int rc = counters()) return rc;
            if (!cnt[dt::C_FLIPS]) break;
        }
        if (int rc = relocate()) return rc;
        if (cnt[dt::C_ERR]) return RTX_E_UNSUPPORTED;  // a broken invariant, never expected
    }
    // the finite triangles in slot order
    dt::finite_kernel<<<grid(tcur), 256, 0, st>>>(w, tcur);
    ctx->launches++;
    int nfin = 0;
    if (int rc = scan(tcur, &nfin)) return rc;
    dt::output_kernel<<<grid(tcur), 256, 0, st>>>(w, tcur, simplices, neighbors, (double*)transform);
    ctx->launches++;
    CK(cudaGetLastError());
    CK(cudaEventRecord(ctx->k1, st));
    ctx->kernel_timed = true;
    CK(cudaStreamSynchronize(st));
    *T = nfin;
    return 0;
}

}  // extern "C"
