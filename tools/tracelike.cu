// tracelike.cu -- synthetic kernel with the trace kernel's memory pattern and
// a tunable amount of dependent FP64 work, to separate memory-pattern effects
// from compute effects.  Per warp tile (32*RPT rays): for s in 0..S-1:
// D dependent DFMAs per ray, stage 10 values/ray, NARR bulk stores to row s.
// `kc`: the trace kernel's per-CTA stores, optionally in thread-block clusters
// whose CTAs store adjacent tiles in lockstep (cluster barrier per surface).
// `kf` (`tracelike.bin study [rounds]`): the clustered kernel's stores with
// one switch per store-pattern lever (DESIGN.md 3.7).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tracelike.bin tracelike.cu
#include <cuda_runtime.h>
#include <algorithm>
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <vector>

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

struct P {
    double *Y, *U, *I, *T;
    const double* in;
    long long N, ld;
    int S, D, mode;  // mode bit0: __syncthreads per surface (CTA lockstep); bit1: tile-major output layout
};

template <int RPT>
__global__ void __launch_bounds__(1024) k(P p) {
    extern __shared__ __align__(128) unsigned char sm[];
    const int lane = threadIdx.x & 31;
    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
    const int W = blockDim.x >> 5;
    constexpr int G = 32 * RPT;
    double* stage = reinterpret_cast<double*>(sm) + (size_t)warp * 2 * 10 * G;
    const long long stride = (long long)gridDim.x * W * G;
    const bool lock = p.mode & 1, tilemajor = p.mode & 2;
    int buf = 0;
    // all warps of a CTA run the same number of iterations when lockstep is on
    const long long nt = (p.N + stride - 1) / stride;
    for (long long it = 0; it < nt; ++it) {
        long long base = ((long long)blockIdx.x * W + warp) * G + it * stride;
        const bool live = base < p.N;
        if (!live) base = 0;
        double v[RPT][6];
#pragma unroll
        for (int r = 0; r < RPT; ++r)
#pragma unroll
            for (int c = 0; c < 6; ++c) v[r][c] = __ldg(p.in + (base + r * 32 + lane) * 6 + c);
#pragma unroll 1
        for (int s = 0; s < p.S; ++s) {
#pragma unroll
            for (int r = 0; r < RPT; ++r) {
                double a = v[r][0];
#pragma unroll 1
                for (int d = 0; d < p.D; ++d) a = fma(a, 1.0000001, v[r][1]);
                v[r][0] = a * 1e-9 + v[r][2];
            }
            double* sb = stage + buf * 10 * G;
            if (lock) __syncthreads();
            if (lane == 0) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
            __syncwarp();
#pragma unroll
            for (int r = 0; r < RPT; ++r) {
                int o = (r * 32 + lane) * 3;
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    sb[o + c] = v[r][c];
                    sb[3 * G + o + c] = v[r][3 + c];
                    sb[6 * G + o + c] = v[r][c] + 1.0;
                }
                sb[9 * G + r * 32 + lane] = v[r][0];
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncwarp();
            if (lane == 0 && live) {
                long long o = tilemajor ? (base * p.S + (long long)s * G) : ((long long)s * p.ld + base);
                asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(p.Y + o * 3), "r"(smem_u32(sb)), "r"(24 * G) : "memory");
                asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(p.U + o * 3), "r"(smem_u32(sb + 3 * G)), "r"(24 * G) : "memory");
                asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(p.I + o * 3), "r"(smem_u32(sb + 6 * G)), "r"(24 * G) : "memory");
                asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(p.T + o), "r"(smem_u32(sb + 9 * G)), "r"(8 * G) : "memory");
                asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            }
            buf ^= 1;
        }
    }
    if (lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

// The trace kernel's per-CTA store path (one staging buffer, thread 0 issues
// one bulk store per array and surface, a __syncthreads on either side of the
// staging), launched in clusters of CS CTAs: CTA r of cluster c owns CTA tile
// (c + k*nclusters)*CS + r, and the cluster barrier keeps the CTAs of a
// cluster within one surface of each other, so that their runs of a row are
// adjacent and leave together (CS x 24 KB per array in FP64).  CS = 1 is the
// trace kernel's current pattern.
template <int RPT>
__global__ void __launch_bounds__(512, 1) kc(P p) {
    extern __shared__ __align__(128) unsigned char sm[];
    const int lane = threadIdx.x & 31;
    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
    constexpr int G = 32 * RPT;
    const int CT = (blockDim.x >> 5) * G;
    double* sb = reinterpret_cast<double*>(sm);
    unsigned cs, rank, cid, ncl;
    asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(cs));
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(rank));
    asm volatile("mov.u32 %0, %%clusterid.x;" : "=r"(cid));
    asm volatile("mov.u32 %0, %%nclusterid.x;" : "=r"(ncl));
    const long long tiles = (p.N + CT - 1) / CT;
    const long long groups = (tiles + cs - 1) / cs;
    // same trip count for every CTA of a cluster: equal numbers of barriers
    const long long nt = cid < groups ? (groups - cid + ncl - 1) / ncl : 0;
    bool pending = false;
    for (long long it = 0; it < nt; ++it) {
        const long long cta_base = ((cid + it * ncl) * cs + rank) * CT;
        long long base = cta_base + warp * G;
        if (base >= p.N) base = 0;
        double v[RPT][6];
#pragma unroll
        for (int r = 0; r < RPT; ++r)
#pragma unroll
            for (int c = 0; c < 6; ++c) v[r][c] = __ldg(p.in + (base + r * 32 + lane) * 6 + c);
#pragma unroll 1
        for (int s = 0; s < p.S; ++s) {
#pragma unroll
            for (int r = 0; r < RPT; ++r) {
                double a = v[r][0];
#pragma unroll 1
                for (int d = 0; d < p.D; ++d) a = fma(a, 1.0000001, v[r][1]);
                v[r][0] = a * 1e-9 + v[r][2];
            }
            if (pending) asm volatile("barrier.cluster.wait.aligned;" ::: "memory");
            if (threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
            __syncthreads();
#pragma unroll
            for (int r = 0; r < RPT; ++r) {
                const int q = warp * G + r * 32 + lane;
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    sb[q * 3 + c] = v[r][c];
                    sb[3 * CT + q * 3 + c] = v[r][3 + c];
                    sb[6 * CT + q * 3 + c] = v[r][c] + 1.0;
                }
                sb[9 * CT + q] = v[r][0];
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncthreads();
            if (threadIdx.x == 0 && cta_base < p.N) {
                long long n = p.N - cta_base;
                if (n > CT) n = CT;
                n = (n + G - 1) / G * G;
                const long long o = (long long)s * p.ld + cta_base;
                asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(p.Y + o * 3), "r"(smem_u32(sb)), "r"((unsigned)(24 * n)) : "memory");
                asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(p.U + o * 3), "r"(smem_u32(sb + 3 * CT)), "r"((unsigned)(24 * n)) : "memory");
                asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(p.I + o * 3), "r"(smem_u32(sb + 6 * CT)), "r"((unsigned)(24 * n)) : "memory");
                asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(p.T + o), "r"(smem_u32(sb + 9 * CT)), "r"((unsigned)(8 * n)) : "memory");
                asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            }
            asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory");
            pending = true;
        }
    }
    if (pending) asm volatile("barrier.cluster.wait.aligned;" ::: "memory");
    if (threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

// `kf`: the clustered trace kernel's store path as it ships (16-CTA clusters,
// L2 evict_first stores, separate y0 / u0 launch arrays, a path-sum
// accumulator per ray) with each store-pattern lever on its own switch:
//   KF_PF    per-ray prefetch.global.L2 of the CTA's next tile (the kernel's
//            ray loads; off: __ldg only)
//   KF_TMAIN one cp.async.bulk of the CTA's next 24 KB y0 + 24 KB u0 into a
//            shared-memory slot under an mbarrier, instead of __ldg + prefetch
//   PAIR     (template) every CTA marches two adjacent 1024-ray tiles per
//            stored surface; tile A's state in registers, tile B's y, u and
//            accumulator (56 KB) in shared memory, both staged in turn through
//            the one 80 KB buffer: a 16-CTA cluster writes 768 KB per array
//            and row between two cluster barriers instead of 384 KB
// The number of resident clusters is the launch's grid (capped by the host).
enum { KF_PF = 1, KF_TMAIN = 2 };

struct PF {
    double *Y, *U, *I, *T, *tsum;
    const double *y0, *u0;
    long long N, ld;
    int S, D, flags;
};

__device__ __forceinline__ void kf_march(double (&v)[2][7], int D) {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        double a = v[r][0];
#pragma unroll 1
        for (int d = 0; d < D; ++d) a = fma(a, 1.0000001, v[r][1]);
        v[r][0] = a * 1e-9 + v[r][2];
        v[r][6] += v[r][0];
    }
}

// stage one tile's 10 values per ray and issue its four bulk stores (the
// trace kernel's STORE_CTA sequence with NBUF = 1)
__device__ __forceinline__ void kf_store(const PF& p, double* sb, const double (&v)[2][7],
                                         long long tbase, int s, uint64_t pol) {
    constexpr int G = 64, CT = 1024;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
    __syncthreads();
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int q = warp * G + r * 32 + lane;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            sb[q * 3 + c] = v[r][c];
            sb[3 * CT + q * 3 + c] = v[r][3 + c];
            sb[6 * CT + q * 3 + c] = v[r][c] + 1.0;
        }
        sb[9 * CT + q] = v[r][0];
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    if (threadIdx.x == 0 && tbase < p.N) {
        long long n = (p.N - tbase + G - 1) / G * G;
        if (n > CT) n = CT;
        const long long o = (long long)s * p.ld + tbase;
        const unsigned b3 = (unsigned)(24 * n);
        asm volatile("cp.async.bulk.global.shared::cta.bulk_group.L2::cache_hint [%0], [%1], %2, %3;" ::"l"(p.Y + o * 3), "r"(smem_u32(sb)), "r"(b3), "l"(pol) : "memory");
        asm volatile("cp.async.bulk.global.shared::cta.bulk_group.L2::cache_hint [%0], [%1], %2, %3;" ::"l"(p.U + o * 3), "r"(smem_u32(sb + 3 * CT)), "r"(b3), "l"(pol) : "memory");
        asm volatile("cp.async.bulk.global.shared::cta.bulk_group.L2::cache_hint [%0], [%1], %2, %3;" ::"l"(p.I + o * 3), "r"(smem_u32(sb + 6 * CT)), "r"(b3), "l"(pol) : "memory");
        asm volatile("cp.async.bulk.global.shared::cta.bulk_group.L2::cache_hint [%0], [%1], %2, %3;" ::"l"(p.T + o), "r"(smem_u32(sb + 9 * CT)), "r"((unsigned)(8 * n)), "l"(pol) : "memory");
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    }
}

template <bool PAIR>
__global__ void __launch_bounds__(512, 1) kf(PF p) {
    extern __shared__ __align__(128) unsigned char sm[];
    constexpr int G = 64, CT = 1024, NT = PAIR ? 2 : 1;
    const int lane = threadIdx.x & 31;
    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
    double* sb = reinterpret_cast<double*>(sm);   // 80 KB staging
    double* xb = sb + 10 * CT;                    // PAIR: tile B state [7][CT]; TMAIN: [y0 | u0]
    uint64_t* bar = reinterpret_cast<uint64_t*>(xb + (PAIR ? 7 : 6) * CT);
    unsigned cs, rank, cid, ncl;
    asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(cs));
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(rank));
    asm volatile("mov.u32 %0, %%clusterid.x;" : "=r"(cid));
    asm volatile("mov.u32 %0, %%nclusterid.x;" : "=r"(ncl));
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    const bool pf = p.flags & KF_PF, tmain = !PAIR && (p.flags & KF_TMAIN);
    const long long tiles = (p.N + CT - 1) / CT;
    const long long units = (tiles + NT - 1) / NT;  // a CTA's tile (pair)
    const long long groups = (units + cs - 1) / cs;
    const long long nt = cid < groups ? (groups - cid + ncl - 1) / ncl : 0;
    const long long ustride = (long long)ncl * cs * NT * CT;  // rays to the CTA's next unit
    auto ubase = [&](long long it) { return ((cid + it * ncl) * cs + rank) * NT * CT; };
    // TMAIN: one bulk load of a whole tile's y0 and u0 (the last tile takes a
    // shorter copy, N is even so 24 * n is a multiple of 16; a tile wholly past
    // the end, which the last group of a cluster can have, loads nothing)
    auto load_in = [&](long long b0) {
        long long n = p.N - b0;
        if (n > CT) n = CT;
        if (n <= 0) {
            asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
            return;
        }
        const unsigned bytes = (unsigned)(24 * n);
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(2 * bytes) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(xb)), "l"(p.y0 + b0 * 3), "r"(bytes), "r"(smem_u32(bar)) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(xb + 3 * CT)), "l"(p.u0 + b0 * 3), "r"(bytes), "r"(smem_u32(bar)) : "memory");
    };
    uint32_t phase = 0;
    if (tmain) {
        if (threadIdx.x == 0) {
            asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(bar)));
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
            if (nt > 0) load_in(ubase(0));
        }
        __syncthreads();
    }
    // (the kernel's __ldg path, with its clamp and optional prefetch)
    auto ldg_tile = [&](double (&v)[2][7], long long tb) {
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            long long ray = tb + warp * G + r * 32 + lane;
            const long long idx = ray < p.N ? ray : p.N - 1;
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                v[r][c] = __ldg(p.y0 + idx * 3 + c);
                v[r][3 + c] = __ldg(p.u0 + idx * 3 + c);
            }
            v[r][6] = 0.0;
            const long long nxt = ray + ustride;
            if (pf && nxt < p.N) {
                asm volatile("prefetch.global.L2 [%0];" ::"l"(p.y0 + nxt * 3));
                asm volatile("prefetch.global.L2 [%0];" ::"l"(p.u0 + nxt * 3));
            }
        }
    };
    asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory");
    for (long long it = 0; it < nt; ++it) {
        const long long b0 = ubase(it);
        double v[2][7];
        if (tmain) {
            asm volatile(
                "{\n.reg .pred q;\nW_%=:\nmbarrier.try_wait.parity.shared::cta.b64 q, [%0], %1;\n@q bra D_%=;\nbra W_%=;\nD_%=:\n}\n" ::"r"(smem_u32(bar)),
                "r"(phase)
                : "memory");
            phase ^= 1u;
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const int q = warp * G + r * 32 + lane;
                const long long ray = b0 + q;
                // (past the end: the tile's last ray, or slot 0 of a tile that
                // loaded nothing and stores nothing)
                const int qq = ray < p.N ? q : b0 < p.N ? (int)(p.N - 1 - b0) : 0;
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    v[r][c] = xb[qq * 3 + c];
                    v[r][3 + c] = xb[3 * CT + qq * 3 + c];
                }
                v[r][6] = 0.0;
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncthreads();
            if (threadIdx.x == 0 && it + 1 < nt) load_in(ubase(it + 1));
        } else {
            ldg_tile(v, b0);
        }
        if constexpr (PAIR) {
            double w[2][7];
            ldg_tile(w, b0 + CT);
#pragma unroll
            for (int r = 0; r < 2; ++r)
#pragma unroll
                for (int c = 0; c < 7; ++c) xb[c * CT + warp * G + r * 32 + lane] = w[r][c];
        }
#pragma unroll 1
        for (int s = 0; s < p.S; ++s) {
            kf_march(v, p.D);
            asm volatile("barrier.cluster.wait.aligned;" ::: "memory");
            kf_store(p, sb, v, b0, s, pol);
            if constexpr (PAIR) {
                double w[2][7];
#pragma unroll
                for (int r = 0; r < 2; ++r)
#pragma unroll
                    for (int c = 0; c < 7; ++c) w[r][c] = xb[c * CT + warp * G + r * 32 + lane];
                kf_march(w, p.D);
#pragma unroll
                for (int r = 0; r < 2; ++r)
#pragma unroll
                    for (int c = 0; c < 7; ++c) xb[c * CT + warp * G + r * 32 + lane] = w[r][c];
                kf_store(p, sb, w, b0 + CT, s, pol);
            }
            asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory");
        }
#pragma unroll
        for (int t = 0; t < NT; ++t)
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const long long ray = b0 + t * CT + warp * G + r * 32 + lane;
                const double acc = t == 0 ? v[r][6] : xb[6 * CT + warp * G + r * 32 + lane];
                if (p.tsum != nullptr && ray < p.N) p.tsum[ray] = acc;
            }
    }
    asm volatile("barrier.cluster.wait.aligned;" ::: "memory");
    if (threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

// number of non-finite values in p[0, n) (checks that a variant wrote every row)
__global__ void count_nonfinite(const double* p, long long n, unsigned long long* out) {
    unsigned long long c = 0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        c += !isfinite(p[i]);
    atomicAdd(out, c);
}

// The store-pattern study: every kf variant at D = 0 and 57, rounds
// alternating over the variants, then median and range per variant.
static int study(double* Y, double* U, double* I, double* T, double* in, long long N, long long ld, int sms, int rounds) {
    const int S = 12;
    unsigned long long* cnt;
    cudaMalloc(&cnt, 8);
    struct Var { const char* name; bool pair; int flags; int cap; };
    const Var vars[] = {
        {"kernel (prefetch, 7 clusters)", false, KF_PF, 0},
        {"no prefetch", false, 0, 0},
        {"(a) 6 clusters", false, KF_PF, 6},
        {"(a) 5 clusters", false, KF_PF, 5},
        {"(a) 4 clusters", false, KF_PF, 4},
        {"(a) 6 clusters, no prefetch", false, 0, 6},
        {"(b) tile pairs", true, KF_PF, 0},
        {"(b) tile pairs, 5 clusters", true, KF_PF, 5},
        {"(c) TMA ray loads", false, KF_TMAIN, 0},
    };
    const int NV = sizeof(vars) / sizeof(vars[0]);
    const size_t smem1 = (size_t)(10 + 6) * 1024 * 8 + 16, smem2 = (size_t)(10 + 7) * 1024 * 8 + 16;
    cudaFuncSetAttribute(kf<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem1);
    cudaFuncSetAttribute(kf<false>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
    cudaFuncSetAttribute(kf<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem2);
    cudaFuncSetAttribute(kf<true>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    std::vector<float> res[16][2];
    const int Ds[2] = {0, 57};
    for (int round = 0; round < rounds; ++round)
        for (int di = 0; di < 2; ++di)
            for (int v = 0; v < NV; ++v) {
                const Var& va = vars[v];
                const bool pair = va.pair;
                PF p{Y, U, I, T, nullptr, in, in + 3 * N, N, ld, S, Ds[di], va.flags};
                cudaLaunchConfig_t cfg = {};
                cudaLaunchAttribute attr[1];
                attr[0].id = cudaLaunchAttributeClusterDimension;
                attr[0].val.clusterDim.x = 16;
                attr[0].val.clusterDim.y = 1;
                attr[0].val.clusterDim.z = 1;
                cfg.blockDim = dim3(512);
                cfg.dynamicSmemBytes = pair ? smem2 : smem1;
                cfg.attrs = attr;
                cfg.numAttrs = 1;
                cfg.gridDim = dim3(sms / 16 * 16);
                int ncl = 0;
                cudaError_t eo = pair ? cudaOccupancyMaxActiveClusters(&ncl, kf<true>, &cfg)
                                      : cudaOccupancyMaxActiveClusters(&ncl, kf<false>, &cfg);
                if (eo != cudaSuccess || ncl < 1) {
                    printf("%s: no active cluster (%s)\n", va.name, cudaGetErrorString(eo));
                    return 1;
                }
                if (va.cap > 0 && va.cap < ncl) ncl = va.cap;
                cfg.gridDim = dim3(ncl * 16);
                auto launch = [&] { if (pair) cudaLaunchKernelEx(&cfg, kf<true>, p); else cudaLaunchKernelEx(&cfg, kf<false>, p); };
                if (round == 0 && di == 0) {  // every row written: no NaN left of the fill
                    cudaMemset(T, 0xff, (size_t)S * ld * 8);
                    cudaMemset(Y, 0xff, (size_t)S * ld * 24);
                    cudaMemset(cnt, 0, 8);
                    launch();
                    count_nonfinite<<<sms * 4, 256>>>(T, (long long)S * ld, cnt);
                    count_nonfinite<<<sms * 4, 256>>>(Y, (long long)S * ld * 3, cnt);
                    unsigned long long c = 0;
                    const cudaError_t ec = cudaMemcpy(&c, cnt, 8, cudaMemcpyDeviceToHost);
                    if (ec != cudaSuccess) {
                        printf("check %s: %s\n", va.name, cudaGetErrorString(ec));
                        return 1;
                    }
                    printf("check %-30s ctas %3d: %llu non-finite of %lld\n", va.name, ncl * 16, c, (long long)S * ld * 4);
                }
                std::vector<float> t;
                for (int i = 0; i < 8; ++i) {
                    cudaEventRecord(e0);
                    launch();
                    cudaEventRecord(e1); cudaEventSynchronize(e1);
                    float ms; cudaEventElapsedTime(&ms, e0, e1);
                    if (i >= 2) t.push_back(ms);
                }
                cudaError_t e = cudaGetLastError();
                if (e != cudaSuccess) { printf("%s: %s\n", va.name, cudaGetErrorString(e)); return 1; }
                std::sort(t.begin(), t.end());
                res[v][di].push_back(t[t.size() / 2]);
            }
    const double gb = (double)N * (48 + 80.0 * S) / 1e9;
    printf("\nstore-pattern study: S %d, N %lld, 16-CTA clusters, %d rounds x median of 6 launches\n", S, N, rounds);
    printf("%-30s %-36s %-36s\n", "variant", "D = 0: median ms (min-max) GB/s", "D = 57: median ms (min-max) GB/s");
    for (int v = 0; v < NV; ++v) {
        printf("%-30s", vars[v].name);
        for (int di = 0; di < 2; ++di) {
            std::vector<float> r = res[v][di];
            std::sort(r.begin(), r.end());
            const double med = r[r.size() / 2];
            printf(" %6.3f (%6.3f-%6.3f) %7.1f    ", med, r.front(), r.back(), gb / (med * 1e-3));
        }
        printf("\n");
    }
    cudaFree(cnt);
    return 0;
}

int main(int argc, char** argv) {
    const long long N = 10000000, ld = N;
    const int Smax = 12;
    double *Y, *U, *I, *T, *in;
    cudaMalloc(&Y, (size_t)Smax * ld * 24); cudaMalloc(&U, (size_t)Smax * ld * 24);
    cudaMalloc(&I, (size_t)Smax * ld * 24); cudaMalloc(&T, (size_t)Smax * ld * 8);
    cudaMalloc(&in, (size_t)N * 48);
    cudaMemset(in, 0, (size_t)N * 48);
    int sms; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    auto run = [&](const char* name, int rpt, int threads, int occ, int S, int D, int mode) {
        P p{Y, U, I, T, in, N, ld, S, D, mode};
        size_t smem = (size_t)(threads / 32) * 2 * 10 * 32 * rpt * 8;
        std::vector<float> t;
        for (int i = 0; i < 8; ++i) {
            cudaEventRecord(e0);
            if (rpt == 1) { cudaFuncSetAttribute(k<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); k<1><<<sms * occ, threads, smem>>>(p); }
            else { cudaFuncSetAttribute(k<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); k<2><<<sms * occ, threads, smem>>>(p); }
            cudaEventRecord(e1); cudaEventSynchronize(e1);
            float ms; cudaEventElapsedTime(&ms, e0, e1);
            if (i >= 2) t.push_back(ms);
        }
        cudaError_t e = cudaGetLastError();
        std::sort(t.begin(), t.end());
        double gb = (double)N * (48 + 80.0 * S) / 1e9;
        printf("%-10s rpt %d thr %4d occ %d S %2d D %3d lock %d tilemajor %d: %7.3f ms  %7.1f GB/s %s\n", name, rpt, threads, occ, S, D, mode & 1, (mode >> 1) & 1, t[t.size() / 2], gb / (t[t.size() / 2] * 1e-3), e == cudaSuccess ? "" : cudaGetErrorString(e));
    };
    // `tracelike.bin study [rounds]`: the kf levers, then the tile-major ceiling
    if (argc > 1 && !strcmp(argv[1], "study")) {
        const int rc = study(Y, U, I, T, in, N, ld, sms, argc > 2 ? atoi(argv[2]) : 3);
        for (int i = 0; i < 3; ++i) run("tilemajor", 2, 256, 2, 12, 0, 2);
        return rc;
    }
    // upper bound with perfect locality (tile-major layout)
    for (int occ : {2, 4}) run("tilemajor", 1, 256, occ, 12, 0, 2);
    run("tilemajor", 2, 256, 2, 12, 0, 2);
    run("tilemajor", 2, 256, 2, 12, 64, 2);
    // CTA lockstep with growing CTA size (contiguous burst per row = threads*rpt*24 B)
    for (int thr : {256, 512, 1024})
        for (int lockm : {0, 1}) {
            int occ = thr == 1024 ? 1 : (thr == 512 ? 2 : 4);
            run("rowmajor", 1, thr, occ, 12, 0, lockm);
            run("rowmajor", 1, thr, occ, 12, 64, lockm);
        }
    for (int lockm : {0, 1}) { run("rowmajor", 2, 1024, 1, 12, 0, lockm); run("rowmajor", 2, 1024, 1, 12, 32, lockm); run("rowmajor", 2, 512, 2, 12, 32, lockm); }

    // cluster lockstep at the trace kernel's shape: 512 threads, RPT 2, one
    // CTA per SM (the kernel's 105 registers allow no second one; here the
    // shared memory request is padded so that two do not fit either)
    const size_t smem_c = 116 * 1024;
    cudaFuncSetAttribute(kc<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_c);
    cudaFuncSetAttribute(kc<2>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
    auto runc = [&](int cs, int S, int D) {
        P p{Y, U, I, T, in, N, ld, S, D, 1};
        cudaLaunchConfig_t cfg = {};
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeClusterDimension;
        attr[0].val.clusterDim.x = cs;
        attr[0].val.clusterDim.y = 1;
        attr[0].val.clusterDim.z = 1;
        cfg.blockDim = dim3(512);
        cfg.dynamicSmemBytes = smem_c;
        cfg.attrs = attr;
        cfg.numAttrs = 1;
        cfg.gridDim = dim3(sms / cs * cs);
        int ncl = 0;
        cudaError_t eo = cudaOccupancyMaxActiveClusters(&ncl, kc<2>, &cfg);
        if (eo != cudaSuccess || ncl < 1) {
            printf("cluster    CS %d: no active cluster (%s)\n", cs, cudaGetErrorString(eo));
            cudaGetLastError();
            return;
        }
        cfg.gridDim = dim3(ncl * cs);
        std::vector<float> t;
        for (int i = 0; i < 8; ++i) {
            cudaEventRecord(e0);
            cudaLaunchKernelEx(&cfg, kc<2>, p);
            cudaEventRecord(e1); cudaEventSynchronize(e1);
            float ms; cudaEventElapsedTime(&ms, e0, e1);
            if (i >= 2) t.push_back(ms);
        }
        cudaError_t e = cudaGetLastError();
        std::sort(t.begin(), t.end());
        double gb = (double)N * (48 + 80.0 * S) / 1e9;
        double med = t[t.size() / 2];
        printf("cluster    rpt 2 thr  512 occ 1 S %2d D %3d CS %d ctas %3d: %7.3f ms (min %7.3f)  %7.1f GB/s %s\n", S, D, cs, ncl * cs, med, t.front(), gb / (med * 1e-3), e == cudaSuccess ? "" : cudaGetErrorString(e));
    };
    // (16 is a non-portable cluster size: it needs a GPC with 16 free SMs)
    for (int D : {0, 32, 57})
        for (int cs : {1, 2, 4, 8, 16}) runc(cs, 12, D);
    for (int cs : {1, 2, 4, 8, 16}) runc(cs, 1, 0);
    // repeat the D = 0 row to show the run-to-run spread
    for (int cs : {1, 2, 4, 8, 16}) runc(cs, 12, 0);
    return 0;
}
