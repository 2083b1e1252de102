// tracelike.cu -- synthetic kernel with the trace kernel's memory pattern and
// a tunable amount of dependent FP64 work, to separate memory-pattern effects
// from compute effects.  Per warp tile (32*RPT rays): for s in 0..S-1:
// D dependent DFMAs per ray, stage 10 values/ray, NARR bulk stores to row s.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tracelike.bin tracelike.cu
#include <cuda_runtime.h>
#include <algorithm>
#include <cstdio>
#include <cstdint>
#include <cstdlib>
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
    return 0;
}
