// membw.cu -- HBM bandwidth ceilings for the access patterns of the trace
// kernel (write-dominated): plain STG.128 fill, TMA bulk-store fill from
// shared memory (the kernel's store path), read-only, and copy (the pattern
// MEASURED_PEAKS.json's hbm_gbs was measured with).  CUDA events, 10 GB
// buffers (>> 126 MB L2), best and median of 10.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o membw.bin membw.cu
#include <cuda_runtime.h>
#include <algorithm>
#include <cstdio>
#include <cstdint>
#include <vector>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); return 1; } } while (0)

__global__ void fill128(double2* p, size_t n, double v) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t st = (size_t)gridDim.x * blockDim.x;
    double2 x = make_double2(v, v);
    for (; i < n; i += st) p[i] = x;
}
__global__ void fill128_cs(double2* p, size_t n, double v) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t st = (size_t)gridDim.x * blockDim.x;
    double2 x = make_double2(v, v);
    for (; i < n; i += st) __stcs(p + i, x);
}
__global__ void read128(const double2* p, size_t n, double* out) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t st = (size_t)gridDim.x * blockDim.x;
    double acc = 0;
    for (; i < n; i += st) { double2 x = __ldg(p + i); acc += x.x + x.y; }
    if (acc == 1.2345) *out = acc;
}
__global__ void copy128(double2* d, const double2* s, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t st = (size_t)gridDim.x * blockDim.x;
    for (; i < n; i += st) d[i] = __ldg(s + i);
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// every warp owns a CHUNK-byte staging buffer (x2) and streams it out with
// cp.async.bulk; `narr` separate output arrays written round-robin like y,u,i
template <int CHUNK>
__global__ void __launch_bounds__(256) bulk_fill(char* base, size_t bytes_per_arr, int narr, double v) {
    extern __shared__ __align__(128) unsigned char sm[];
    const int lane = threadIdx.x & 31;
    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
    double* buf = reinterpret_cast<double*>(sm + (size_t)warp * 2 * CHUNK);
    size_t nchunk = bytes_per_arr / CHUNK;
    size_t stride = (size_t)gridDim.x * 8;
    int b = 0;
    for (size_t c = (size_t)blockIdx.x * 8 + warp; c < nchunk; c += stride) {
        for (int a = 0; a < narr; ++a) {
            double* sb = buf + b * (CHUNK / 8);
            if (lane == 0) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
            __syncwarp();
            for (int k = lane; k < CHUNK / 8; k += 32) sb[k] = v + k;
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncwarp();
            if (lane == 0) {
                char* dst = base + (size_t)a * bytes_per_arr + c * CHUNK;
                asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(smem_u32(sb)), "r"(CHUNK) : "memory");
                asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            }
            b ^= 1;
        }
    }
    if (lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

template <class F>
int timeit(const char* name, double gbytes, F f) {
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    std::vector<float> t;
    for (int i = 0; i < 13; ++i) {
        cudaEventRecord(e0);
        f();
        cudaEventRecord(e1);
        cudaEventSynchronize(e1);
        float ms; cudaEventElapsedTime(&ms, e0, e1);
        if (i >= 3) t.push_back(ms);
    }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { printf("%s: CUDA error %s\n", name, cudaGetErrorString(e)); return 1; }
    std::sort(t.begin(), t.end());
    printf("%-44s best %7.1f GB/s   median %7.1f GB/s\n", name, gbytes / (t.front() * 1e-3), gbytes / (t[t.size() / 2] * 1e-3));
    return 0;
}

int main() {
    const size_t bytes = (size_t)10 << 30;  // 10 GiB
    const double gb = bytes / 1e9;
    char *a, *b;
    CK(cudaMalloc(&a, bytes)); CK(cudaMalloc(&b, bytes));
    double* out; CK(cudaMalloc(&out, 8));
    CK(cudaMemset(a, 0, bytes)); CK(cudaMemset(b, 0, bytes));
    int sms; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    const size_t n16 = bytes / 16;
    for (int occ : {4, 8}) {
        char nm[96];
        snprintf(nm, 96, "write STG.128 fill (grid %dx%d)", sms, occ);
        timeit(nm, gb, [&] { fill128<<<sms * occ, 256>>>((double2*)a, n16, 1.0); });
    }
    timeit("write STG.128.CS (evict-first) fill", gb, [&] { fill128_cs<<<sms * 8, 256>>>((double2*)a, n16, 1.0); });
    timeit("write cudaMemsetAsync", gb, [&] { cudaMemsetAsync(a, 1, bytes); });
    timeit("read LDG.128", gb, [&] { read128<<<sms * 8, 256>>>((const double2*)a, n16, out); });
    timeit("copy LDG.128->STG.128 (read+write bytes)", 2 * gb, [&] { copy128<<<sms * 8, 256>>>((double2*)b, (const double2*)a, n16); });
    timeit("copy cudaMemcpyAsync D2D (read+write bytes)", 2 * gb, [&] { cudaMemcpyAsync(b, a, bytes, cudaMemcpyDeviceToDevice); });
    // TMA bulk-store fills: chunk size / number of arrays / CTAs per SM
    cudaFuncSetAttribute(bulk_fill<768>, cudaFuncAttributeMaxDynamicSharedMemorySize, 8 * 2 * 768);
    cudaFuncSetAttribute(bulk_fill<1536>, cudaFuncAttributeMaxDynamicSharedMemorySize, 8 * 2 * 1536);
    cudaFuncSetAttribute(bulk_fill<4096>, cudaFuncAttributeMaxDynamicSharedMemorySize, 8 * 2 * 4096);
    for (int occ : {2, 4}) {
        char nm[96];
        snprintf(nm, 96, "write TMA bulk 768 B x1 array (occ %d)", occ);
        timeit(nm, gb, [&] { bulk_fill<768><<<sms * occ, 256, 8 * 2 * 768>>>(a, bytes, 1, 1.0); });
        snprintf(nm, 96, "write TMA bulk 768 B x4 arrays (occ %d)", occ);
        timeit(nm, gb, [&] { bulk_fill<768><<<sms * occ, 256, 8 * 2 * 768>>>(a, bytes / 4, 4, 1.0); });
        snprintf(nm, 96, "write TMA bulk 1536 B x4 arrays (occ %d)", occ);
        timeit(nm, gb, [&] { bulk_fill<1536><<<sms * occ, 256, 8 * 2 * 1536>>>(a, bytes / 4, 4, 1.0); });
        snprintf(nm, 96, "write TMA bulk 4096 B x1 array (occ %d)", occ);
        timeit(nm, gb, [&] { bulk_fill<4096><<<sms * occ, 256, 8 * 2 * 4096>>>(a, bytes, 1, 1.0); });
    }
    return 0;
}
