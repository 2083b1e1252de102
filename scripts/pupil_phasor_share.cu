// Share of the phasor generation in rtx_pupil_sum's kernel: the kernel as the
// library builds it against the same kernel with the products left out
// (PHASORS_ONLY), on the same synthetic rays and grids, CUDA events, median
// of repeats.  Built and run by scripts/pupil_timing.py; prints JSON lines.
#include "../include/rtx.h"
#include "../rayopt_b200/csrc/rtx_pupil.cuh"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <vector>

using namespace rtx;

template <int WR, int WC, bool P>
float run(PupilDev d, int reps) {
    using SM = PupilSmem<WR, WC>;
    d.tiles_x = (int)((d.nx + SM::TA - 1) / SM::TA);
    d.tiles_y = (int)((d.ny + SM::TB - 1) / SM::TB);
    const long long items = d.slots * d.groups * d.tiles_x * d.tiles_y;
    const size_t smem = (size_t)SM::doubles * sizeof(double);
    auto k = pupil_sum_kernel<WR, WC, P>;
    cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    cudaEvent_t a, b;
    cudaEventCreate(&a);
    cudaEventCreate(&b);
    std::vector<float> ms;
    for (int r = 0; r <= reps; ++r) {   // the first is the warm-up
        cudaEventRecord(a);
        k<<<(unsigned)items, PUP_THREADS, smem>>>(d);
        cudaEventRecord(b);
        cudaEventSynchronize(b);
        float t = 0;
        cudaEventElapsedTime(&t, a, b);
        if (r) ms.push_back(t);
    }
    std::sort(ms.begin(), ms.end());
    return ms[ms.size() / 2];
}

int main() {
    const double lam = 5e-4, R = 50., pitch = .61 * lam / .2 / 8;
    for (long long N : {100000LL, 1000000LL}) {
        std::vector<double> A(N), P(3 * N);
        for (long long j = 0; j < N; ++j) {   // a golden-angle spiral over NA 0.2
            const double r = 10 * std::sqrt((j + .5) / N), th = 2.399963229728653 * j;
            P[3 * j] = r * std::cos(th);
            P[3 * j + 1] = r * std::sin(th);
            P[3 * j + 2] = -std::sqrt(R * R - r * r);
            A[j] = 100 + 3e-4 * std::pow(r / 10, 4);
        }
        double *dA, *dP, *part;
        cudaMalloc(&dA, N * 8);
        cudaMalloc(&dP, 3 * N * 8);
        cudaMemcpy(dA, A.data(), N * 8, cudaMemcpyHostToDevice);
        cudaMemcpy(dP, P.data(), 3 * N * 8, cudaMemcpyHostToDevice);
        for (int n : {256, 512})
            for (int K : {1, 5}) {
                PupilDev d = {};
                d.K = K;
                d.groups = 1;
                d.KG = K;
                d.nx = d.ny = n;
                d.N = N;
                long long L = std::max<long long>(RTX_PUPIL_SLOT, (N + RTX_PUPIL_MAX_SLOTS - 1) / RTX_PUPIL_MAX_SLOTS);
                d.L = (L + PUP_CH - 1) / PUP_CH * PUP_CH;
                d.slots = (N + d.L - 1) / d.L;
                d.a0 = 100;
                d.lambda = lam;
                d.kappa = 1 / lam;
                d.radius = R;
                d.p0 = d.q0 = -(n / 2) * pitch;
                d.dp = d.dq = pitch;
                for (int k = 0; k < K; ++k) d.z[k] = .01 * k;
                d.A = dA;
                d.P = dP;
                cudaMalloc(&part, (size_t)d.slots * (2LL * K * n * n + 2) * 8);
                d.part = part;
                float full, phas;
                if (K == 1) {
                    full = run<2, 4, false>(d, 5);
                    phas = run<2, 4, true>(d, 5);
                } else {
                    full = run<1, 1, false>(d, 5);
                    phas = run<1, 1, true>(d, 5);
                }
                printf("{\"N\": %lld, \"grid\": %d, \"K\": %d, \"kernel_ms\": %.4f, "
                       "\"phasors_only_ms\": %.4f, \"phasor_share\": %.3f, \"error\": \"%s\"}\n",
                       N, n, K, full, phas, phas / full, cudaGetErrorString(cudaGetLastError()));
                cudaFree(part);
            }
        cudaFree(dA);
        cudaFree(dP);
    }
    return 0;
}
