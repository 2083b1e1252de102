// rtx_pupil.cuh -- device side of the direct-sum diffraction PSF (sm_90a,
// FP64): rtx_pupil_sum and rtx_pupil_intensity (include/rtx.h).
//
//   sum        U_k = X^T diag(c_k) Y per plane on the FP64 tensor cores
//              (mma.m16n8k16.f64).  A CTA owns one slot of rays and one tile
//              of pixels for a group of up to 8 planes; per chunk of
//              PUP_CH rays it builds X (rays x tile rows), Y (rays x tile
//              columns) and c (planes x rays) in shared memory, then every
//              warp multiplies its 32 x 16 pixels of one plane.  Each chunk
//              is summed into a fresh accumulator and added to the slot sum
//              in chunk order; pupil_fold_kernel adds the slots in order.
//   intensity  scale |U|^2 added to the PSF, with per-plane sums, maximum
//              and first moments reduced in a fixed order.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace rtx {

constexpr int PUP_CH = RTX_PUPIL_CHUNK;   // rays per chunk: two k16 steps
constexpr int PUP_WARPS = 8;
constexpr int PUP_THREADS = PUP_WARPS * 32;
constexpr int PUP_BLK = 8;                // pixels per sincospi, then phasor steps
constexpr int PUP_GROUP = 8;              // planes that share a chunk's X and Y
constexpr int PUP_RED = 2048;             // pixels per block of the intensity reduction
static_assert(PUP_CH == 32, "the chunk is two k16 steps of the mma");

// rtx_pupil as the kernels read it (rtx.cu has checked it)
struct PupilDev {
    int K, KG, groups;          // planes, planes per group, plane groups
    int tiles_x, tiles_y;       // pixel tiles along a and b
    long long nx, ny, N, L;     // L: rays per slot
    long long slots;
    double a0, lambda, kappa, radius;
    double p0, dp, q0, dq;
    double z[RTX_PUPIL_MAX_PLANES];
    const double* A;
    const double* P;
    const double* w;            // NULL: all 1
    double* part;               // slots x (2 K nx ny + 2): U, then count and sum w
};

// D = C + A B, A 16x16 (row), B 16x8 (col), FP64.  Fragments (lane = 4 g + t):
// a[i] = A[g + 8 (i & 1)][t + 4 (i >> 1)], b[i] = B[t + 4 i][g],
// c[i] = C[g + 8 (i >> 1)][2 t + (i & 1)].
__device__ __forceinline__ void dmma16816(double (&c)[4], const double (&a)[8],
                                          const double (&b)[4]) {
    asm("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 "
        "{%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, {%0,%1,%2,%3};"
        : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
        : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]),
          "d"(a[7]), "d"(b[0]), "d"(b[1]), "d"(b[2]), "d"(b[3]));
}

// (xr + i xi)(yr + i yi), each component one fma on one rounded product
__device__ __forceinline__ void cmul(double xr, double xi, double yr, double yi, double& r,
                                     double& i) {
    r = __fma_rn(xr, yr, -__dmul_rn(xi, yi));
    i = __fma_rn(xr, yi, __dmul_rn(xi, yr));
}

// Shared memory of pupil_sum_kernel<WR, WC> in doubles: the chunk's ray
// terms, c (re, im) of PUP_GROUP planes, X (re, im) and Y (re, im) with row
// pitches 4 mod 16 doubles, so that the fragment loads do not conflict.
template <int WR, int WC>
struct PupilSmem {
    static constexpr int TA = 32 * WR, TB = 16 * WC;   // CTA tile per plane
    static constexpr int LDX = TA + 4, LDY = TB + 4;
    static constexpr int RAY = 10 * PUP_CH;            // kx ky kz d w Dx Dy valid
    static constexpr int CS = 2 * PUP_GROUP * PUP_CH;
    static constexpr int XS = 2 * PUP_CH * LDX, YS = 2 * PUP_CH * LDY;
    static constexpr int doubles = RAY + CS + XS + YS;
};

// PHASORS_ONLY (scripts/pupil_phasor_share.cu, never in the library): the
// same kernel without the products, to time the phasor generation alone
template <int WR, int WC, bool PHASORS_ONLY = false>
__global__ void __launch_bounds__(PUP_THREADS, 1) pupil_sum_kernel(const PupilDev s) {
    using SM = PupilSmem<WR, WC>;
    constexpr int TA = SM::TA, TB = SM::TB, LDX = SM::LDX, LDY = SM::LDY;
    constexpr int WPP = WR * WC;                       // warps per plane
    extern __shared__ double smem[];
    double* rkx = smem;
    double* rky = rkx + PUP_CH;
    double* rkz = rky + PUP_CH;
    double* rd = rkz + PUP_CH;
    double* rw = rd + PUP_CH;
    double* rdx = rw + PUP_CH;                         // (re, im) of the dp step
    double* rdy = rdx + 2 * PUP_CH;                    // (re, im) of the dq step
    double* rok = rdy + 2 * PUP_CH;                    // 1: summed, 0: left out
    double* csr = smem + SM::RAY;
    double* csi = csr + PUP_GROUP * PUP_CH;
    double* xr = csr + SM::CS;
    double* xi = xr + PUP_CH * LDX;
    double* yr = xr + SM::XS;
    double* yi = yr + PUP_CH * LDY;

    const int tiles = s.tiles_x * s.tiles_y;
    const long long item = blockIdx.x;
    const long long slot = item / ((long long)s.groups * tiles);
    const int group = (int)((item / tiles) % s.groups);
    const int tile = (int)(item % tiles);
    const long long ta0 = (long long)(tile / s.tiles_y) * TA;
    const long long tb0 = (long long)(tile % s.tiles_y) * TB;
    const bool tally = group == 0 && tile == 0;        // this CTA counts the slot
    const long long j0 = slot * s.L;
    const long long j1 = min(s.N, j0 + s.L);

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int g = lane >> 2, t = lane & 3;
    const int kk = warp / WPP;                         // plane within the group
    const int plane = group * s.KG + kk;
    const bool active = kk < s.KG && plane < s.K;
    const int wr = (warp % WPP) / WC, wc = (warp % WPP) % WC;

    double tot[2][2][2][4], acc[2][2][2][4];           // [row][col][re, im][frag]
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
        for (int c = 0; c < 2; ++c)
#pragma unroll
            for (int q = 0; q < 2; ++q)
#pragma unroll
                for (int i = 0; i < 4; ++i) tot[r][c][q][i] = 0.0;
    double count = 0.0, sumw = 0.0;

    for (long long c0 = j0; c0 < j1; c0 += PUP_CH) {
        // 1. the chunk's rays: left-out rays and those past the slot get
        //    zero directions and weight, so their terms are exactly 0
        if (threadIdx.x < PUP_CH) {
            const int j = threadIdx.x;
            const long long r = c0 + j;
            double kx = 0.0, ky = 0.0, kz = 0.0, d = 0.0, w = 0.0, ok = 0.0;
            if (r < j1) {
                const double a = s.A[r];
                const double px = s.P[3 * r], py = s.P[3 * r + 1], pz = s.P[3 * r + 2];
                const double wr_ = s.w ? s.w[r] : 1.0;
                if (isfinite(a) && isfinite(px) && isfinite(py) && isfinite(pz) && isfinite(wr_)) {
                    kx = __dmul_rn(s.kappa, __ddiv_rn(-px, s.radius));
                    ky = __dmul_rn(s.kappa, __ddiv_rn(-py, s.radius));
                    kz = __dmul_rn(s.kappa, __ddiv_rn(-pz, s.radius));
                    d = __ddiv_rn(__dsub_rn(a, s.a0), s.lambda);
                    w = wr_;
                    ok = 1.0;
                }
            }
            rkx[j] = kx;
            rky[j] = ky;
            rkz[j] = kz;
            rd[j] = d;
            rw[j] = w;
            rok[j] = ok;
            double sn, cs;
            sincospi(2.0 * __dmul_rn(kx, s.dp), &sn, &cs);
            rdx[2 * j] = cs;
            rdx[2 * j + 1] = sn;
            sincospi(2.0 * __dmul_rn(ky, s.dq), &sn, &cs);
            rdy[2 * j] = cs;
            rdy[2 * j + 1] = sn;
        }
        __syncthreads();
        if (tally && threadIdx.x == 0) {
            double n = 0.0, sw = 0.0;
            for (int j = 0; j < PUP_CH; ++j) {
                n += rok[j];
                sw += rw[j];
            }
            count += n;
            sumw += sw;
        }
        // 2. c of the group's planes, X and Y in blocks of PUP_BLK pixels
        constexpr int NC = PUP_GROUP * PUP_CH, NX = PUP_CH * (TA / PUP_BLK),
                      NY = PUP_CH * (TB / PUP_BLK);
        for (int e = threadIdx.x; e < NC + NX + NY; e += PUP_THREADS) {
            if (e < NC) {
                const int k = e / PUP_CH, j = e % PUP_CH, pk = group * s.KG + k;
                double sn = 0.0, cs = 0.0;
                if (k < s.KG && pk < s.K) {
                    sincospi(2.0 * __dadd_rn(rd[j], __dmul_rn(rkz[j], s.z[pk])), &sn, &cs);
                    sn = __dmul_rn(rw[j], sn);
                    cs = __dmul_rn(rw[j], cs);
                }
                csr[k * PUP_CH + j] = cs;
                csi[k * PUP_CH + j] = sn;
                continue;
            }
            const bool isx = e < NC + NX;
            const int f = isx ? e - NC : e - NC - NX;
            const int nb = (isx ? TA : TB) / PUP_BLK;
            const int j = f / nb, blk = f % nb;
            const long long a = (isx ? ta0 : tb0) + blk * PUP_BLK;
            const double k = isx ? rkx[j] : rky[j];
            const double p = isx ? __dadd_rn(s.p0, __dmul_rn((double)a, s.dp))
                                 : __dadd_rn(s.q0, __dmul_rn((double)a, s.dq));
            const double* st = isx ? rdx + 2 * j : rdy + 2 * j;
            const double sr = st[0], si = st[1];
            double er, ei;
            sincospi(2.0 * __dmul_rn(k, p), &ei, &er);
            double* outr = isx ? xr + j * LDX + blk * PUP_BLK : yr + j * LDY + blk * PUP_BLK;
            double* outi = isx ? xi + j * LDX + blk * PUP_BLK : yi + j * LDY + blk * PUP_BLK;
#pragma unroll
            for (int i = 0; i < PUP_BLK; ++i) {
                outr[i] = er;
                outi[i] = ei;
                double nr, ni;
                cmul(er, ei, sr, si, nr, ni);
                er = nr;
                ei = ni;
            }
        }
        __syncthreads();
        // 3. this warp's 32 x 16 pixels of plane `plane`: a fresh accumulator
        if (active && !PHASORS_ONLY) {
#pragma unroll
            for (int r = 0; r < 2; ++r)
#pragma unroll
                for (int c = 0; c < 2; ++c)
#pragma unroll
                    for (int q = 0; q < 2; ++q)
#pragma unroll
                        for (int i = 0; i < 4; ++i) acc[r][c][q][i] = 0.0;
#pragma unroll
            for (int step = 0; step < PUP_CH / 16; ++step) {
                const int kb = 16 * step;
                double br[2][4], bi[2][4], bn[2][4];   // c_k Y: re, im, -im
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    const int col = wc * 16 + c * 8 + g;
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const int j = kb + t + 4 * i;
                        cmul(csr[kk * PUP_CH + j], csi[kk * PUP_CH + j], yr[j * LDY + col],
                             yi[j * LDY + col], br[c][i], bi[c][i]);
                        bn[c][i] = -bi[c][i];
                    }
                }
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    const int row = wr * 32 + r * 16 + g;
                    double ar[8], ai[8];
#pragma unroll
                    for (int i = 0; i < 8; ++i) {
                        const int j = kb + t + 4 * (i >> 1), m = row + 8 * (i & 1);
                        ar[i] = xr[j * LDX + m];
                        ai[i] = xi[j * LDX + m];
                    }
#pragma unroll
                    for (int c = 0; c < 2; ++c) {
                        dmma16816(acc[r][c][0], ar, br[c]);
                        dmma16816(acc[r][c][0], ai, bn[c]);
                        dmma16816(acc[r][c][1], ar, bi[c]);
                        dmma16816(acc[r][c][1], ai, br[c]);
                    }
                }
            }
#pragma unroll
            for (int r = 0; r < 2; ++r)
#pragma unroll
                for (int c = 0; c < 2; ++c)
#pragma unroll
                    for (int q = 0; q < 2; ++q)
#pragma unroll
                        for (int i = 0; i < 4; ++i)
                            tot[r][c][q][i] = __dadd_rn(tot[r][c][q][i], acc[r][c][q][i]);
        }
        // (the next chunk's stage 1 writes only the ray terms; the barrier
        // after it orders stage 3's reads of X, Y, c before stage 2's writes)
    }
    double* out = s.part + slot * (2 * s.K * s.nx * s.ny + 2);
    if (active) {
#pragma unroll
        for (int r = 0; r < 2; ++r)
#pragma unroll
            for (int c = 0; c < 2; ++c)
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const long long a = ta0 + wr * 32 + r * 16 + g + 8 * (i >> 1);
                    const long long b = tb0 + wc * 16 + c * 8 + 2 * t + (i & 1);
                    if (a < s.nx && b < s.ny) {
                        const long long e = ((long long)plane * s.nx + a) * s.ny + b;
                        out[2 * e] = tot[r][c][0][i];
                        out[2 * e + 1] = tot[r][c][1][i];
                    }
                }
    }
    if (tally && threadIdx.x == 0) {
        out[2 * s.K * s.nx * s.ny] = count;
        out[2 * s.K * s.nx * s.ny + 1] = sumw;
    }
}

// U[e] += sum over the slots, in slot order, of part[slot][e]
__global__ void __launch_bounds__(256) pupil_fold_kernel(const double* __restrict__ part,
                                                         long long row, long long n,
                                                         long long slots, double* U) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    double v = 0.0;
    for (long long q = 0; q < slots; ++q) v = __dadd_rn(v, part[q * row + e]);
    U[e] = __dadd_rn(U[e], v);
}

// psf += scale |U|^2 per pixel; per block of PUP_RED pixels of one plane:
// sum, max, its index, sum psf p, sum psf q (pixels in index order per
// thread, then a fixed tree)
__global__ void __launch_bounds__(256) pupil_intensity_kernel(const double* __restrict__ U,
                                                              double scale, double* psf,
                                                              long long nx, long long ny,
                                                              double p0, double dp, double q0,
                                                              double dq, double* part) {
    __shared__ double red[5][256];
    const int k = blockIdx.y;
    const long long npix = nx * ny;
    const long long e0 = (long long)blockIdx.x * PUP_RED + threadIdx.x * (PUP_RED / 256);
    double sum = 0.0, mx = -1.0, at = -1.0, sp = 0.0, sq = 0.0;
    for (int i = 0; i < PUP_RED / 256; ++i) {
        const long long e = e0 + i;
        if (e >= npix) break;
        const long long f = (long long)k * npix + e;
        const double re = U[2 * f], im = U[2 * f + 1];
        const double v = __dadd_rn(psf[f], __dmul_rn(scale, __fma_rn(re, re, __dmul_rn(im, im))));
        psf[f] = v;
        const long long a = e / ny, b = e % ny;
        sum = __dadd_rn(sum, v);
        sp = __fma_rn(v, __dadd_rn(p0, __dmul_rn((double)a, dp)), sp);
        sq = __fma_rn(v, __dadd_rn(q0, __dmul_rn((double)b, dq)), sq);
        if (v > mx) {
            mx = v;
            at = (double)e;
        }
    }
    red[0][threadIdx.x] = sum;
    red[1][threadIdx.x] = mx;
    red[2][threadIdx.x] = at;
    red[3][threadIdx.x] = sp;
    red[4][threadIdx.x] = sq;
    __syncthreads();
    for (int h = 128; h > 0; h >>= 1) {
        if (threadIdx.x < h) {
            const int o = threadIdx.x + h;
            red[0][threadIdx.x] = __dadd_rn(red[0][threadIdx.x], red[0][o]);
            red[3][threadIdx.x] = __dadd_rn(red[3][threadIdx.x], red[3][o]);
            red[4][threadIdx.x] = __dadd_rn(red[4][threadIdx.x], red[4][o]);
            // the larger value wins, on a tie the smaller index: the first maximum
            if (red[1][o] > red[1][threadIdx.x] ||
                (red[1][o] == red[1][threadIdx.x] && red[2][o] < red[2][threadIdx.x])) {
                red[1][threadIdx.x] = red[1][o];
                red[2][threadIdx.x] = red[2][o];
            }
        }
        __syncthreads();
    }
    if (threadIdx.x < 5)
        part[((long long)k * gridDim.x + blockIdx.x) * 5 + threadIdx.x] = red[threadIdx.x][0];
}

}  // namespace rtx
