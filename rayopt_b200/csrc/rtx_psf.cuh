// rtx_psf.cuh -- device side of the diffraction PSF (sm_90a, FP64):
// GeometricTrace.psf (rayopt/geometric_trace.py:133-169) after the per-ray OPD.
//
//   regridding  griddata(method="linear") on a GIVEN Delaunay triangulation
//               (simplices, transform of scipy.spatial.Delaunay), evaluated by
//               rasterising the triangles: a claim pass (atomicMin of the
//               simplex index per grid node) and an evaluation pass, so that
//               the result does not depend on scheduling
//   pupil       exp(-2 pi i o)/sqrt(#finite) into the zero-padded complex grid
//   intensity   |fft|^2/(nx ny) and a deterministic reduction of sum, max and
//               the first moments over the frequency indices
//
// The barycentric coordinates and the interpolated value use the evaluation
// order of scipy's _qhull / interpnd (c_k accumulated from 0 in index order,
// c_2 = (1 - c_0) - c_1, value = ((0 + c_0 v_0) + c_1 v_1) + c_2 v_2) with
// unfused IEEE operations, so a node evaluated on the simplex scipy's
// find_simplex returns is bit-identical to griddata.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <climits>
#include <cfloat>

namespace rtx {

constexpr double GRID_EPS = 100.0 * DBL_EPSILON;  // scipy's inside tolerance
constexpr int GRID_WARP_NODES = 64;   // a simplex whose box has more nodes is rasterised by a warp
constexpr int PSF_RED_BLOCKS = 1024;  // fixed grid of the reduction: deterministic sums

struct Bary {
    double c0, c1, c2;
};

// scipy _barycentric_coordinates, ndim = 2; tr = {T00, T01, T10, T11, r0, r1}
__device__ __forceinline__ Bary barycentric(const double* __restrict__ tr, double x, double y) {
    const double dx = __dsub_rn(x, tr[4]), dy = __dsub_rn(y, tr[5]);
    Bary b;
    b.c0 = __dadd_rn(__dadd_rn(0.0, __dmul_rn(tr[0], dx)), __dmul_rn(tr[1], dy));
    b.c1 = __dadd_rn(__dadd_rn(0.0, __dmul_rn(tr[2], dx)), __dmul_rn(tr[3], dy));
    b.c2 = __dsub_rn(__dsub_rn(1.0, b.c0), b.c1);
    return b;
}

__device__ __forceinline__ bool inside(double c) {  // NaN (degenerate simplex): outside
    return c >= -GRID_EPS && c <= 1.0 + GRID_EPS;
}

__global__ void fill_i32_kernel(int* __restrict__ a, long long n, int v) {
    for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < n;
         k += (long long)gridDim.x * blockDim.x)
        a[k] = v;
}

// index range [lo, hi] of the grid nodes whose axis value lies in [vmin, vmax],
// widened by the nearest node beyond each end and clamped to the grid.  The
// axis gh is strictly monotone, ascending (s = 1) or descending (s = -1): in
// the key s gh[i] it is ascending, and the box is [a, b] = s [vmin, vmax]
// sorted.  The first node with key >= a is found by binary search, the last
// one <= b by walking on from it (boxes are a few nodes wide).  A node that
// passes scipy's 100-eps test lies within ~2 GRID_EPS (vmax - vmin) of the box
// plus the rounding of its coordinates, far less than one spacing, so the one
// node of margin covers every node a simplex can claim.
__device__ __forceinline__ void node_range(double vmin, double vmax, const double* __restrict__ gh,
                                           int n, double s, int& lo, int& hi) {
    const double a = s > 0.0 ? vmin : -vmax, b = s > 0.0 ? vmax : -vmin;
    int first = 0, len = n;  // first index with s gh[i] >= a, n if none
    while (len > 0) {
        const int half = len >> 1;
        if (s * gh[first + half] < a) {
            first += half + 1;
            len -= half + 1;
        } else {
            len = half;
        }
    }
    int last = first;  // first index with s gh[i] > b, n if none
    while (last < n && s * gh[last] <= b) ++last;
    lo = first > 0 ? first - 1 : 0;
    hi = last < n ? last : n - 1;
}

// claim pass: one lane per simplex; boxes of more than GRID_WARP_NODES nodes
// (hull slivers) are rasterised by the whole warp, one such simplex at a time
__global__ void __launch_bounds__(256) grid_claim_kernel(
    const double* __restrict__ pts, long long M, const int* __restrict__ simp,
    const double* __restrict__ transform, long long T, const double* __restrict__ gh, int n,
    int* __restrict__ winner) {
    const long long s = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    const double dir = gh[n - 1] < gh[0] ? -1.0 : 1.0;
    int i0 = 0, i1 = -1, j0 = 0, j1 = -1;
    const double* tr = transform + 6 * s;
    if (s < T && tr[0] == tr[0]) {  // NaN transform: degenerate, never a winner (as in scipy)
        const int a = simp[3 * s], b = simp[3 * s + 1], c = simp[3 * s + 2];
        if (a >= 0 && a < M && b >= 0 && b < M && c >= 0 && c < M) {
            const double xa = pts[2 * a], xb = pts[2 * b], xc = pts[2 * c];
            const double ya = pts[2 * a + 1], yb = pts[2 * b + 1], yc = pts[2 * c + 1];
            node_range(fmin(xa, fmin(xb, xc)), fmax(xa, fmax(xb, xc)), gh, n, dir, i0, i1);
            node_range(fmin(ya, fmin(yb, yc)), fmax(ya, fmax(yb, yc)), gh, n, dir, j0, j1);
        }
    }
    const int wi = i1 >= i0 ? i1 - i0 + 1 : 0, wj = j1 >= j0 ? j1 - j0 + 1 : 0;
    const int cnt = wi * wj;  // n <= 46340: no int overflow
    const bool big = cnt > GRID_WARP_NODES;
    if (!big) {
        for (int i = i0; i <= i1; ++i)
            for (int j = j0; j <= j1; ++j) {
                const Bary c = barycentric(tr, gh[i], gh[j]);
                if (inside(c.c0) && inside(c.c1) && inside(c.c2))
                    atomicMin(winner + (long long)i * n + j, (int)s);
            }
    }
    unsigned todo = __ballot_sync(0xffffffffu, big);
    while (todo) {
        const int src = __ffs(todo) - 1;
        todo &= todo - 1;
        const long long ss = __shfl_sync(0xffffffffu, s, src);
        const int bi = __shfl_sync(0xffffffffu, i0, src), bj = __shfl_sync(0xffffffffu, j0, src);
        const int bwj = __shfl_sync(0xffffffffu, wj, src);
        const int bcnt = __shfl_sync(0xffffffffu, cnt, src);
        const double* btr = transform + 6 * ss;
        for (int k = lane; k < bcnt; k += 32) {
            const int i = bi + k / bwj, j = bj + k % bwj;
            const Bary c = barycentric(btr, gh[i], gh[j]);
            if (inside(c.c0) && inside(c.c1) && inside(c.c2))
                atomicMin(winner + (long long)i * n + j, (int)ss);
        }
    }
}

// evaluation pass: the winning simplex's barycentric interpolation, NaN
// (griddata's fill_value) where no simplex claimed the node
__global__ void __launch_bounds__(256) grid_eval_kernel(
    const double* __restrict__ vals, const int* __restrict__ simp,
    const double* __restrict__ transform, const double* __restrict__ gh, int n,
    const int* __restrict__ winner, double* __restrict__ out) {
    const long long nn = (long long)n * n;
    for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < nn;
         k += (long long)gridDim.x * blockDim.x) {
        const int w = winner[k];
        double v = CUDART_NAN;
        if (w != INT_MAX) {
            const Bary c = barycentric(transform + 6 * (long long)w, gh[k / n], gh[k % n]);
            const int* sv = simp + 3 * (long long)w;
            v = __dadd_rn(0.0, __dmul_rn(c.c0, vals[sv[0]]));
            v = __dadd_rn(v, __dmul_rn(c.c1, vals[sv[1]]));
            v = __dadd_rn(v, __dmul_rn(c.c2, vals[sv[2]]));
        }
        out[k] = v;
    }
}

// number of finite nodes of the regridded OPD (integer atomics: deterministic)
__global__ void __launch_bounds__(256) count_finite_kernel(const double* __restrict__ o, long long nn,
                                                           unsigned long long* __restrict__ count) {
    unsigned long long c = 0;
    for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < nn;
         k += (long long)gridDim.x * blockDim.x)
        c += isfinite(o[k]) ? 1ull : 0ull;
    for (int off = 16; off; off >>= 1) c += __shfl_down_sync(0xffffffffu, c, off);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(count, c);
}

// the zero-padded pupil function: np.where(good, exp(-2j pi o), 0)/sqrt(count)
// in the top-left n x n corner of the (nx, ny) array (fft2(o, (nx, ny)) pads
// at the end); numpy's complex division by the real sqrt(count) multiplies by
// its reciprocal
__global__ void __launch_bounds__(256) pupil_kernel(const double* __restrict__ o, int n, long long nx,
                                                    long long ny,
                                                    const unsigned long long* __restrict__ count,
                                                    double2* __restrict__ out) {
    const double scl = __ddiv_rn(1.0, __dsqrt_rn((double)*count));
    const long long tot = nx * ny;
    for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < tot;
         k += (long long)gridDim.x * blockDim.x) {
        const long long I = k / ny, J = k % ny;
        double2 z = make_double2(0.0, 0.0);
        if (I < n && J < n) {
            const double v = o[I * n + J];
            double re = 0.0, im = 0.0;
            if (isfinite(v)) sincos(__dmul_rn(-6.283185307179586, v), &im, &re);
            z = make_double2(__dmul_rn(re, scl), __dmul_rn(im, scl));
        }
        out[k] = z;
    }
}

// signed frequency index of np.fft.fftfreq(m): 0 .. (m-1)/2, then -(m/2) .. -1
__device__ __forceinline__ double freq_index(long long i, long long m) {
    return (double)(i < (m - 1) / 2 + 1 ? i : i - m);
}

// psf = |z|^2/(nx ny) and per-block partials {sum, max, sum psf k_p, sum psf k_q}
// in a fixed order (grid of PSF_RED_BLOCKS blocks)
__global__ void __launch_bounds__(256) intensity_kernel(const double2* __restrict__ z, long long nx,
                                                        long long ny, double* __restrict__ psf,
                                                        double* __restrict__ part) {
    const long long tot = nx * ny;
    const double size = (double)tot;
    double s = 0.0, mx = -CUDART_INF, sp = 0.0, sq = 0.0;
    for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < tot;
         k += (long long)gridDim.x * blockDim.x) {
        const double2 a = z[k];
        const double v = __ddiv_rn(__dadd_rn(__dmul_rn(a.x, a.x), __dmul_rn(a.y, a.y)), size);
        psf[k] = v;
        s += v;
        mx = fmax(mx, v);
        sp += v * freq_index(k / ny, nx);
        sq += v * freq_index(k % ny, ny);
    }
    for (int off = 16; off; off >>= 1) {
        s += __shfl_down_sync(0xffffffffu, s, off);
        mx = fmax(mx, __shfl_down_sync(0xffffffffu, mx, off));
        sp += __shfl_down_sync(0xffffffffu, sp, off);
        sq += __shfl_down_sync(0xffffffffu, sq, off);
    }
    __shared__ double sh[4][8];
    const int w = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0) {
        sh[0][w] = s;
        sh[1][w] = mx;
        sh[2][w] = sp;
        sh[3][w] = sq;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        double r[4] = {0.0, -CUDART_INF, 0.0, 0.0};
        for (int k = 0; k < (int)(blockDim.x >> 5); ++k) {
            r[0] += sh[0][k];
            r[1] = fmax(r[1], sh[1][k]);
            r[2] += sh[2][k];
            r[3] += sh[3][k];
        }
        for (int q = 0; q < 4; ++q) part[4 * blockIdx.x + q] = r[q];
    }
}

// stats = {#finite, sum, max, sum psf k_p, sum psf k_q} from the partials, one
// thread in block order
__global__ void psf_stats_kernel(const double* __restrict__ part, int nblocks,
                                 const unsigned long long* __restrict__ count,
                                 double* __restrict__ stats) {
    double r[4] = {0.0, -CUDART_INF, 0.0, 0.0};
    for (int b = 0; b < nblocks; ++b) {
        r[0] += part[4 * b];
        r[1] = fmax(r[1], part[4 * b + 1]);
        r[2] += part[4 * b + 2];
        r[3] += part[4 * b + 3];
    }
    stats[0] = (double)*count;
    for (int q = 0; q < 4; ++q) stats[1 + q] = r[q];
}

// ---- radial and line sums of a PSF (Analysis.opds, rayopt/analysis.py:330-346)
//
// The PSF is read in its stored FFT order; (I, J) are the indices of the
// fftshifted image, stored at ((I - nx/2) mod nx, (J - ny/2) mod ny).  Bin of
// (I, J) about the centre (c0, c1): trunc(sqrt((J - c1)^2 + (I - c0)^2)) with
// numpy's separately rounded operations (polar_sum, aspect 1, binsize 1).
//
// Deterministic without float atomics: PROF_BLOCKS blocks (a constant, not the
// SM count) each take a fixed contiguous range of 64 x 64 tiles of the shifted
// image and accumulate into block-private rows of partial sums (bins, row sums,
// column sums) in tile order; profile_combine_kernel then sums the rows in
// block order.  Inside a tile each warp owns 4 rows: along a row the bin is
// monotone on each side of the centre column, so equal (bin, side) keys are
// contiguous lanes and a segmented scan sums them in a fixed order; the
// segment tails add into the warp's shared histogram (side j < 0 first), and
// the 16 warp histograms are summed in warp order at the end of the tile.
constexpr int PROF_TILE = 64;
constexpr int PROF_WARPS = 16;                     // 512 threads, 4 rows each
constexpr int PROF_ROWS = PROF_TILE / PROF_WARPS;
constexpr int PROF_TILE_BINS = 96;                 // a 64 x 64 tile spans <= 91 bins
constexpr int PROF_BLOCKS = 132;

__host__ __device__ __forceinline__ long long profile_bin(double I, double J, double c0, double c1) {
#ifdef __CUDA_ARCH__
    const double i = __dsub_rn(I, c0), j = __dsub_rn(J, c1);
    return (long long)__dsqrt_rn(__dadd_rn(__dmul_rn(j, j), __dmul_rn(i, i)));
#else
    volatile double i = I - c0, j = J - c1;  // volatile: no contraction on the host
    volatile double jj = j * j, ii = i * i;
    volatile double s = jj + ii;
    return (long long)sqrt((double)s);
#endif
}

// stored index of the shifted index k along an axis of m
__device__ __forceinline__ long long unshift(long long k, long long m) {
    const long long s = k - m / 2;
    return s < 0 ? s + m : s;
}

// partial rows: block g owns part[g*stride, (g+1)*stride) = [bins | row sums (nx) |
// column sums (ny)], the rows and columns in stored order.  flag bit 0: a
// negative or non-finite pixel; bit 1: a tile spanned more than PROF_TILE_BINS
// bins (cannot happen for in-range centres; reported rather than dropped)
__global__ void __launch_bounds__(PROF_WARPS * 32) profile_tiles_kernel(
    const double* __restrict__ psf, long long nx, long long ny, double c0, double c1,
    long long nbins, double* __restrict__ part, long long stride, int* __restrict__ flag) {
    __shared__ double hist[PROF_WARPS][PROF_TILE_BINS];
    __shared__ double cols[PROF_WARPS][PROF_TILE];
    __shared__ long long s_b0;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    double* mine = part + (long long)blockIdx.x * stride;
    double* rows = mine + nbins;
    double* colsum = rows + nx;
    for (long long k = threadIdx.x; k < stride; k += blockDim.x) mine[k] = 0.0;
    for (int k = threadIdx.x; k < PROF_WARPS * PROF_TILE_BINS; k += blockDim.x)
        (&hist[0][0])[k] = 0.0;
    const long long ntr = (nx + PROF_TILE - 1) / PROF_TILE, ntc = (ny + PROF_TILE - 1) / PROF_TILE;
    const long long T = ntr * ntc;
    const long long t0 = T * blockIdx.x / gridDim.x, t1 = T * (blockIdx.x + 1) / gridDim.x;
    int bad = 0;
    for (long long t = t0; t < t1; ++t) {
        const long long I0 = (t / ntc) * PROF_TILE, J0 = (t % ntc) * PROF_TILE;
        const long long I1 = min(I0 + PROF_TILE, nx) - 1, J1 = min(J0 + PROF_TILE, ny) - 1;
        if (threadIdx.x == 0) {
            // the lowest bin of the tile: the radius is monotone in |I - c0| and
            // |J - c1|, whose minima over the tile's integers are at a clamped
            // floor or ceil of the centre
            long long b0 = LLONG_MAX;
            const double fi = floor(c0), fj = floor(c1);
            for (int a = 0; a < 2; ++a)
                for (int b = 0; b < 2; ++b) {
                    const double I = fmin(fmax(fi + a, (double)I0), (double)I1);
                    const double J = fmin(fmax(fj + b, (double)J0), (double)J1);
                    b0 = min(b0, profile_bin(I, J, c0, c1));
                }
            s_b0 = b0;
        }
        __syncthreads();
        const long long b0 = s_b0;
        // loads first: 8 pixels per lane in flight
        double v[PROF_ROWS][2];
        bool ok[PROF_ROWS][2];
#pragma unroll
        for (int r = 0; r < PROF_ROWS; ++r) {
            const long long I = I0 + w * PROF_ROWS + r;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const long long J = J0 + 32 * h + lane;
                ok[r][h] = I <= I1 && J <= J1;
                v[r][h] = ok[r][h] ? __ldcs(psf + unshift(I, nx) * ny + unshift(J, ny)) : 0.0;
            }
        }
        double csum[2] = {0.0, 0.0};
#pragma unroll
        for (int r = 0; r < PROF_ROWS; ++r) {
            const long long I = I0 + w * PROF_ROWS + r;
            double rsum = 0.0;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const double x = v[r][h];
                const long long J = J0 + 32 * h + lane;
                if (ok[r][h] && !(x >= 0.0 && x <= DBL_MAX)) bad |= 1;
                csum[h] = __dadd_rn(csum[h], x);
                rsum = __dadd_rn(rsum, x);
                long long key = -1;  // 2 bin + (j >= 0); -1 outside the array
                if (ok[r][h]) {
                    const long long b = profile_bin((double)I, (double)J, c0, c1) - b0;
                    if (b < 0 || b >= PROF_TILE_BINS) bad |= 2;
                    else key = 2 * b + (__dsub_rn((double)J, c1) >= 0.0 ? 1 : 0);
                }
                // segmented inclusive scan over runs of equal keys
                const long long prev = __shfl_up_sync(0xffffffffu, key, 1);
                const unsigned heads = __ballot_sync(0xffffffffu, lane == 0 || prev != key);
                const int start = 31 - __clz(heads & (0xffffffffu >> (31 - lane)));
                double s = x;
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) {
                    const double u = __shfl_up_sync(0xffffffffu, s, d);
                    if (lane - d >= start) s = __dadd_rn(s, u);
                }
                const bool tail = lane == 31 || ((heads >> (lane + 1)) & 1u);
                if (tail && key >= 0 && (key & 1) == 0) hist[w][key >> 1] += s;
                __syncwarp();
                if (tail && key >= 0 && (key & 1) == 1) hist[w][key >> 1] += s;
                __syncwarp();
            }
            for (int off = 16; off; off >>= 1) rsum = __dadd_rn(rsum, __shfl_xor_sync(0xffffffffu, rsum, off));
            if (lane == 0 && I <= I1) rows[unshift(I, nx)] += rsum;
        }
        cols[w][lane] = csum[0];
        cols[w][lane + 32] = csum[1];
        __syncthreads();
        const int k = threadIdx.x;
        if (k < PROF_TILE) {
            if (J0 + k <= J1) {
                double s = 0.0;
                for (int q = 0; q < PROF_WARPS; ++q) s = __dadd_rn(s, cols[q][k]);
                colsum[unshift(J0 + k, ny)] += s;
            }
        } else if (k < PROF_TILE + PROF_TILE_BINS) {
            const int b = k - PROF_TILE;
            double s = 0.0;
            for (int q = 0; q < PROF_WARPS; ++q) {
                s = __dadd_rn(s, hist[q][b]);
                hist[q][b] = 0.0;
            }
            if (b0 + b < nbins) mine[b0 + b] += s;
        }
        __syncthreads();
    }
    bad = __reduce_or_sync(0xffffffffu, bad);
    if (lane == 0 && bad) atomicOr(flag, bad);
}

// out[k] = sum over the blocks' partial rows, in block order
__global__ void __launch_bounds__(256) profile_combine_kernel(const double* __restrict__ part, int nblocks,
                                                              long long stride, double* __restrict__ out) {
    for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < stride;
         k += (long long)gridDim.x * blockDim.x) {
        double s = 0.0;
        for (int g = 0; g < nblocks; ++g) s = __dadd_rn(s, part[g * stride + k]);
        out[k] = s;
    }
}

// ---- exit-pupil points of the per-ray OPD (rtx_opd_points) ----------------
//
// Ray j's point and OPD relative to the reference ray, with numpy's separately
// rounded operations (ResidentMixin.opd_rays): t = -(A[j] - A[ref])/k and
// (x, y) = P[j].xy - P[ref].xy; the ray is kept when x, y and t are finite.
// The kept rays are written in increasing j at the ranks an exclusive prefix
// sum of the keep flags gives (dt::scan_*_kernel), so the compacted arrays are
// those of numpy's boolean mask.
struct OpdPoint {
    double x, y, t;
    bool keep;
};

__device__ __forceinline__ OpdPoint opd_point(const double* __restrict__ A, const double* __restrict__ P,
                                              long long j, long long ref, double k) {
    OpdPoint q;
    q.t = __ddiv_rn(-__dsub_rn(A[j], A[ref]), k);
    q.x = __dsub_rn(P[3 * j], P[3 * ref]);
    q.y = __dsub_rn(P[3 * j + 1], P[3 * ref + 1]);
    q.keep = isfinite(q.x) && isfinite(q.y) && isfinite(q.t);
    return q;
}

__global__ void __launch_bounds__(256) opd_flag_kernel(const double* __restrict__ A,
                                                       const double* __restrict__ P, long long N,
                                                       long long ref, double k, int* __restrict__ flag) {
    for (long long j = blockIdx.x * (long long)blockDim.x + threadIdx.x; j < N;
         j += (long long)gridDim.x * blockDim.x)
        flag[j] = opd_point(A, P, j, ref, k).keep ? 1 : 0;
}

// the kept rays to their ranks; hbits receives max(|x|, |y|) of them as the
// bits of a non-negative double, whose integer order is the numeric order
__global__ void __launch_bounds__(256) opd_scatter_kernel(
    const double* __restrict__ A, const double* __restrict__ P, long long N, long long ref, double k,
    const int* __restrict__ rank, double* __restrict__ pts, double* __restrict__ vals,
    unsigned long long* __restrict__ hbits) {
    unsigned long long m = 0;
    for (long long j = blockIdx.x * (long long)blockDim.x + threadIdx.x; j < N;
         j += (long long)gridDim.x * blockDim.x) {
        const OpdPoint q = opd_point(A, P, j, ref, k);
        if (!q.keep) continue;
        const long long r = rank[j];
        pts[2 * r] = q.x;
        pts[2 * r + 1] = q.y;
        vals[r] = q.t;
        const unsigned long long bx = (unsigned long long)__double_as_longlong(fabs(q.x));
        const unsigned long long by = (unsigned long long)__double_as_longlong(fabs(q.y));
        m = max(m, max(bx, by));
    }
    for (int off = 16; off; off >>= 1) m = max(m, __shfl_down_sync(0xffffffffu, m, off));
    if ((threadIdx.x & 31) == 0 && m) atomicMax(hbits, m);
}

// ---- finite count, min and max of a grid (rtx_grid_range) ------------------
//
// Integer atomics on order keys (the sign bit flipped for non-negative values,
// every bit for negative ones): the unsigned order of the keys is the numeric
// order with -0 < +0, so the result is exact and independent of the schedule.
// acc = {count, min key, max key}, initialised to {0, ~0, 0}.
__device__ __forceinline__ unsigned long long order_key(double v) {
    const unsigned long long b = (unsigned long long)__double_as_longlong(v);
    return (b >> 63) ? ~b : b | 0x8000000000000000ull;
}

__global__ void __launch_bounds__(256) grid_range_kernel(const double* __restrict__ o, long long n,
                                                         unsigned long long* __restrict__ acc) {
    unsigned long long c = 0, lo = ~0ull, hi = 0;
    for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < n;
         k += (long long)gridDim.x * blockDim.x) {
        const double v = o[k];
        if (!isfinite(v)) continue;
        const unsigned long long key = order_key(v);
        ++c;
        lo = min(lo, key);
        hi = max(hi, key);
    }
    for (int off = 16; off; off >>= 1) {
        c += __shfl_down_sync(0xffffffffu, c, off);
        lo = min(lo, __shfl_down_sync(0xffffffffu, lo, off));
        hi = max(hi, __shfl_down_sync(0xffffffffu, hi, off));
    }
    if ((threadIdx.x & 31) == 0 && c) {
        atomicAdd(acc, c);
        atomicMin(acc + 1, lo);
        atomicMax(acc + 2, hi);
    }
}

}  // namespace rtx
