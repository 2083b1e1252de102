// rtx_delaunay.cuh -- Delaunay triangulation of 2-d points on the device
// (sm_90a, FP64): what scipy.spatial.Delaunay gives rtx_grid_linear
// (simplices, neighbors, transform), without the host.
//
// Predicates.  orient2d and incircle are exact for every input in the domain
// (each coordinate 0 or 2^-200 <= |x| <= 2^200): a floating-point filter with
// Shewchuk's static error bounds ("Adaptive precision floating-point
// arithmetic and fast robust geometric predicates", 1997), computed with
// separately rounded operations, then an exact evaluation as an expansion
// (two-sum, two-product by fma) of the determinant's monomials in the raw
// coordinates.  In the domain every monomial (degree <= 4) and every
// component of its expansion is a multiple of 2^-1008 below 2^806, so no
// product underflows or overflows and the sign is exact.
//
// Triangulation.  Parallel incremental insertion with Lawson flips over
// triangle slots; vertex k of slot t is opposite its edge k = (v[k+1], v[k+2])
// and the neighbour across that edge is tn[3t+k].  A symbolic infinite vertex
// (INF) closes the hull: a ghost slot (y, x, INF) lies on hull edge x -> y and
// contains the points strictly outside it.  Every round
//   pick      each slot takes one uninserted point located in it: the one
//             nearest its circumcentre (ghosts: the farthest from the edge),
//             ties to the lowest index, by a 64-bit atomicMin;
//   split     1 -> 3, or 2 -> 4 with the neighbour for a point exactly on an
//             edge; a split that touches a slot claimed with a lower priority
//             (1 -> 3 before 2 -> 4, then slot order) waits a round; new slots
//             are numbered by a prefix sum in slot order;
//   flip      passes of Lawson flips until none remains: a dirty slot flags
//             its edges whose opposite vertex lies strictly inside its
//             circumcircle (exact incircle; a ghost's "circle" is the open
//             half plane outside its edge, so an infinite edge flips only at a
//             strictly reflex hull vertex and a hull edge never flips), and
//             every flagged edge votes for both its slots with the key
//             (min slot, max slot); an edge flips when it holds both votes;
//   fix       after every split or flip step, slots that were rewritten patch
//             the neighbour pointers across their edges;
//   relocate  uninserted points walk (visibility walk, first edge in index
//             order) from the slot they were in to the slot containing them;
//             a point on an interior edge takes the lower of its two slots, a
//             point outside the hull the last ghost of its visible chain, so
//             equal points always meet in one slot.  A point equal to a
//             vertex is a duplicate and never inserted.
// Nothing depends on scheduling: no floating-point atomics, every choice is a
// minimum of integer keys, and slots are numbered by prefix sums.  The step
// bodies are __host__ __device__: tests/delaunay_host.cu runs them sequentially
// on the CPU.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <cfloat>

#ifndef __CUDACC__  // a plain host compiler
#define __noinline__ __attribute__((noinline))
#endif

#ifdef __CUDA_ARCH__
#define DT_ADD(a, b) __dadd_rn(a, b)
#define DT_SUB(a, b) __dsub_rn(a, b)
#define DT_MUL(a, b) __dmul_rn(a, b)
#define DT_DIV(a, b) __ddiv_rn(a, b)
#define DT_FMA(a, b, c) __fma_rn(a, b, c)
#else
#include <cmath>
#include <cstring>
#define DT_ADD(a, b) ((a) + (b))
#define DT_SUB(a, b) ((a) - (b))
#define DT_MUL(a, b) ((a) * (b))
#define DT_DIV(a, b) ((a) / (b))
#define DT_FMA(a, b, c) std::fma(a, b, c)
#endif

namespace rtx {
namespace dt {

constexpr int INF = -1;                 // the infinite vertex
constexpr double EPS = 0x1p-53;
constexpr double CCW_BOUND = (3.0 + 16.0 * EPS) * EPS;
constexpr double ICC_BOUND = (10.0 + 96.0 * EPS) * EPS;
constexpr double ABS_SLACK = 0x1p-1000;  // covers gradual underflow of the filter's products
constexpr double DOMAIN_MAX = 0x1p200, DOMAIN_MIN = 0x1p-200;
constexpr int ICC_TERMS = 48 * 8;        // monomials of the 4x4 determinant x their expansion

__host__ __device__ __forceinline__ bool in_domain(double x) {
    const double a = fabs(x);
    return x == 0.0 || (a >= DOMAIN_MIN && a <= DOMAIN_MAX);
}

__host__ __device__ __forceinline__ void two_sum(double a, double b, double& s, double& e) {
    s = DT_ADD(a, b);
    const double bv = DT_SUB(s, a);
    const double av = DT_SUB(s, bv);
    e = DT_ADD(DT_SUB(a, av), DT_SUB(b, bv));
}

__host__ __device__ __forceinline__ void two_prod(double a, double b, double& p, double& e) {
    p = DT_MUL(a, b);
    e = DT_FMA(a, b, -p);
}

// h <- h + b exactly: GROW-EXPANSION with zero elimination, in place; h is
// non-overlapping in increasing magnitude; returns the new length
__host__ __device__ __forceinline__ int grow(double* h, int n, double b) {
    double q = b;
    int k = 0;
    for (int i = 0; i < n; ++i) {
        double s, e;
        two_sum(q, h[i], s, e);
        q = s;
        if (e != 0.0) h[k++] = e;
    }
    if (q != 0.0 || k == 0) h[k++] = q;
    return k;
}

__host__ __device__ __forceinline__ int sgn(double x) { return (x > 0.0) - (x < 0.0); }

// sign of det [[ax ay 1] [bx by 1] [cx cy 1]] from its six exact monomials
__host__ __device__ __noinline__ int orient_exact(double ax, double ay, double bx, double by,
                                                  double cx, double cy) {
    const double X[3] = {ax, bx, cx}, Y[3] = {ay, by, cy};
    const int I[6] = {0, 0, 1, 1, 2, 2}, J[6] = {1, 2, 0, 2, 0, 1};
    const double S[6] = {1.0, -1.0, -1.0, 1.0, 1.0, -1.0};
    double h[13];
    int n = 0;
    for (int m = 0; m < 6; ++m) {
        double p, e;
        two_prod(S[m] * X[I[m]], Y[J[m]], p, e);
        n = grow(h, n, p);
        n = grow(h, n, e);
    }
    return sgn(h[n - 1]);
}

// > 0: c lies left of a -> b (a, b, c counter-clockwise)
__host__ __device__ __forceinline__ int orient2d(double2 a, double2 b, double2 c) {
    const double l = DT_MUL(DT_SUB(a.x, c.x), DT_SUB(b.y, c.y));
    const double r = DT_MUL(DT_SUB(a.y, c.y), DT_SUB(b.x, c.x));
    const double det = DT_SUB(l, r);
    const double bound = DT_ADD(DT_MUL(CCW_BOUND, DT_ADD(fabs(l), fabs(r))), ABS_SLACK);
    if (det > bound) return 1;
    if (-det > bound) return -1;
    return orient_exact(a.x, a.y, b.x, b.y, c.x, c.y);
}

// sign of det [[x y x^2+y^2 1]] over the rows a, b, c, d: expansion along the
// column of ones into 4 minors of 6 terms x_i y_j l_k, l_k = x_k^2 + y_k^2
__host__ __device__ __noinline__ int incircle_exact(double2 a, double2 b, double2 c, double2 d) {
    const double2 P[4] = {a, b, c, d};
    const int PI[6] = {0, 0, 1, 1, 2, 2}, PJ[6] = {1, 2, 0, 2, 0, 1}, PK[6] = {2, 1, 2, 0, 1, 0};
    const double PS[6] = {1.0, -1.0, -1.0, 1.0, 1.0, -1.0};
    double h[ICC_TERMS + 1];
    int n = 0;
    for (int r = 0; r < 4; ++r) {
        int rows[3], k = 0;
        for (int q = 0; q < 4; ++q)
            if (q != r) rows[k++] = q;
        const double sr = (r % 2 == 0) ? -1.0 : 1.0;
        for (int m = 0; m < 6; ++m) {
            const double2 pi = P[rows[PI[m]]], pj = P[rows[PJ[m]]], pk = P[rows[PK[m]]];
            for (int sq = 0; sq < 2; ++sq) {
                const double z = sq ? pk.y : pk.x;
                double t2[2], t4[4], t8[8];
                two_prod(sr * PS[m] * pi.x, pj.y, t2[1], t2[0]);
                for (int u = 0; u < 2; ++u) two_prod(t2[u], z, t4[2 * u + 1], t4[2 * u]);
                for (int u = 0; u < 4; ++u) two_prod(t4[u], z, t8[2 * u + 1], t8[2 * u]);
                for (int u = 0; u < 8; ++u) n = grow(h, n, t8[u]);
            }
        }
    }
    return sgn(h[n - 1]);
}

// > 0: d lies inside the circle through the counter-clockwise a, b, c
__host__ __device__ __forceinline__ int incircle(double2 a, double2 b, double2 c, double2 d) {
    const double adx = DT_SUB(a.x, d.x), bdx = DT_SUB(b.x, d.x), cdx = DT_SUB(c.x, d.x);
    const double ady = DT_SUB(a.y, d.y), bdy = DT_SUB(b.y, d.y), cdy = DT_SUB(c.y, d.y);
    const double bdxcdy = DT_MUL(bdx, cdy), cdxbdy = DT_MUL(cdx, bdy);
    const double cdxady = DT_MUL(cdx, ady), adxcdy = DT_MUL(adx, cdy);
    const double adxbdy = DT_MUL(adx, bdy), bdxady = DT_MUL(bdx, ady);
    const double alift = DT_ADD(DT_MUL(adx, adx), DT_MUL(ady, ady));
    const double blift = DT_ADD(DT_MUL(bdx, bdx), DT_MUL(bdy, bdy));
    const double clift = DT_ADD(DT_MUL(cdx, cdx), DT_MUL(cdy, cdy));
    const double det = DT_ADD(DT_ADD(DT_MUL(alift, DT_SUB(bdxcdy, cdxbdy)),
                                     DT_MUL(blift, DT_SUB(cdxady, adxcdy))),
                              DT_MUL(clift, DT_SUB(adxbdy, bdxady)));
    const double perm = DT_ADD(DT_ADD(DT_MUL(DT_ADD(fabs(bdxcdy), fabs(cdxbdy)), alift),
                                      DT_MUL(DT_ADD(fabs(cdxady), fabs(adxcdy)), blift)),
                               DT_MUL(DT_ADD(fabs(adxbdy), fabs(bdxady)), clift));
    const double bound = DT_ADD(DT_MUL(ICC_BOUND, perm), ABS_SLACK);
    if (det > bound) return 1;
    if (-det > bound) return -1;
    return incircle_exact(a, b, c, d);
}

// ---- atomics (sequential on the host) ---------------------------------------
#ifdef __CUDA_ARCH__
__device__ __forceinline__ void amin64(unsigned long long* p, unsigned long long v) { atomicMin(p, v); }
__device__ __forceinline__ void aadd32(unsigned* p, unsigned v) { atomicAdd(p, v); }
__device__ __forceinline__ void aor32(unsigned* p, unsigned v) { atomicOr(p, v); }
#else
inline void amin64(unsigned long long* p, unsigned long long v) { if (v < *p) *p = v; }
inline void aadd32(unsigned* p, unsigned v) { *p += v; }
inline void aor32(unsigned* p, unsigned v) { *p |= v; }
#endif

constexpr unsigned long long NONE = ~0ull;
// counters: flips of a pass, uninserted points, error bits
enum { C_FLIPS = 0, C_LEFT = 1, C_ERR = 2, C_N = 4 };
enum { ERR_INPUT = 1, ERR_WALK = 2, ERR_LINK = 4 };
constexpr int LEX_BLOCKS = 256, LEX_THREADS = 256;

struct Work {
    const double2* p;  // points
    long long M;
    int* tv;           // 3 vertices per slot, counter-clockwise
    int* tn;           // 3 neighbours per slot, tn[3t+k] across edge k
    int* mod;          // stamp of the step that last rewrote the slot
    int* chk;          // stamp of the flip pass that checks the slot
    int2* ext;         // the other slots that replaced this one in its last step
    unsigned long long* pick;  // per slot: (distance key, point)
    unsigned long long* vote;  // per slot: claim of a split / vote of a flip
    int* op;           // split of the slot (-1, 3 = 1->3, k = 2->4 on edge k); flagged edges in flip passes
    int* flag;         // prefix-sum input
    int* rank;         // prefix-sum output
    int* bsum;         // prefix-sum block totals, then the total
    int* loc;          // per point: its slot; -1 vertex, -2 duplicate
    unsigned* cnt;     // C_N counters
    long long* lex;    // LEX_BLOCKS x 2 partial lexicographic min / max indices, then the two seeds
    unsigned long long* seed_key;  // third seed: (-|area| key, index)
};

__host__ __device__ __forceinline__ int nxt(int k) { return k == 2 ? 0 : k + 1; }
__host__ __device__ __forceinline__ int prv(int k) { return k == 0 ? 2 : k - 1; }

// order-preserving map of a float to 32 bits
__host__ __device__ __forceinline__ unsigned sortable(float f) {
#ifdef __CUDA_ARCH__
    const unsigned u = __float_as_uint(f);
#else
    unsigned u;
    std::memcpy(&u, &f, 4);
#endif
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__host__ __device__ __forceinline__ float clampf(double x) {
    if (!(x <= (double)FLT_MAX)) return FLT_MAX;  // +inf, NaN
    if (!(x >= -(double)FLT_MAX)) return -FLT_MAX;
    return (float)x;
}

__host__ __device__ __forceinline__ int ghost_pos(const int* v) {
    return v[0] == INF ? 0 : (v[1] == INF ? 1 : (v[2] == INF ? 2 : -1));
}

// does (a, ia) come before (b, ib) as the lexicographic minimum (first) or
// maximum (!first) of the coordinates?  Equal points: the lower index, so a
// seed is always the lowest-index copy of its point; -0.0 equals +0.0
__host__ __device__ __forceinline__ bool lex_before(bool first, double2 a, long long ia, double2 b,
                                                    long long ib) {
    if (a.x != b.x) return first ? a.x < b.x : a.x > b.x;
    if (a.y != b.y) return first ? a.y < b.y : a.y > b.y;
    return ia < ib;
}

// ---- set-up: validation, the three seed points, the first four slots -------
// partial lexicographic min and max per block of LEX_THREADS into s[2 thread],
// s[2 thread + 1], and the domain check
__host__ __device__ __forceinline__ void lex_body(const Work& w, int block, int thread, long long* s) {
    long long lo = -1, hi = -1;
    unsigned bad = 0;
    for (long long i = (long long)block * LEX_THREADS + thread; i < w.M;
         i += (long long)LEX_BLOCKS * LEX_THREADS) {
        const double2 q = w.p[i];
        if (!(in_domain(q.x) && in_domain(q.y))) bad = 1;  // NaN fails in_domain
        if (lo < 0 || lex_before(true, q, i, w.p[lo], lo)) lo = i;
        if (hi < 0 || lex_before(false, q, i, w.p[hi], hi)) hi = i;
    }
    if (bad) aor32(w.cnt + C_ERR, ERR_INPUT);
    s[2 * thread] = lo;
    s[2 * thread + 1] = hi;
}

// min of in[2k] and max of in[2k + 1] over k < n (entries < 0 are empty)
__host__ __device__ __forceinline__ void lex_reduce(const Work& w, const long long* in, int n, long long* lo,
                                                    long long* hi) {
    long long a = -1, b = -1;
    for (int k = 0; k < n; ++k) {
        const long long l = in[2 * k], h = in[2 * k + 1];
        if (l >= 0 && (a < 0 || lex_before(true, w.p[l], l, w.p[a], a))) a = l;
        if (h >= 0 && (b < 0 || lex_before(false, w.p[h], h, w.p[b], b))) b = h;
    }
    *lo = a;
    *hi = b;
}

// third seed: the point farthest from the line of the first two among those
// exactly off it (lowest index on ties)
__host__ __device__ __forceinline__ void seed_body(const Work& w, long long i) {
    const double2 a = w.p[w.lex[2 * LEX_BLOCKS]], b = w.p[w.lex[2 * LEX_BLOCKS + 1]], q = w.p[i];
    if (orient2d(a, b, q) == 0) return;
    const double ar = DT_SUB(DT_MUL(DT_SUB(b.x, a.x), DT_SUB(q.y, a.y)),
                             DT_MUL(DT_SUB(b.y, a.y), DT_SUB(q.x, a.x)));
    amin64(w.seed_key, ((unsigned long long)sortable(-clampf(fabs(ar))) << 32) | (unsigned long long)i);
}

// the seed triangle, counter-clockwise, in slot 0 and its three ghosts in 1..3
__host__ __device__ __forceinline__ void init_body(const Work& w) {
    int s[3] = {(int)w.lex[2 * LEX_BLOCKS], (int)w.lex[2 * LEX_BLOCKS + 1],
                (int)(*w.seed_key & 0xffffffffu)};
    if (orient2d(w.p[s[0]], w.p[s[1]], w.p[s[2]]) < 0) {
        const int t = s[1];
        s[1] = s[2];
        s[2] = t;
    }
    for (int k = 0; k < 3; ++k) {
        w.tv[k] = s[k];
        w.tn[k] = 1 + k;
        // ghost 1+k on edge k = (s[k+1], s[k+2]): (s[k+2], s[k+1], INF); across
        // its edge 0 = (s[k+1], INF) lies ghost 1+(k+2), across edge 1 ghost 1+(k+1)
        int* g = w.tv + 3 * (1 + k);
        g[0] = s[prv(k)];
        g[1] = s[nxt(k)];
        g[2] = INF;
        int* gn = w.tn + 3 * (1 + k);
        gn[0] = 1 + prv(k);
        gn[1] = 1 + nxt(k);
        gn[2] = 0;
    }
    for (int t = 0; t < 4; ++t) {
        w.mod[t] = 0;
        w.chk[t] = 0;
        w.ext[t] = make_int2(-1, -1);
    }
    for (int k = 0; k < 3; ++k) w.loc[s[k]] = -1;
}

// ---- one round -----------------------------------------------------------
__host__ __device__ __forceinline__ void pick_body(const Work& w, long long i) {
    const int t = w.loc[i];
    if (t < 0) return;
    const int* v = w.tv + 3 * t;
    const double2 q = w.p[i];
    const int g = ghost_pos(v);
    double key;
    if (g >= 0) {
        const double2 a = w.p[v[nxt(g)]], b = w.p[v[prv(g)]];
        key = -fabs(DT_SUB(DT_MUL(DT_SUB(b.x, a.x), DT_SUB(q.y, a.y)),
                           DT_MUL(DT_SUB(b.y, a.y), DT_SUB(q.x, a.x))));
    } else {
        const double2 a = w.p[v[0]], b = w.p[v[1]], c = w.p[v[2]];
        const double bx = DT_SUB(b.x, a.x), by = DT_SUB(b.y, a.y);
        const double cx = DT_SUB(c.x, a.x), cy = DT_SUB(c.y, a.y);
        const double b2 = DT_ADD(DT_MUL(bx, bx), DT_MUL(by, by)), c2 = DT_ADD(DT_MUL(cx, cx), DT_MUL(cy, cy));
        const double d = DT_MUL(2.0, DT_SUB(DT_MUL(bx, cy), DT_MUL(by, cx)));
        const double ux = DT_DIV(DT_SUB(DT_MUL(cy, b2), DT_MUL(by, c2)), d);
        const double uy = DT_DIV(DT_SUB(DT_MUL(bx, c2), DT_MUL(cx, b2)), d);
        const double dx = DT_SUB(DT_SUB(q.x, a.x), ux), dy = DT_SUB(DT_SUB(q.y, a.y), uy);
        key = DT_ADD(DT_MUL(dx, dx), DT_MUL(dy, dy));
    }
    amin64(w.pick + t, ((unsigned long long)sortable(clampf(key)) << 32) | (unsigned long long)i);
}

__host__ __device__ __forceinline__ unsigned long long split_prio(int t, int op) {
    return (op == 3 ? 0ull : (1ull << 32)) | (unsigned long long)t;
}

// the split a picking slot makes, and its claims
__host__ __device__ __forceinline__ void claim_body(const Work& w, int t) {
    const unsigned long long pk = w.pick[t];
    int op = -1;
    if (pk != NONE) {
        const int* v = w.tv + 3 * t;
        op = 3;
        if (ghost_pos(v) < 0) {
            const double2 q = w.p[pk & 0xffffffffu];
            for (int e = 0; e < 3; ++e)
                if (orient2d(w.p[v[nxt(e)]], w.p[v[prv(e)]], q) == 0) op = e;
        }
        const unsigned long long pr = split_prio(t, op);
        amin64(w.vote + t, pr);
        if (op < 3) amin64(w.vote + w.tn[3 * t + op], pr);
    }
    w.op[t] = op;
}

__host__ __device__ __forceinline__ void decide_body(const Work& w, int t) {
    const int op = w.op[t];
    int go = 0;
    if (op >= 0) {
        const unsigned long long pr = split_prio(t, op);
        go = w.vote[t] == pr && (op == 3 || w.vote[w.tn[3 * t + op]] == pr);
    }
    w.flag[t] = go;
}

__host__ __device__ __forceinline__ void put(const Work& w, int s, const int* v, const int* n, int m, int chk,
                                             int2 ext) {
    for (int k = 0; k < 3; ++k) {
        w.tv[3 * s + k] = v[k];
        w.tn[3 * s + k] = n[k];
    }
    w.mod[s] = m;
    w.chk[s] = chk;
    w.ext[s] = ext;
}

// position of the vertex of v that is neither x nor y
__host__ __device__ __forceinline__ int other(const int* v, int x, int y) {
    return (v[0] != x && v[0] != y) ? 0 : ((v[1] != x && v[1] != y) ? 1 : 2);
}

__host__ __device__ __forceinline__ void split_body(const Work& w, int t, int tcur, int m, int chk) {
    if (!w.flag[t]) return;
    const int op = w.op[t];
    const int q = (int)(w.pick[t] & 0xffffffffu);
    const int n1 = tcur + 2 * w.rank[t], n2 = n1 + 1;
    w.loc[q] = -1;
    int v[3], vn[3];
    for (int k = 0; k < 3; ++k) {
        v[k] = w.tv[3 * t + k];
        vn[k] = w.tn[3 * t + k];
    }
    const int2 none = make_int2(-1, -1);
    if (op == 3) {
        // sub-triangle k replaces vertex k by q: slots t, n1, n2
        const int a[3] = {q, v[1], v[2]}, an[3] = {vn[0], n1, n2};
        const int b[3] = {v[0], q, v[2]}, bn[3] = {t, vn[1], n2};
        const int c[3] = {v[0], v[1], q}, cn[3] = {t, n1, vn[2]};
        put(w, t, a, an, m, chk, make_int2(n1, n2));
        put(w, n1, b, bn, m, chk, none);
        put(w, n2, c, cn, m, chk, none);
        return;
    }
    const int e = op, u = vn[e];
    int x[3], xn[3];
    for (int k = 0; k < 3; ++k) {
        x[k] = w.tv[3 * u + k];
        xn[k] = w.tn[3 * u + k];
    }
    const int f = other(x, v[nxt(e)], v[prv(e)]);  // u's edge f = (v[e+2], v[e+1])
    int a[3], b[3], an[3], bn[3];
    // t: Ta (slot t) replaces v[e+1], Tb (slot n1) replaces v[e+2]
    for (int k = 0; k < 3; ++k) a[k] = b[k] = v[k];
    a[nxt(e)] = q;
    b[prv(e)] = q;
    an[e] = n2;
    an[nxt(e)] = vn[nxt(e)];
    an[prv(e)] = n1;
    bn[e] = u;
    bn[nxt(e)] = t;
    bn[prv(e)] = vn[prv(e)];
    put(w, t, a, an, m, chk, make_int2(n1, -1));
    put(w, n1, b, bn, m, chk, none);
    // u: Ua (slot u) replaces x[f+1] = v[e+2], Ub (slot n2) replaces x[f+2] = v[e+1]
    for (int k = 0; k < 3; ++k) a[k] = b[k] = x[k];
    a[nxt(f)] = q;
    b[prv(f)] = q;
    an[f] = n1;
    an[nxt(f)] = xn[nxt(f)];
    an[prv(f)] = n2;
    bn[f] = t;
    bn[nxt(f)] = u;
    bn[prv(f)] = xn[prv(f)];
    put(w, u, a, an, m, chk, make_int2(n2, -1));
    put(w, n2, b, bn, m, chk, none);
}

__host__ __device__ __forceinline__ bool has2(const int* v, int x, int y) {
    const bool hx = v[0] == x || v[1] == x || v[2] == x;
    const bool hy = v[0] == y || v[1] == y || v[2] == y;
    return hx && hy;
}

// neighbour pointers of the slots step m rewrote: a pointer to a slot the
// same step rewrote is resolved among that slot's replacements; a slot the
// step left alone is pointed back at this one
__host__ __device__ __forceinline__ void fix_body(const Work& w, int s, int m) {
    if (w.mod[s] != m) return;
    for (int e = 0; e < 3; ++e) {
        const int x = w.tv[3 * s + nxt(e)], y = w.tv[3 * s + prv(e)];
        const int p = w.tn[3 * s + e];
        if (w.mod[p] == m) {
            const int2 ex = w.ext[p];
            const int c[3] = {p, ex.x, ex.y};
            int found = -1;
            for (int k = 0; k < 3; ++k)
                if (c[k] >= 0 && c[k] != s && has2(w.tv + 3 * c[k], x, y)) found = c[k];
            if (found < 0) aor32(w.cnt + C_ERR, ERR_LINK);
            else w.tn[3 * s + e] = found;
        } else {
            const int* pv = w.tv + 3 * p;
            if (!has2(pv, x, y)) aor32(w.cnt + C_ERR, ERR_LINK);
            else w.tn[3 * p + other(pv, x, y)] = s;
        }
    }
}

// is d strictly inside the circle of slot v (a ghost's circle: the open half
// plane outside its hull edge)?
__host__ __device__ __forceinline__ bool in_circle(const Work& w, const int* v, int d) {
    if (d == INF) return false;
    const int g = ghost_pos(v);
    if (g >= 0) return orient2d(w.p[v[nxt(g)]], w.p[v[prv(g)]], w.p[d]) > 0;
    return incircle(w.p[v[0]], w.p[v[1]], w.p[v[2]], w.p[d]) > 0;
}

__host__ __device__ __forceinline__ unsigned long long edge_key(int t, int u) {
    return t < u ? ((unsigned long long)t << 32) | (unsigned)u : ((unsigned long long)u << 32) | (unsigned)t;
}

__host__ __device__ __forceinline__ void detect_body(const Work& w, int t, int s) {
    if (w.chk[t] != s) return;
    const int* v = w.tv + 3 * t;
    int bits = 0;
    for (int e = 0; e < 3; ++e) {
        const int u = w.tn[3 * t + e];
        const int* x = w.tv + 3 * u;
        const int d = x[other(x, v[nxt(e)], v[prv(e)])];
        if (in_circle(w, v, d)) {
            bits |= 1 << e;
            const unsigned long long k = edge_key(t, u);
            amin64(w.vote + t, k);
            amin64(w.vote + u, k);
        }
    }
    w.op[t] = bits;
}

// the flip an edge's lower slot executes when the edge holds both votes;
// flagged slots are checked again in the next pass
__host__ __device__ __forceinline__ void flip_body(const Work& w, int t, int s, int m, int s2) {
    if (w.chk[t] == s && w.op[t] != 0) w.chk[t] = s2;
    const unsigned long long k = w.vote[t];
    if (k == NONE || (int)(k >> 32) != t) return;
    const int u = (int)(k & 0xffffffffu);
    if (w.vote[u] != k) return;
    int v[3], vn[3], x[3], xn[3];
    for (int j = 0; j < 3; ++j) {
        v[j] = w.tv[3 * t + j];
        vn[j] = w.tn[3 * t + j];
        x[j] = w.tv[3 * u + j];
        xn[j] = w.tn[3 * u + j];
    }
    const int e = vn[0] == u ? 0 : (vn[1] == u ? 1 : 2);
    const int c = v[e], a = v[nxt(e)], b = v[prv(e)];
    const int f = other(x, a, b);
    const int d = x[f];  // x[f+1] = b, x[f+2] = a
    const int n1a = vn[nxt(e)], n1b = vn[prv(e)], n2b = xn[nxt(f)], n2a = xn[prv(f)];
    const int X[3] = {c, a, d}, Xn[3] = {n2b, u, n1b};
    const int Y[3] = {c, d, b}, Yn[3] = {n2a, n1a, t};
    put(w, t, X, Xn, m, s2, make_int2(u, -1));
    put(w, u, Y, Yn, m, s2, make_int2(t, -1));
    aadd32(w.cnt + C_FLIPS, 1);
}

// ---- point location ------------------------------------------------------
__host__ __device__ __forceinline__ void relocate_body(const Work& w, long long i, long long cap) {
    int t = w.loc[i];
    if (t < 0) return;
    const double2 q = w.p[i];
    int o[3] = {1, 1, 1};
    long long steps = 0;
    bool ghost = false;
    for (;; ++steps) {
        if (steps > cap) {
            aor32(w.cnt + C_ERR, ERR_WALK);
            return;
        }
        const int* v = w.tv + 3 * t;
        const int g = ghost_pos(v);
        if (g >= 0) {
            if (orient2d(w.p[v[nxt(g)]], w.p[v[prv(g)]], q) > 0) {
                ghost = true;
                break;
            }
            t = w.tn[3 * t + g];
            continue;
        }
        int e = 0;
        for (; e < 3; ++e) {
            o[e] = orient2d(w.p[v[nxt(e)]], w.p[v[prv(e)]], q);
            if (o[e] < 0) break;
        }
        if (e == 3) break;
        t = w.tn[3 * t + e];
    }
    if (ghost) {
        // the last ghost of the chain of hull edges q sees, walking towards v[g+2]
        for (;; ++steps) {
            if (steps > cap) {
                aor32(w.cnt + C_ERR, ERR_WALK);
                return;
            }
            const int g = ghost_pos(w.tv + 3 * t);
            const int n = w.tn[3 * t + nxt(g)];
            const int* nv = w.tv + 3 * n;
            const int ng = ghost_pos(nv);
            if (ng < 0 || !(orient2d(w.p[nv[nxt(ng)]], w.p[nv[prv(ng)]], q) > 0)) break;
            t = n;
        }
        w.loc[i] = t;
        aadd32(w.cnt + C_LEFT, 1);
        return;
    }
    const int* v = w.tv + 3 * t;
    for (int k = 0; k < 3; ++k) {
        const double2 c = w.p[v[k]];
        if (c.x == q.x && c.y == q.y) {
            w.loc[i] = -2;  // a duplicate of vertex v[k], whose index is lower
            return;
        }
    }
    for (int e = 0; e < 3; ++e)
        if (o[e] == 0) {
            const int u = w.tn[3 * t + e];
            if (ghost_pos(w.tv + 3 * u) < 0 && u < t) t = u;
        }
    w.loc[i] = t;
    aadd32(w.cnt + C_LEFT, 1);
}

// ---- output ----------------------------------------------------------------
__host__ __device__ __forceinline__ void finite_body(const Work& w, int t) {
    w.flag[t] = ghost_pos(w.tv + 3 * t) < 0;
}

// scipy's layout: simplices and neighbors (T,3), transform (T,3,2) =
// {Tinv, r} with T = [v0 - r, v1 - r] as columns, r = v2
__host__ __device__ __forceinline__ void output_body(const Work& w, int t, int* simp, int* nbr, double* tr) {
    if (!w.flag[t]) return;
    const long long o = w.rank[t];
    const int* v = w.tv + 3 * t;
    for (int k = 0; k < 3; ++k) simp[3 * o + k] = v[k];
    if (nbr)
        for (int k = 0; k < 3; ++k) {
            const int u = w.tn[3 * t + k];
            nbr[3 * o + k] = w.flag[u] ? w.rank[u] : -1;
        }
    if (tr) {
        const double2 a = w.p[v[0]], b = w.p[v[1]], r = w.p[v[2]];
        const double t00 = DT_SUB(a.x, r.x), t01 = DT_SUB(b.x, r.x);
        const double t10 = DT_SUB(a.y, r.y), t11 = DT_SUB(b.y, r.y);
        const double det = DT_SUB(DT_MUL(t00, t11), DT_MUL(t01, t10));
        double* out = tr + 6 * o;
        if (det == 0.0) {
            for (int k = 0; k < 6; ++k) out[k] = NAN;
            return;
        }
        out[0] = DT_DIV(t11, det);
        out[1] = DT_DIV(-t01, det);
        out[2] = DT_DIV(-t10, det);
        out[3] = DT_DIV(t00, det);
        out[4] = r.x;
        out[5] = r.y;
    }
}

// ---- kernels ---------------------------------------------------------------
#ifdef __CUDACC__
#define DT_FOR(i, n)                                                                \
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < (n); \
         i += (long long)gridDim.x * blockDim.x)

__global__ void __launch_bounds__(LEX_THREADS) lex_kernel(Work w) {
    __shared__ long long s[2 * LEX_THREADS];
    lex_body(w, blockIdx.x, threadIdx.x, s);
    __syncthreads();
    if (threadIdx.x == 0) lex_reduce(w, s, LEX_THREADS, w.lex + 2 * blockIdx.x, w.lex + 2 * blockIdx.x + 1);
}
__global__ void lex_final_kernel(Work w) {
    lex_reduce(w, w.lex, LEX_BLOCKS, w.lex + 2 * LEX_BLOCKS, w.lex + 2 * LEX_BLOCKS + 1);
}
__global__ void __launch_bounds__(256) seed_kernel(Work w) { DT_FOR(i, w.M) seed_body(w, i); }
__global__ void init_kernel(Work w) { init_body(w); }
__global__ void __launch_bounds__(256) pick_kernel(Work w) { DT_FOR(i, w.M) pick_body(w, i); }
__global__ void __launch_bounds__(256) claim_kernel(Work w, int n) { DT_FOR(t, n) claim_body(w, (int)t); }
__global__ void __launch_bounds__(256) decide_kernel(Work w, int n) { DT_FOR(t, n) decide_body(w, (int)t); }
__global__ void __launch_bounds__(256) split_kernel(Work w, int n, int m, int chk) {
    DT_FOR(t, n) split_body(w, (int)t, n, m, chk);
}
__global__ void __launch_bounds__(256) fix_kernel(Work w, int n, int m) { DT_FOR(t, n) fix_body(w, (int)t, m); }
__global__ void __launch_bounds__(256) detect_kernel(Work w, int n, int s) {
    DT_FOR(t, n) detect_body(w, (int)t, s);
}
__global__ void __launch_bounds__(256) flip_kernel(Work w, int n, int s, int m, int s2) {
    DT_FOR(t, n) flip_body(w, (int)t, s, m, s2);
}
__global__ void __launch_bounds__(256) relocate_kernel(Work w, long long cap) {
    DT_FOR(i, w.M) relocate_body(w, i, cap);
}
__global__ void __launch_bounds__(256) finite_kernel(Work w, int n) { DT_FOR(t, n) finite_body(w, (int)t); }
__global__ void __launch_bounds__(256) output_kernel(Work w, int n, int* simp, int* nbr, double* tr) {
    DT_FOR(t, n) output_body(w, (int)t, simp, nbr, tr);
}

// exclusive prefix sum of flag[0, n) into rank, the total into bsum[nb]:
// block totals, one block scanning them, then each block's own scan
constexpr int SCAN_THREADS = 1024;
__device__ __forceinline__ int block_exclusive_scan(int x, int* sh, int* total) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    int v = x;
    for (int d = 1; d < 32; d <<= 1) {
        const int u = __shfl_up_sync(0xffffffffu, v, d);
        if (lane >= d) v += u;
    }
    if (lane == 31) sh[wid] = v;
    __syncthreads();
    if (wid == 0) {
        int s = sh[lane];
        for (int d = 1; d < 32; d <<= 1) {
            const int u = __shfl_up_sync(0xffffffffu, s, d);
            if (lane >= d) s += u;
        }
        sh[lane] = s;
    }
    __syncthreads();
    const int r = v - x + (wid ? sh[wid - 1] : 0);
    *total = sh[31];
    __syncthreads();
    return r;
}
__global__ void __launch_bounds__(SCAN_THREADS) scan_block_kernel(const int* flag, int n, int* bsum) {
    __shared__ int sh[32];
    const long long k = (long long)blockIdx.x * SCAN_THREADS + threadIdx.x;
    int total;
    block_exclusive_scan(k < n ? flag[k] : 0, sh, &total);
    if (threadIdx.x == 0) bsum[blockIdx.x] = total;
}
__global__ void __launch_bounds__(SCAN_THREADS) scan_top_kernel(int* bsum, int nb) {
    __shared__ int sh[32];
    const int per = (nb + SCAN_THREADS - 1) / SCAN_THREADS;
    const int b0 = min(nb, (int)threadIdx.x * per), b1 = min(nb, b0 + per);
    int s = 0;
    for (int b = b0; b < b1; ++b) s += bsum[b];
    int total;
    int run = block_exclusive_scan(s, sh, &total);
    for (int b = b0; b < b1; ++b) {
        const int x = bsum[b];
        bsum[b] = run;
        run += x;
    }
    if (threadIdx.x == 0) bsum[nb] = total;
}
__global__ void __launch_bounds__(SCAN_THREADS) scan_apply_kernel(const int* flag, int n, const int* bsum,
                                                                   int* rank) {
    __shared__ int sh[32];
    const long long k = (long long)blockIdx.x * SCAN_THREADS + threadIdx.x;
    int total;
    const int r = block_exclusive_scan(k < n ? flag[k] : 0, sh, &total);
    if (k < n) rank[k] = bsum[blockIdx.x] + r;
}

// orient2d(a, b, c) and incircle(a, b, c, d) of n quadruples (8 doubles each)
__global__ void __launch_bounds__(256) selftest_predicates_kernel(const double* q, long long n, int* out) {
    DT_FOR(i, n) {
        const double* r = q + 8 * i;
        const double2 a = make_double2(r[0], r[1]), b = make_double2(r[2], r[3]);
        const double2 c = make_double2(r[4], r[5]), d = make_double2(r[6], r[7]);
        out[2 * i] = orient2d(a, b, c);
        out[2 * i + 1] = incircle(a, b, c, d);
    }
}
#undef DT_FOR
#endif  // __CUDACC__

}  // namespace dt
}  // namespace rtx
