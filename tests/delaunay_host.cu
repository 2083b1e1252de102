// Sequential host driver of the device triangulation's step bodies
// (rayopt_b200/csrc/rtx_delaunay.cuh), in the order rtx_delaunay launches
// them: the topology (splits, 2 -> 4, ghost flips, pointer repair, relocation)
// can be checked without a GPU.  Built and loaded by tests/test_delaunay_host.py.
#include "../rayopt_b200/csrc/rtx_delaunay.cuh"

#include <vector>

using namespace rtx::dt;

static int prefix_sum(const Work& w, int n) {
    int s = 0;
    for (int k = 0; k < n; ++k) {
        w.rank[k] = s;
        s += w.flag[k];
    }
    return s;
}

// returns 0 and *T triangles (room for 2M) or the refusal / error code
extern "C" int dt_host(long long M, const double* pts, long long* T, int* simp, int* nbr, double* tr) {
    const long long S = 2 * M;
    std::vector<int> tv(3 * S), tn(3 * S), mod(S), chk(S), op(S), flag(S), rank(S), loc(M), bsum(1);
    std::vector<int2> ext(S);
    std::vector<unsigned long long> pick(S), vote(S);
    std::vector<unsigned> cnt(C_N, 0);
    std::vector<long long> lex(2 * LEX_BLOCKS + 2);
    unsigned long long seed = NONE;
    Work w{(const double2*)pts, M,          tv.data(),  tn.data(),   mod.data(),  chk.data(),
           ext.data(),          pick.data(), vote.data(), op.data(),   flag.data(), rank.data(),
           bsum.data(),         loc.data(),  cnt.data(),  lex.data(),  &seed};
    for (int b = 0; b < LEX_BLOCKS; ++b) {
        long long s[2 * LEX_THREADS];
        for (int t = 0; t < LEX_THREADS; ++t) lex_body(w, b, t, s);
        lex_reduce(w, s, LEX_THREADS, &lex[2 * b], &lex[2 * b + 1]);
    }
    lex_reduce(w, lex.data(), LEX_BLOCKS, &lex[2 * LEX_BLOCKS], &lex[2 * LEX_BLOCKS + 1]);
    if (cnt[C_ERR]) return -1;
    for (long long i = 0; i < M; ++i) seed_body(w, i);
    if (seed == NONE) return -1;
    for (long long i = 0; i < M; ++i) loc[i] = 0;
    init_body(w);
    int tcur = 4, stamp = 1;
    const long long cap = 2 * M + 16;
    for (long long i = 0; i < M; ++i) relocate_body(w, i, cap);
    while (cnt[C_LEFT]) {
        for (int t = 0; t < tcur; ++t) pick[t] = vote[t] = NONE;
        for (long long i = 0; i < M; ++i) pick_body(w, i);
        for (int t = 0; t < tcur; ++t) claim_body(w, t);
        for (int t = 0; t < tcur; ++t) decide_body(w, t);
        const int added = prefix_sum(w, tcur);
        const int m = stamp++;
        int s = stamp++;
        for (int t = 0; t < tcur; ++t) split_body(w, t, tcur, m, s);
        tcur += 2 * added;
        for (int t = 0; t < tcur; ++t) fix_body(w, t, m);
        for (;;) {
            for (int t = 0; t < tcur; ++t) vote[t] = NONE;
            cnt[C_FLIPS] = 0;
            const int m2 = stamp++, s2 = stamp++;
            for (int t = 0; t < tcur; ++t) detect_body(w, t, s);
            for (int t = 0; t < tcur; ++t) flip_body(w, t, s, m2, s2);
            for (int t = 0; t < tcur; ++t) fix_body(w, t, m2);
            s = s2;
            if (!cnt[C_FLIPS]) break;
        }
        cnt[C_LEFT] = 0;
        for (long long i = 0; i < M; ++i) relocate_body(w, i, cap);
        if (cnt[C_ERR]) return -2;
    }
    for (int t = 0; t < tcur; ++t) finite_body(w, t);
    *T = prefix_sum(w, tcur);
    for (int t = 0; t < tcur; ++t) output_body(w, t, simp, nbr, tr);
    return 0;
}
