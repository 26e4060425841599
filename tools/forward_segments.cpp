// forward_segments.cpp - developer tool (tools/forward_segments.py): model of a SEGMENTED prediction walk for the
// chain kernel's forward pass (CoopEvaluator::forward_coop, metis_coop.cuh), measured on every balancer run the
// chain kernel makes.
//
// The walk predicts the stage starts one stage after the other; the start of stage s + 1 depends only on the start
// of stage s.  A segmented walk splits the warp into G lane groups: group g walks the stages [s_g, s_{g+1} + K) from
// a GUESSED start of s_g with a 32/G-entry window, all groups at once.  At boundary g the true path of group g - 1
// is compared with group g's over the K overlap stages: from the first stage where both start at the same sub-layer
// on, group g's path is the true one.  If they do not meet, the uniform walk continues from the true state until its
// start equals the recorded start of the group that owns the stage, or to the end.  Counted per run: the concurrent
// steps (the longest group's walk) plus the continuation steps, against today's S - 1.
//
// The runs come from the host build of the search's schedule (first-task round, then the chain evaluator for the
// plans that continue, like tests/hostsim mode 1); a lane policy on top of OneLane reads the forward pass's input
// (w.perf) at the mark that opens the balancer's fill.  Nothing here is part of the library.
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <vector>

#include "../metis_b200/csrc/metis_eval.cuh"
#include "../metis_b200/csrc/metis_coop.cuh"

#ifndef FS_MAXS
#define FS_MAXS METIS_MAX_STAGES
#endif
#ifndef FS_MAXL
#define FS_MAXL METIS_MAX_LAYERS
#endif
#ifndef FS_ONE
#define FS_ONE 0
#endif

using namespace metis;

namespace {

constexpr int kS = FS_MAXS, kL = FS_MAXL;
constexpr bool kOne = FS_ONE != 0;

constexpr int kNG = 3, kNK = 3, kNGuess = 3, kHist = 34;
const int kG[kNG] = {2, 4, 8};
const int kK[kNK] = {2, 4, 8};
const char *kGuessName[kNGuess] = {"perf prefix", "perf prefix + d/2 per stage", "stage lengths"};
int g_place = 0;   // window placement: 0 = today's (previous stage's length), 1 = from the stage's demand

// first i in [0, n] with P[i] >= t (OneLane::first_ge)
int fge(const double *P, int n, double t) {
    int lo = 0, hi = n + 1;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (P[mid] >= t) hi = mid; else lo = mid + 1; }
    return lo;
}
// OneLane::first_ge_window with a W-entry window
int first_ge_window(const double *P, int n, int i0, int lo, double t, int W) {
    for (int k = 0; k < W && i0 + k <= n; ++k)
        if (P[i0 + k] >= t) return (k > 0 || i0 <= lo) ? i0 + k : -1;
    return -1;
}

struct Walk { int a, span; };
// one step of forward_coop's walk with a W-entry window; returns the stage's start
int walk_step(const double *P, int N, int lim, const double *perf, int s, Walk &st, int W, long &miss) {
    const int a = st.a;
    if (a >= lim) return a;
    const double t = perf[s] + P[a];
    int i0;
    if (g_place) {
        const double d = P[a + 1] - P[a];
        i0 = a + (d > 0.0 ? (int)(perf[s] / d) : st.span) + 2 - W / 2;
    } else {
        i0 = a + st.span - (W / 2 - 2);
    }
    if (i0 < a + 1) i0 = a + 1;
    int i = first_ge_window(P, N, i0, a + 1, t, W);
    if (i < 0) { ++miss; i = fge(P, N, t); }
    int b = i - 1 > a ? i - 1 : a;
    const bool closed = b < lim;
    if (!closed) b = lim;
    st.span = b - a;
    st.a = closed ? b + 1 : lim;
    return a;
}

struct Stats {
    long runs = 0, steps = 0, miss = 0;
    long sh[METIS_MAX_STAGES + 2] = {};
    long gsteps[kNG][kNGuess] = {}, gmiss[kNG][kNGuess] = {};
    long hist[kNG][kNGuess][kHist] = {};                       // stages until the paths merge, per boundary
    long model[kNG][kNK][kNGuess] = {}, cont[kNG][kNK][kNGuess] = {};
    long bnd[kNG][kNK][kNGuess] = {}, nomerge[kNG][kNK][kNGuess] = {};
} g_st;

void model_run(const double *P, int N, int lim, int last, const double *perf) {
    Stats &A = g_st;
    ++A.runs;
    ++A.sh[last + 1];
    std::vector<int> truth(last);
    Walk w0{0, lim / last};
    for (int s = 0; s < last; ++s) truth[s] = walk_step(P, N, lim, perf, s, w0, 32, A.miss);
    A.steps += last;
    std::vector<double> pre(last + 1, 0.0);
    for (int s = 0; s < last; ++s) pre[s + 1] = pre[s] + perf[s];
    for (int gi = 0; gi < kNG; ++gi) {
        const int G = kG[gi], W = 32 / G, seg = (last + G - 1) / G;
        for (int q = 0; q < kNGuess; ++q) {
            std::vector<std::vector<int>> rec(G);
            for (int g = 0; g < G; ++g) {
                const int sg = g * seg;
                if (sg >= last) break;
                int a0 = 0;
                if (g > 0 && q < 2) {
                    const int ia = fge(P, N, pre[sg]);
                    const double d = ia < N ? P[ia + 1] - P[ia] : 0.0;
                    a0 = fge(P, N, pre[sg] + (q == 1 ? 0.5 * sg * d : 0.0));
                } else if (g > 0) {
                    // each earlier stage's length from its start estimated by the perf prefix, added up
                    for (int t = 0; t < sg && a0 < lim; ++t) {
                        const int at = fge(P, N, pre[t]);
                        if (at >= lim) { a0 = lim; break; }
                        const int i = fge(P, N, perf[t] + P[at]);
                        const int b = i - 1 > at ? i - 1 : at;
                        a0 = b >= lim ? lim : a0 + b + 1 - at;
                    }
                }
                if (a0 > lim) a0 = lim;
                Walk wg{a0, lim / last};
                for (int s = sg; s < last && s < sg + seg + kK[kNK - 1]; ++s) {
                    rec[g].push_back(walk_step(P, N, lim, perf, s, wg, W, A.gmiss[gi][q]));
                    ++A.gsteps[gi][q];
                }
            }
            for (int g = 1; g < G && g * seg < last; ++g) {
                const int sg = g * seg;
                int j = 0;
                while (j < kHist - 1 && j < (int)rec[g].size() && rec[g][j] != truth[sg + j]) ++j;
                if (j == (int)rec[g].size()) j = kHist - 1;
                ++A.hist[gi][q][j < kHist - 1 ? j : kHist - 1];
            }
            for (int ki = 0; ki < kNK; ++ki) {
                const int K = kK[ki];
                long cont = 0;
                int g = 1;
                while (g < G && g * seg < last) {
                    const int sg = g * seg;
                    ++A.bnd[gi][ki][q];
                    const int kc = K < last - sg ? K : last - sg;
                    int j = 0;
                    while (j < kc && rec[g][j] != truth[sg + j]) ++j;
                    if (j < kc) { ++g; continue; }
                    ++A.nomerge[gi][ki][q];
                    int s = sg + kc;
                    bool met = false;
                    for (; s < last; ++s) {
                        ++cont;
                        const int h = s / seg;
                        if (rec[h][s - h * seg] == truth[s]) { met = true; g = h + 1; break; }
                    }
                    if (!met) break;
                }
                A.model[gi][ki][q] += (seg + K < last ? seg + K : last) + cont;
                A.cont[gi][ki][q] += cont;
            }
        }
    }
}

// OneLane with a look at the forward pass's input: mark 10 opens the balancer's fill (CoopEvaluator::balance_coop)
struct ProbeLane : OneLane {
    const Tables *T = nullptr;
    const Scratch<kS, kL> *w = nullptr;
    const int *S = nullptr;
    void mark(int id) const {
        if (id != 10) return;
        const int L = T->p.num_layers, n = *S;
        if (n < 4 || T->p.norm_len < L) return;             // forward_coop runs the sequential pass
        const int N = kH * L, lim = (N - 1 - kH) > 0 ? (N - 1 - kH) : 0;
        model_run(T->psub, N, lim, n - 1, w->perf);
    }
};

struct NullSink {
    void phase(int) {}
    void partition_call() {}
    void balancer_run() {}
    void keyerror() {}
    void fatal(uint32_t, int, uint32_t) {}
    void emit(const PlanDesc &, int, int, double, const uint8_t *, const uint16_t *) {}
};

bool decode(const MetisPlanSpace &sp, int64_t ordinal, PlanDesc &pd) {
    if (ordinal < 0 || ordinal >= sp.num_plans) return false;
    int b = 0;
    for (int i = 0; i < sp.num_blocks; ++i)
        if (sp.blocks[i].first_ordinal <= ordinal) b = i;
    const MetisPlanBlock &blk = sp.blocks[b];
    const int64_t rel = ordinal - blk.first_ordinal;
    const int64_t row = rel / sp.num_div;
    pd.ordinal = (uint32_t)ordinal;
    pd.ns = blk.ns_idx;
    pd.S = blk.num_stage;
    pd.label = blk.label_stage;
    pd.batches = sp.batches[rel - row * sp.num_div];
    pd.row = sp.rows + blk.rows_offset + row * blk.num_stage;
    pd.geo = pack_geo(blk.rows_offset + row * blk.num_stage, blk.num_stage, blk.label_stage, blk.ns_idx,
                      (int)(rel - row * sp.num_div));
    return true;
}

}  // namespace

extern "C" {

// runs the search's schedule over the whole space and prints the model's table; returns 0, or -1 when the space is
// outside this build's instantiation
int forward_segments(const MetisProblem *p, const MetisPlanSpace *sp, int place) {
    if (sp->max_stage > kS || p->num_layers > kL || (kOne && p->num_types != 1)) return -1;
    g_place = place;
    g_st = Stats();
    Tables T;
    T.p = *p;
    const int L = p->num_layers;
    const size_t n = (size_t)L + 1;
    std::vector<double> rs((size_t)range_sum_tables(*p) * n * n, -1.0);
    for (int t = 0; t < range_sum_tables(*p); ++t) {
        const double *row = range_sum_row(*p, t, p->layer_memory, p->layer_compute, p->norm_lc);
        if (!row) continue;
        for (int a = 0; a < L; ++a) fill_range_sums(row, L, a, rs.data() + (size_t)t * n * n);
    }
    T.rsum = rs.data();
    T.key_index = p->key_index;
    T.lc = p->layer_compute;
    T.mem = p->layer_memory;
    T.exec_full = p->exec_full;
    T.fb_sync = p->fb_sync;
    T.norm_lc = p->norm_lc;
    const DerivedLayout d = derived_layout(*p);
    std::vector<double> dlay(d.total);
    for (int i = 0; i < d.total; ++i) dlay[i] = derive_entry(*p, d, p->norm_lc, p->exec_full, p->type_bw_first, i);
    T.type_memory = p->type_memory;
    T.bw_first = p->type_bw_first;
    T.bw_min = p->type_bw_min;
    T.run_type = p->ns_run_type;
    T.run_end = p->ns_run_end;
    T.q10_end = p->ns_q10_end;
    bind_derived(T, dlay.data());

    static Scratch<kS, kL> w;
    static CoopMail mail;
    NullSink sink;
    int S = 0;
    ProbeLane lanes;
    lanes.T = &T; lanes.w = &w; lanes.S = &S;
    std::vector<double> saved;
    for (int64_t o = 0; o < sp->num_plans; ++o) {
        PlanDesc pd;
        if (!decode(*sp, o, pd)) continue;
        {
            PlanEvaluator<kS, kL, Serial, kOne> probe(T, w);
            if (probe.begin(pd) <= 0) continue;
        }
        int hint = 0, start = 1;
        if (!first_task<kS, kL, kOne>(T, w, sink, true, pd, hint, start)) continue;   // finished by the bulk round
        if (start == 2) saved.assign(w.perf, w.perf + pd.S);
        S = pd.S;
        CoopEvaluator<kS, kL, ProbeLane, kOne> ev(T, w, mail, lanes);
        ev.run_chain(pd, sink, start, saved.data(), 1);
    }

    const Stats &A = g_st;
    const double runs = A.runs ? (double)A.runs : 1.0;
    printf("chain-kernel balancer runs with a predicted forward pass: %ld, walk steps per run today %.2f, "
           "window misses %.2f %%\n", A.runs, A.steps / runs, 100.0 * A.miss / (A.steps ? A.steps : 1));
    printf("stages per run:");
    for (int i = 0; i < METIS_MAX_STAGES + 2; ++i) if (A.sh[i]) printf(" %d:%ld", i, A.sh[i]);
    printf("\n");
    for (int q = 0; q < kNGuess; ++q) {
        printf("guess: %s\n", kGuessName[q]);
        for (int gi = 0; gi < kNG; ++gi) {
            long tot = 0, at0 = 0, within = 0;
            for (int j = 0; j < kHist; ++j) tot += A.hist[gi][q][j];
            at0 = A.hist[gi][q][0];
            for (int j = 0; j < kHist - 1; ++j) within += A.hist[gi][q][j];
            printf("  G=%d  window %2d: misses %5.2f %%  boundaries %ld: merged at the boundary %5.1f %%, later %5.1f %%, "
                   "never %5.1f %%\n", kG[gi], 32 / kG[gi], 100.0 * A.gmiss[gi][q] / (A.gsteps[gi][q] ? A.gsteps[gi][q] : 1),
                   tot, 100.0 * at0 / (tot ? tot : 1), 100.0 * (within - at0) / (tot ? tot : 1),
                   100.0 * (tot - within) / (tot ? tot : 1));
            for (int ki = 0; ki < kNK; ++ki)
                printf("     K=%d  no merge within K %5.1f %%  steps/run %6.2f = %5.3f of today (continuation %5.2f)\n",
                       kK[ki], 100.0 * A.nomerge[gi][ki][q] / (A.bnd[gi][ki][q] ? A.bnd[gi][ki][q] : 1),
                       A.model[gi][ki][q] / runs, (double)A.model[gi][ki][q] / (A.steps ? A.steps : 1),
                       A.cont[gi][ki][q] / runs);
        }
    }
    fflush(stdout);
    return 0;
}

}  // extern "C"
