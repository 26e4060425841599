// forward_index_sim.cpp - test-only g++ build of the chain kernel's forward prediction (CoopEvaluator::forward_coop,
// metis_coop.cuh) with and without the bucket index of psub (Tables::pidx), for tests/test_forward_index.py.
//
// Every comparison runs forward_coop twice on the same stage performances: once on the tables as derive_entry builds
// them, once on a copy whose index is empty (scale 0.0), which walks with today's window probes.  The predicted
// interval starts and ends (w.first, w.fe), the verdict of the replay and, when it verifies, the residual capacities
// and the mailbox must be identical.  The index walk's refine steps are counted from the data: the answer minus the
// index's guess max(IX[g], a + 1).
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../metis_b200/csrc/metis_eval.cuh"
#include "../../metis_b200/csrc/metis_coop.cuh"

#ifndef FI_MAXS
#define FI_MAXS METIS_MAX_STAGES
#endif
#ifndef FI_MAXL
#define FI_MAXL METIS_MAX_LAYERS
#endif
#ifndef FI_ONE
#define FI_ONE 0
#endif

using namespace metis;

namespace {

constexpr int kS = FI_MAXS, kL = FI_MAXL;
constexpr bool kOne = FI_ONE != 0;

// counters returned to Python (fi_* out arrays), in this order
enum {
    kRuns,          // forward passes compared (S >= 4, psub present)
    kIndexed,       // of which the tables had an index
    kMismatch,      // runs whose two predictions differ in anything
    kSteps,         // walked stages (a < lim)
    kTail,          // walked stages with t > P[lim]: open, no lookup
    kStep0,         // lookups whose guess was the answer
    kStep1,         // one step up
    kWindow,        // the answer 2 .. 31 above the guess: the window at the guess finds it
    kFar,           // anything else: the whole-table search
    kFirstGeIndex,  // whole-table searches of the index walk (kPathFirstGe notes)
    kFirstGeToday,  // whole-table searches of today's walk
    kVerified,      // runs whose prediction verified
    kNumCounters
};

struct CountLane : OneLane {
    int64_t *searches = nullptr;
    void note(int p) const { if (p == kPathFirstGe) ++*searches; }
};

Tables without_index(const Tables &T, std::vector<double> &scale) {
    Tables U = T;
    scale.assign(1, 0.0);
    U.pidx = scale.data();
    return U;
}

// both walks on the stage performances perf[0 .. S): counters += what happened
void compare(const Tables &T, const Tables &U, const double *perf, int S, int64_t *c) {
    static Scratch<kS, kL> w1, w2;
    static CoopMail m1, m2;
    const int L = T.p.num_layers;
    if (S < 4 || T.p.norm_len < L) return;
    memset(&m1, 0, sizeof(m1));
    memset(&m2, 0, sizeof(m2));
    for (int s = 0; s < S; ++s) { w1.perf[s] = w2.perf[s] = perf[s]; w1.capa[s] = w2.capa[s] = perf[s]; }
    CountLane x1, x2;
    x1.searches = &c[kFirstGeIndex];
    x2.searches = &c[kFirstGeToday];
    CoopEvaluator<kS, kL, CountLane, kOne> e1(T, w1, m1, x1), e2(U, w2, m2, x2);
    e1.pd.S = S;
    e2.pd.S = S;
    const bool r1 = e1.forward_coop(), r2 = e2.forward_coop();
    ++c[kRuns];
    c[kIndexed] += T.pidx[0] > 0.0;
    c[kVerified] += r1;
    bool same = r1 == r2;
    for (int s = 0; s + 1 < S; ++s) same = same && w1.first[s] == w2.first[s] && w1.fe[s] == w2.fe[s];
    if (same && r1) {
        for (int s = 0; s + 1 < S; ++s) same = same && memcmp(&w1.capa[s], &w2.capa[s], sizeof(double)) == 0;
        same = same && m1.k == m2.k && m1.s_top == m2.s_top && m1.top_skip == m2.top_skip;
    }
    c[kMismatch] += !same;
    // refine steps of the index walk, from the prediction
    const double scale = T.pidx[0];
    if (!(scale > 0.0)) return;
    const uint16_t *IX = reinterpret_cast<const uint16_t *>(T.pidx + 1);
    const double *P = T.psub;
    const int N = kH * L, lim = (N - 1 - kH) > 0 ? (N - 1 - kH) : 0;
    for (int s = 0; s + 1 < S; ++s) {
        const int a = w1.first[s];
        if (a >= lim) break;
        ++c[kSteps];
        const double t = perf[s] + P[a];
        if (!(t <= P[lim])) { ++c[kTail]; continue; }
        int guess = IX[bucket_of(t * scale)];
        if (guess < a + 1) guess = a + 1;
        const int d = (int)(w1.fe[s] & kPos) + 1 - guess;
        ++c[d == 0 ? kStep0 : d == 1 ? kStep1 : (d >= 2 && d <= 31) ? kWindow : kFar];
    }
}

// OneLane with a look at the balancer's input: mark 10 opens the fill (CoopEvaluator::balance_coop)
struct ProbeLane : OneLane {
    const Tables *T = nullptr, *U = nullptr;
    const Scratch<kS, kL> *w = nullptr;
    const int *S = nullptr;
    int64_t *c = nullptr;
    void mark(int id) const { if (id == 10) compare(*T, *U, w->perf, *S, c); }
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

// derived tables of a minimal problem (no keys, batch sizes or tp), entry by entry like pack_tables_kernel
Tables minimal_tables(MetisProblem &p, const double *lc, int norm_len, int num_layers, std::vector<double> &derived) {
    memset(&p, 0, sizeof(p));
    p.num_layers = num_layers;
    p.norm_len = norm_len;
    static const double bw[1] = {1.0};
    const DerivedLayout d = derived_layout(p);
    derived.assign(d.total + 1, 0.0);
    for (int i = 0; i < d.total; ++i) derived[i] = derive_entry(p, d, lc, nullptr, bw, i);
    Tables T;
    memset(&T, 0, sizeof(T));
    T.p = p;
    T.norm_lc = lc;
    bind_derived(T, derived.data());
    return T;
}

}  // namespace

extern "C" {

uint64_t fi_instantiation() { return (uint64_t)kS | (uint64_t)kL << 16 | (uint64_t)kOne << 32; }
int fi_num_counters() { return kNumCounters; }

// every balancer run the chain kernel makes in the search's schedule (bulk round on the host, then the chain
// evaluator for the plans that continue, like tests/hostsim mode 1): both walks compared at the start of each fill
int fi_search(const MetisProblem *p, const MetisPlanSpace *sp, int64_t *counters) {
    if (sp->max_stage > kS || p->num_layers > kL || (kOne && p->num_types != 1)) return -1;
    memset(counters, 0, sizeof(int64_t) * kNumCounters);
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
    std::vector<double> derived(d.total + 1);
    for (int i = 0; i < d.total; ++i) derived[i] = derive_entry(*p, d, p->norm_lc, p->exec_full, p->type_bw_first, i);
    T.type_memory = p->type_memory;
    T.bw_first = p->type_bw_first;
    T.bw_min = p->type_bw_min;
    T.run_type = p->ns_run_type;
    T.run_end = p->ns_run_end;
    T.q10_end = p->ns_q10_end;
    bind_derived(T, derived.data());
    std::vector<double> copy;
    const Tables U = without_index(T, copy);

    static Scratch<kS, kL> w;
    static CoopMail mail;
    NullSink sink;
    int S = 0;
    ProbeLane lanes;
    lanes.T = &T; lanes.U = &U; lanes.w = &w; lanes.S = &S; lanes.c = counters;
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
    return 0;
}

// both walks on capacity rows (stage performances) over the normalised layer weights lc[0 .. norm_len)
int fi_rows(const double *capa, const int32_t *num_stage, int64_t n, int32_t stride, const double *lc, int32_t norm_len,
            int32_t num_layers, int64_t *counters) {
    if (num_layers > kL) return -1;
    for (int64_t i = 0; i < n; ++i)
        if (num_stage[i] < 1 || num_stage[i] > kS || num_stage[i] > stride) return -1;
    memset(counters, 0, sizeof(int64_t) * kNumCounters);
    MetisProblem p;
    std::vector<double> derived, copy;
    const Tables T = minimal_tables(p, lc, norm_len, num_layers, derived);
    const Tables U = without_index(T, copy);
    for (int64_t i = 0; i < n; ++i) compare(T, U, capa + i * stride, num_stage[i], counters);
    return 0;
}

// psub and its index for lc: P[0 .. 7 L] and the scale (0.0: no index); returns 7 L, or -1 without psub
int fi_psub(const double *lc, int32_t norm_len, int32_t num_layers, double *P, double *scale) {
    if (norm_len < num_layers) return -1;
    MetisProblem p;
    std::vector<double> derived;
    const Tables T = minimal_tables(p, lc, norm_len, num_layers, derived);
    const int N = kH * num_layers;
    for (int i = 0; i <= N; ++i) P[i] = T.psub[i];
    *scale = T.pidx[0];
    return N;
}

// psub_lookup (metis_coop.cuh) for queries (t, lo) with t <= psub[lim], 1 <= lo <= lim; out[q] = the index, and
// the entry it returned must be psub[out[q]] (else out[q] = -1)
int fi_lookup(const double *lc, int32_t norm_len, int32_t num_layers, const double *t, const int32_t *lo, int64_t n,
              int32_t *out) {
    if (norm_len < num_layers) return -1;
    MetisProblem p;
    std::vector<double> derived;
    const Tables T = minimal_tables(p, lc, norm_len, num_layers, derived);
    if (!(T.pidx[0] > 0.0)) return -2;
    const uint16_t *IX = reinterpret_cast<const uint16_t *>(T.pidx + 1);
    const int N = kH * num_layers;
    OneLane x;
    for (int64_t q = 0; q < n; ++q) {
        double v = NAN;
        const int i = psub_lookup(x, T.psub, IX, T.pidx[0], N, lo[q], t[q], v);
        out[q] = (i >= 0 && i <= N && memcmp(&v, &T.psub[i], sizeof(v)) == 0) ? i : -1;
    }
    return 0;
}

}  // extern "C"
