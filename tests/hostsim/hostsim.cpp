// hostsim.cpp - TEST-ONLY host build of the device evaluator (metis_b200/csrc/metis_eval.cuh).
//
// The build container has nvcc but no GPU.  Compiling the very same per-plan evaluator with
// g++ lets the CPU test-suite check the *device logic* (compact load-balancer state, chain,
// cost model) against the oracle before spending GPU time.  This shim is built and loaded only
// by tests/ (tests/hostsim_util.py); the metis_b200 package never loads it and has no CPU path.
// Build: g++ -O2 -ffp-contract=off -shared -fPIC (no FMA contraction, like nvcc -fmad=false).
// -DHOSTSIM_MAXS=S -DHOSTSIM_MAXL=L -DHOSTSIM_ONE=0/1 pick the instantiation <MAXS, MAXL, ONE> of the evaluator,
// like metis_het_search picks one of its search kernels (default: the compiled limits, general case).
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../metis_b200/csrc/metis_eval.cuh"
#include "../../metis_b200/csrc/metis_coop.cuh"
#include "../../metis_b200/csrc/metis_trace.cuh"
#include "../../metis_b200/csrc/metis_rows.cuh"

#ifndef HOSTSIM_MAXS
#define HOSTSIM_MAXS METIS_MAX_STAGES
#endif
#ifndef HOSTSIM_MAXL
#define HOSTSIM_MAXL METIS_MAX_LAYERS
#endif
#ifndef HOSTSIM_ONE
#define HOSTSIM_ONE 0
#endif

using namespace metis;

namespace {

constexpr int kS = HOSTSIM_MAXS, kL = HOSTSIM_MAXL;
constexpr bool kOne = HOSTSIM_ONE != 0;
static_assert(kS <= METIS_MAX_STAGES && kL <= METIS_MAX_LAYERS, "tier beyond the compiled limits");

// `with_rsum`: the range-sum tables of the search kernels (filled by the same fill_range_sums); without them the
// evaluator adds the slices up, like the replay / trace kernels do
Tables host_tables(const MetisProblem &p, std::vector<double> &dlay, bool with_rsum = false) {
    Tables T;
    T.p = p;
    T.rsum = nullptr;
    if (with_rsum) {
        static thread_local std::vector<double> rs;
        const int L = p.num_layers;
        const size_t n = (size_t)L + 1;
        rs.assign((size_t)range_sum_tables(p) * n * n, -1.0);
        for (int t = 0; t < range_sum_tables(p); ++t) {
            const double *row = range_sum_row(p, t, p.layer_memory, p.layer_compute, p.norm_lc);
            if (!row) continue;
            for (int a = 0; a < L; ++a) fill_range_sums(row, L, a, rs.data() + (size_t)t * n * n);
        }
        T.rsum = rs.data();
    }
    T.key_index = p.key_index;
    T.lc = p.layer_compute;
    T.mem = p.layer_memory;
    T.exec_full = p.exec_full;
    T.fb_sync = p.fb_sync;
    T.norm_lc = p.norm_lc;
    const DerivedLayout d = derived_layout(p);
    dlay.resize(d.total);
    for (int i = 0; i < d.total; ++i) dlay[i] = derive_entry(p, d, p.norm_lc, p.exec_full, p.type_bw_first, i);
    T.type_memory = p.type_memory;
    T.bw_first = p.type_bw_first;
    T.bw_min = p.type_bw_min;
    T.run_type = p.ns_run_type;
    T.run_end = p.ns_run_end;
    T.q10_end = p.ns_q10_end;
    bind_derived(T, dlay.data());
    return T;
}

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

struct HostSink {
    MetisRecord *records;
    int64_t capacity;
    uint8_t *detail;
    int stride;
    MetisSearchSummary *sum;
    void phase(int) {}
    void partition_call() { ++sum->num_partition_calls; }
    void balancer_run() { ++sum->num_balancer_runs; }
    void keyerror() { ++sum->num_keyerror; }
    void fatal(uint32_t ordinal, int code, uint32_t aux) {
        if ((uint64_t)ordinal < sum->fatal_ordinal) {
            sum->fatal_ordinal = ordinal;
            sum->fatal_code = (uint32_t)code;
            sum->fatal_aux = aux;
        }
    }
    void emit(const PlanDesc &pd, int step, int nrep, double cost, const uint8_t *tpc, const uint16_t *part) {
        const int64_t slot = (int64_t)sum->num_records++;
        if (slot < capacity) {
            MetisRecord r;
            r.cost = cost; r.ordinal = pd.ordinal; r.step = (uint16_t)step;
            r.num_repartition = (uint8_t)nrep; r.num_stage = (uint8_t)pd.S;
            records[slot] = r;
            if (detail) {
                uint8_t *d = detail + (size_t)slot * stride;
                for (int s = 0; s < pd.S; ++s) { d[s] = (uint8_t)(pd.row[s] - tpc[s]); d[pd.S + s] = tpc[s]; }
                for (int s = 0; s <= pd.S; ++s) d[2 * pd.S + s] = (uint8_t)part[s];
            }
        }
        MetisRecord &b = sum->best;
        if (cost < b.cost || (cost == b.cost && (pd.ordinal < b.ordinal || (pd.ordinal == b.ordinal && step < b.step)))) {
            b.cost = cost; b.ordinal = pd.ordinal; b.step = (uint16_t)step;
            b.num_repartition = (uint8_t)nrep; b.num_stage = (uint8_t)pd.S;
        }
    }
};

// the host policies with a record of the balancer paths taken (bit p of *notes = BalancerPath p, metis_eval.cuh)
struct NoteSerial : Serial {
    unsigned *notes;
    void note(int p) const { *notes |= 1u << p; }
};
struct NoteLane : OneLane {
    unsigned *notes;
    void note(int p) const { *notes |= 1u << p; }
};
// found by argument-dependent lookup ahead of the generic template: keeps OneLane's reverse order of PAR iterations
int par_index(const NoteLane &x, int i, int n) { return x.reverse ? n - 1 - i : i; }

}  // namespace

extern "C" {

// the instantiation this build was compiled for: MAXS | MAXL << 16 | ONE << 32 (MetisSearchSummary.reserved[2])
uint64_t hostsim_instantiation() { return (uint64_t)kS | (uint64_t)kL << 16 | (uint64_t)kOne << 32; }

int hostsim_het_search(const MetisProblem *p, const MetisPlanSpace *sp, const MetisShard *sh, MetisRecord *records,
                       int64_t capacity, uint8_t *detail, int32_t stride, MetisSearchSummary *summary, int32_t mode) {
    // a problem outside this instantiation's scratch or type specialisation is never given to it by the dispatch
    if (sp->max_stage > kS || p->num_layers > kL || (kOne && p->num_types != 1)) return -1;
    std::vector<double> dlay;
    const Tables T = host_tables(*p, dlay, mode != 0);
    memset(summary, 0, sizeof(*summary));
    summary->fatal_ordinal = ~0ULL;
    summary->best.cost = INFINITY;
    summary->best.ordinal = 0xFFFFFFFFu;
    summary->best.step = 0xFFFF;
    summary->reserved[2] = hostsim_instantiation();
    HostSink sink{records, capacity, detail, stride, summary};
    static thread_local Scratch<kS, kL> w;
    const int64_t tile = sh->tile, world = sh->world;
    const int64_t rounds = (sp->num_plans + tile * world - 1) / (tile * world);
    if (mode == 0) {                      // sequential PlanEvaluator::run (also used by the replay kernel)
        for (int64_t i = 0; i < rounds * tile; ++i) {
            const int64_t ordinal = ((i / tile) * world + sh->rank) * tile + (i % tile);
            PlanDesc pd;
            if (!decode(*sp, ordinal, pd)) continue;
            PlanEvaluator<kS, kL, Serial, kOne> ev(T, w);
            ev.run(pd, sink);
        }
    } else {
        // the search kernel's schedule: mode 1 = first-task round (one plan per thread) + chain evaluator for the
        // plans that continue, from where the first-task round left them; mode 4 = the same, the chain evaluator
        // replaying the first attempt (hand-over store full); mode 2 = chain evaluator for every admitted plan;
        // mode 3 = mode 2 with the iterations of every PAR section visited in reverse order (they must be independent)
        static thread_local CoopMail mail;
        OneLane lanes;
        lanes.reverse = mode == 3;
        for (int64_t i = 0; i < rounds * tile; ++i) {
            const int64_t ordinal = ((i / tile) * world + sh->rank) * tile + (i % tile);
            PlanDesc pd;
            if (!decode(*sp, ordinal, pd)) continue;
            {
                PlanEvaluator<kS, kL, Serial, kOne> probe(T, w);     // admission
                const int ok = probe.begin(pd);
                if (ok < 0) { sink.fatal(pd.ordinal, METIS_FATAL_SCRATCH, 0); continue; }
                if (ok == 0) continue;
            }
            int start = 0;                                    // CoopEvaluator::kFresh
            static thread_local std::vector<double> saved;
            if (mode == 1 || mode == 4) {
                int hint = 0, resume = 1;
                if (!first_task<kS, kL, kOne>(T, w, sink, true, pd, hint, resume)) continue;
                start = resume;
                if (mode == 4 && start == 2) start = 1;       // no room in the hand-over store: replay the attempt
                if (start == 2) saved.assign(w.perf, w.perf + pd.S);
            }
            CoopEvaluator<kS, kL, OneLane, kOne> ev(T, w, mail, lanes);
            ev.run_chain(pd, sink, start, saved.data(), 1);
        }
    }
    return 0;
}

// the device's trace replay (metis_trace.cuh) on the host: lets the CPU suite check the verbose transcript
int hostsim_het_trace(const MetisProblem *p, const MetisPlanSpace *sp, const uint32_t *ordinals, int64_t n,
                      uint64_t *trace, int32_t words) {
    std::vector<double> dlay;
    const Tables T = host_tables(*p, dlay);
    static thread_local Scratch<kS, kL> w;
    for (int64_t i = 0; i < n; ++i) {
        TraceOut out(trace + (size_t)i * words, words);
        PlanDesc pd;
        if (decode(*sp, ordinals[i], pd)) {
            TraceEvaluator<kS, kL> ev(T, w, out);
            ev.run_traced(pd);
        }
        out.finish();
    }
    return 0;
}

// the row generator of SURVEY.md 8(f)-1 (metis_rows.cuh) on the host, composition by composition
int hostsim_generate_rows(const MetisCompRec *recs, int64_t ncomp, const uint8_t *pool, uint8_t *rows) {
    for (int64_t c = 0; c < ncomp; ++c) write_composition_rows(recs[c], pool, rows);
    return 0;
}

// developer statistics: LayerComputeBalancer runs per inter-stage plan (0 = plan without a valid strategy)
int hostsim_runs_per_plan(const MetisProblem *p, const MetisPlanSpace *sp, int32_t *runs_out, int32_t *hints_out) {
    std::vector<double> dlay;
    const Tables T = host_tables(*p, dlay);
    MetisSearchSummary sum;
    memset(&sum, 0, sizeof(sum));
    sum.fatal_ordinal = ~0ULL;
    sum.best.cost = INFINITY;
    HostSink sink{nullptr, 0, nullptr, 0, &sum};
    static thread_local Scratch<kS, kL> w;
    static thread_local CoopMail mail;
    OneLane lanes;
    for (int64_t ordinal = 0; ordinal < sp->num_plans; ++ordinal) {
        PlanDesc pd;
        runs_out[ordinal] = 0;
        if (!decode(*sp, ordinal, pd)) continue;
        PlanEvaluator<kS, kL, Serial, kOne> probe(T, w);
        if (probe.begin(pd) != 1) continue;
        if (hints_out) {                                  // the scheduling hint of the bulk round (-1: plan ends there)
            MetisSearchSummary scratch_sum;
            memset(&scratch_sum, 0, sizeof(scratch_sum));
            scratch_sum.fatal_ordinal = ~0ULL;
            scratch_sum.best.cost = INFINITY;
            HostSink quiet{nullptr, 0, nullptr, 0, &scratch_sum};
            int hint = 0, resume = 1;
            const bool cont = first_task<kS, kL, kOne>(T, w, quiet, true, pd, hint, resume);
            hints_out[ordinal] = cont ? hint : -1;
        }
        const uint64_t before = sum.num_balancer_runs;
        CoopEvaluator<kS, kL, OneLane, kOne> ev(T, w, mail, lanes);
        ev.run_chain(pd, sink, false);
        runs_out[ordinal] = (int32_t)(sum.num_balancer_runs - before);
    }
    return 0;
}

int hostsim_homo_cost(const MetisProblem *p, int32_t type_id, const int32_t *plans, int64_t n, double *cost,
                      int32_t *status) {
    std::vector<double> dlay;
    const Tables T = host_tables(*p, dlay);
    for (int64_t i = 0; i < n; ++i) {
        const int32_t *q = plans + i * 5;
        double c = 0.0;
        int oom = 0;
        const int rc = homo_cost(T, type_id, q[0], q[1], q[2], q[3], q[4], c, oom);
        cost[i] = rc ? NAN : c;
        status[i] = rc ? 1 : (oom ? 2 : 0);
    }
    return 0;
}

int hostsim_layer_balance(const double *capa, const int32_t *num_stage, int64_t n, int32_t stride, const double *lc,
                          int32_t norm_len, int32_t num_layers, uint16_t *partition) {
    if (num_layers > kL) return -1;
    for (int64_t i = 0; i < n; ++i)
        if (num_stage[i] > kS) return -1;
    std::vector<double> dlay(norm_len);
    for (int r = 0; r < norm_len; ++r) dlay[r] = lc[r] / 7.0;
    Tables T;
    memset(&T, 0, sizeof(T));
    T.p.num_layers = num_layers;
    T.p.norm_len = norm_len;
    T.norm_lc = lc;
    T.dlay = dlay.data();
    static thread_local Scratch<kS, kL> w;
    for (int64_t i = 0; i < n; ++i) {
        const int S = num_stage[i];
        uint16_t *out = partition + i * (stride + 1);
        for (int s = 0; s < S; ++s) w.perf[s] = capa[i * stride + s];
        const int rc = balance_run<kS, kL>(T, S, w, Serial());
        if (rc) { out[0] = 0xFFFF; continue; }
        for (int s = 0; s <= S; ++s) out[s] = w.part[s];
    }
    return 0;
}

// One balancer form over n rows, like tests/devsim's devsim_balance: policy 0 = balance_run (Serial), 1 = balance_coop
// (OneLane), 2 = balance_coop visiting the PAR iterations in reverse.  The tables are derived from a minimal problem
// (no keys, batch sizes or tp) by derive_entry, so the predictor of the forward pass sees the bits a search gives it.
// Per row: partition, METIS_FATAL_* code, BalancerPath bits and the middle block's length (coop; -1 for Serial).
int hostsim_balance(int32_t policy, const double *capa, const int32_t *num_stage, int64_t n, int32_t stride,
                    const double *lc, int32_t norm_len, int32_t num_layers, uint16_t *partition, int32_t *rc,
                    uint32_t *notes, int32_t *block) {
    if (policy < 0 || policy > 2 || num_layers > kL) return -1;
    for (int64_t i = 0; i < n; ++i)
        if (num_stage[i] < 1 || num_stage[i] > kS || num_stage[i] > stride) return -1;
    MetisProblem p;
    memset(&p, 0, sizeof(p));
    p.num_layers = num_layers;
    p.norm_len = norm_len;
    const double bw[1] = {1.0};
    const DerivedLayout d = derived_layout(p);
    std::vector<double> derived(d.total + 1);
    for (int i = 0; i < d.total; ++i) derived[i] = derive_entry(p, d, lc, nullptr, bw, i);
    Tables T;
    memset(&T, 0, sizeof(T));
    T.p = p;
    T.norm_lc = lc;
    bind_derived(T, derived.data());
    static thread_local Scratch<kS, kL> w;
    static thread_local CoopMail mail;
    for (int64_t i = 0; i < n; ++i) {
        const int S = num_stage[i];
        for (int s = 0; s < S; ++s) w.perf[s] = capa[i * stride + s];
        unsigned got = 0;
        int r, blk = -1;
        if (policy == 0) {
            NoteSerial x;
            x.notes = &got;
            r = balance_run<kS, kL>(T, S, w, x);
        } else {
            NoteLane x;
            x.notes = &got;
            x.reverse = policy == 2;
            CoopEvaluator<kS, kL, NoteLane> ev(T, w, mail, x);
            ev.pd.S = S;
            r = ev.balance_coop();
            if (!r) blk = mail.m > mail.k ? mail.m - mail.k : 0;
        }
        rc[i] = r;
        notes[i] = got;
        block[i] = blk;
        if (!r)
            for (int s = 0; s <= S; ++s) partition[i * (stride + 1) + s] = w.part[s];
    }
    return 0;
}

}  // extern "C"
