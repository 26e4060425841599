// metis_trace.cuh - replay of single inter-stage plans that RECORDS what the reference prints for every candidate
// (search_space/plan.py:207-218, model/load_balancer.py:92,132-133,143, model/cost_estimator.py:193,201-203,239-240,
// cost_het_cluster.py:43,48): strategies, stage performance, every partition attempt with its memory demand and
// state, the re-weighted performance, the cost terms and which KeyError skipped a candidate.  One thread per plan
// (the sequential PlanEvaluator of metis_eval.cuh, unchanged arithmetic); the host formats the lines
// (metis_b200/verbose.py).  Debug path of the drop-in CLI (METIS_VERBOSE=1), never used by a search.
// Also the cost breakdown of chosen candidates (BreakdownEvaluator, homo_breakdown): the same tap, structured output.
//
// Event stream per plan: 64-bit words.  A header word  tag | n << 8 | aux << 32  is followed by its payload.
#pragma once

#include "metis_eval.cuh"

namespace metis {

enum TraceTag : uint32_t {
    kTrEnd = 0,        //                                   end of the plan's stream
    kTrStrategy = 1,   // n = S, payload ceil(S/8) words     log2(tp) per stage, packed bytes  -> valid_strategies
    kTrPerf = 2,       // n = S, payload S doubles           stage_compute_performance
    kTrAttempt = 3,    // n = S, aux = attempt               layer_partition (S+1 u16, 4 per word), demand[S], state[S]
    kTrAdjust = 4,     // n = S or 0 (None)                  adj_stage_compute_performance (aux = next attempt number)
    kTrResult = 5,     // aux = num_repartition (0 = None)   'layer_partition: ...' of plan.py:218
    kTrSplit = 6,      // n = dp, aux = stage                'data loadbalancer: [...]' (hetero_bs), one int per word
    kTrCost = 7,       // payload 6 doubles                  execution, fb_sync, parameter update, dp, pp, cost
    kTrKeyError = 8,   // aux = site, payload 2 words (a, b) which KeyError skipped the candidate
    kTrFatal = 9,      // aux = METIS_FATAL_*, payload 1 word (aux value): the reference aborts here
    kTrOverflow = 10,  //                                    stream buffer too small
};

// KeyError sites of HeteroCostEstimator.get_cost, in the order the reference reaches them within a stage
enum TraceKeySite : uint32_t {
    kKeyExec = 1,        // key(tp{a}_bs{b}) not found in profile_data          cost_estimator.py:182-183
    kKeySplitProfile = 2,// 'tp{a}_bs1' (dict KeyError inside partition_data)   load_balancer.py:152-153
    kKeySliceTooBig = 3, // batch_size({b}) not found in profile_data           cost_estimator.py:166-167
    kKeySliceProfile = 4,// 'tp{a}_bs{b}' (dict KeyError)                        cost_estimator.py:150
    kKeyFbSync = 5,      // key(fb_sync) not found in profile_data              cost_estimator.py:68-69
    kKeyRank = 6,        // {a} (rank missing in rank_node_map, quirk Q10)      cluster_bandwidth.py:144,181
};

struct TraceOut {
    uint64_t *buf;
    int cap, len;
    bool overflow;
    MB_HD TraceOut(uint64_t *b, int capacity) : buf(b), cap(capacity), len(0), overflow(false) {}
    MB_HD void word(uint64_t v) { if (len < cap - 2) buf[len++] = v; else overflow = true; }
    MB_HD void head(uint32_t tag, uint32_t n, uint32_t aux) { word((uint64_t)tag | ((uint64_t)(n & 0xFFFFFF) << 8) | ((uint64_t)aux << 32)); }
    MB_HD void real(double d) { uint64_t v; memcpy(&v, &d, 8); word(v); }
    MB_HD void finish() {
        if (overflow) { len = 0; buf[len++] = kTrOverflow; }
        buf[len] = kTrEnd;
    }
};

struct NullSink {
    MB_HD void phase(int) {}
    MB_HD void partition_call() {}
    MB_HD void balancer_run() {}
    MB_HD void keyerror() {}
    MB_HD void fatal(uint32_t, int, uint32_t) {}
    MB_HD void emit(const PlanDesc &, int, int, double, const uint8_t *, const uint16_t *) {}
};

template <int MAXS, int MAXL>
struct TraceEvaluator : PlanEvaluator<MAXS, MAXL, Serial, false> {
    using Base = PlanEvaluator<MAXS, MAXL, Serial, false>;
    using Base::T; using Base::w; using Base::pd; using Base::bs_total; using Base::aux;
    TraceOut &out;
    double tap_demand[MAXS], tap_state[MAXS];
    TraceTap tap_store;

    MB_HD TraceEvaluator(const Tables &t, Scratch<MAXS, MAXL> &s, TraceOut &o) : Base(t, s), out(o) {
        tap_store.demand = tap_demand;
        tap_store.state = tap_state;
        this->tap = &tap_store;
    }

    MB_HD void emit_strategy() {
        out.head(kTrStrategy, (uint32_t)pd.S, 0);
        for (int s0 = 0; s0 < pd.S; s0 += 8) {
            uint64_t v = 0;
            for (int k = 0; k < 8 && s0 + k < pd.S; ++k) v |= (uint64_t)w.tpc[s0 + k] << (8 * k);
            out.word(v);
        }
    }
    MB_HD void emit_attempt(int attempt) {
        out.head(kTrAttempt, (uint32_t)pd.S, (uint32_t)attempt);
        for (int s0 = 0; s0 <= pd.S; s0 += 4) {
            uint64_t v = 0;
            for (int k = 0; k < 4 && s0 + k <= pd.S; ++k) v |= (uint64_t)w.part[s0 + k] << (16 * k);
            out.word(v);
        }
        for (int s = 0; s < pd.S; ++s) out.real(tap_demand[s]);
        for (int s = 0; s < pd.S; ++s) out.real(tap_state[s]);
    }

    // HeteroCostEstimator.get_cost stage by stage in the reference's order (cost_estimator.py:208-233): the
    // 'data loadbalancer' lines of mixed-type stages and the FIRST KeyError.  returns true when a KeyError was found
    MB_HD bool walk_cost_messages() {
        const int nstage = pd.label < pd.S ? pd.label : pd.S;
        const int per = T.p.devices_per_node;
        (void)per;
        for (int s = 0; s < nstage; ++s) {
            const int g = w.gcode[s], tpc = w.tpc[s], ldp = g - tpc;
            const int a = this->rank_start(s), b = a + (1 << g);
            const int ta = type_of_rank(T, pd.ns, a), tb = type_of_rank(T, pd.ns, b - 1);
            const int mbs = bs_total >> ldp;
            if (ta == tb) {
                if (key_of(T, ta, tpc, mbs) < 0) return key_error(kKeyExec, 1 << tpc, mbs);
            } else {
                HSplit hs;
                uint32_t dummy = 0;
                if (partition_data(T, pd.ns, a, b - a, 1 << ldp, tpc, bs_total, hs, dummy)) return key_error(kKeySplitProfile, 1 << tpc, 1);
                out.head(kTrSplit, (uint32_t)(1 << ldp), (uint32_t)s);
                for (int r = 0; r < hs.nruns; ++r)
                    for (int i = 0; i < hs.n[r]; ++i) out.word((uint64_t)(hs.base[r] + (i < hs.plus[r] ? 1 : 0)));
                for (int r = 0; r < hs.nruns; ++r)
                    for (int i = 0; i < hs.n[r]; ++i) {          // replicas in order (cost_estimator.py:156-171)
                        const int h = hs.base[r] + (i < hs.plus[r] ? 1 : 0);
                        for (int bit = 30; bit >= 0; --bit) {
                            const int piece = 1 << bit;
                            if (!(h & piece)) continue;
                            if (piece > T.p.max_bs) return key_error(kKeySliceTooBig, 1 << tpc, piece);
                            if (key_of(T, hs.type[r], tpc, piece) < 0) return key_error(kKeySliceProfile, 1 << tpc, piece);
                        }
                    }
            }
            if (s == nstage - 1) {
                for (int r = a; r < b; ++r) {                    // _get_fb_sync_cost over every device of the stage
                    const int key = key_of(T, type_of_rank(T, pd.ns, r), tpc, mbs);
                    if (key < 0 || T.fb_sync[key] == 0.0) return key_error(kKeyFbSync, 0, 0);
                }
            } else {
                const int hi = this->rank_start(s + 2);          // pp group: ranks of stages s and s + 1, ascending
                if (hi > T.p.q10_devices) {
                    const int first = a > T.p.q10_devices ? a : T.p.q10_devices;
                    return key_error(kKeyRank, first, 0);
                }
            }
            {                                                     // dp groups: group d holds ranks a + d + i * dp
                const int dp = 1 << ldp, tp = 1 << tpc;
                if (b > T.p.q10_devices)
                    for (int d = 0; d < dp; ++d)
                        for (int i = 0; i < tp; ++i)
                            if (a + d + i * dp >= T.p.q10_devices) return key_error(kKeyRank, a + d + i * dp, 0);
            }
        }
        return false;
    }
    MB_HD bool key_error(uint32_t site, int a, int b) {
        out.head(kTrKeyError, 2, site);
        out.word((uint64_t)(uint32_t)a);
        out.word((uint64_t)(uint32_t)b);
        return true;
    }
    MB_HD void fatal(int code) {
        out.head(kTrFatal, 1, (uint32_t)code);
        out.word((uint64_t)aux);
    }

    // cost_het_cluster.py:31-48 for one plan, like PlanEvaluator::run, recording every printed value.  The strategy
    // walk itself (including the invalid strategies the reference prints) is replayed by the host from the recorded
    // memory states; the device records only the valid strategies it evaluates.
    MB_HD void run_traced(const PlanDesc &plan) {
        const int ok = this->begin(plan);
        if (ok < 0) { fatal(METIS_FATAL_SCRATCH); return; }
        if (ok == 0) return;
        bool started = false, have_state = false;
        int nrep = 0;
        for (;;) {
            if (nrep == 1) return;                            // plan.py:194-195
            int attempt = 0;
            for (;;) {
                if (!started) started = true;
                else if (!this->next_strategy(have_state)) return;
                if (!this->valid()) continue;
                emit_strategy();
                int rc = this->compute_performance();
                if (rc) { fatal(rc); return; }
                out.head(kTrPerf, (uint32_t)pd.S, 0);
                for (int s = 0; s < pd.S; ++s) out.real(w.perf[s]);
                attempt = 0;
                for (int a = 1; a <= 3; ++a) {                // LayerLoadBalancer.partition_layer (:121-144)
                    rc = balance_run<MAXS, MAXL>(T, pd.S, w, Serial());
                    if (rc) { fatal(rc); return; }
                    // memory_phase re-weights in place; the 3rd failed attempt still calls _adj_compute_performance
                    // in the reference (its result is printed when it is not None), hence attempt numbers below 4
                    const int r = this->memory_phase(a < 3 ? a : 2);
                    if (r < 0) { fatal(-r); return; }
                    emit_attempt(a);
                    if (r == 1) { attempt = a; break; }
                    if (r == 0) { out.head(kTrAdjust, 0, (uint32_t)(a + 1)); break; }
                    out.head(kTrAdjust, (uint32_t)pd.S, (uint32_t)(a + 1));
                    for (int s = 0; s < pd.S; ++s) out.real(w.perf[s]);
                }
                out.head(kTrResult, 0, (uint32_t)attempt);
                have_state = attempt > 0;
                if (attempt > 0) break;
            }
            nrep = attempt;
            if (!walk_cost_messages()) {
                double cost = 0.0;
                if (this->get_cost(cost) == 0) {
                    out.head(kTrCost, 6, 0);
                    for (int k = 0; k < 5; ++k) out.real(tap_store.cost[k]);
                    out.real(cost);
                } else {
                    key_error(kKeyFbSync, 0, 0);               // not reached: walk_cost_messages finds every KeyError first
                }
            }
        }
    }
};

// ---------------------------------------------------------------------------
// Cost breakdown of costed candidates (metis_het_breakdown).  PlanEvaluator::run replays one plan's chain once, up to
// the last requested step, with this evaluator as its own sink.  The tap holds the memory demand and state of the
// last partition attempt and the five printed cost terms; at an emitted step that attempt is the accepted one, and
// the scratch still holds the performance fed to its balancer run, the strategies and the partition.  The per-stage
// cost values come from the same stage_time / stage_terms members get_cost adds up, so they are the same bits.
// ---------------------------------------------------------------------------
template <int MAXS, int MAXL>
struct BreakdownEvaluator : PlanEvaluator<MAXS, MAXL, Serial, false> {
    using Base = PlanEvaluator<MAXS, MAXL, Serial, false>;
    using Base::T; using Base::w;
    double tap_demand[MAXS], tap_state[MAXS];
    TraceTap tap_store;
    const MetisRecord *picks;     // picks[at, end): the requested steps of this plan, ascending
    int64_t at, end;
    MetisBreakdown *out;
    double *stage_out;            // null, or METIS_BD_FIELDS x stride doubles per pick
    int stride;

    MB_HD BreakdownEvaluator(const Tables &t, Scratch<MAXS, MAXL> &s, const MetisRecord *p, int64_t first, int64_t last,
                             MetisBreakdown *o, double *so, int st)
        : Base(t, s), picks(p), at(first), end(last), out(o), stage_out(so), stride(st) {
        tap_store.demand = tap_demand;
        tap_store.state = tap_state;
        this->tap = &tap_store;
    }

    // sink interface of PlanEvaluator::run
    MB_HD void phase(int) {}
    MB_HD void partition_call() {}
    MB_HD void balancer_run() {}
    MB_HD void keyerror() {}
    MB_HD void fatal(uint32_t, int, uint32_t) {}
    MB_HD void emit(const PlanDesc &pd, int step, int, double, const uint8_t *, const uint16_t *) {
        while (at < end && (int)picks[at].step < step) ++at;  // a step the chain never yields keeps its empty row
        for (; at < end && (int)picks[at].step == step; ++at) write(pd, at);
    }

    // every requested row empty first: num_stage 0, NaN everywhere
    MB_HD void clear(int64_t i) {
        MetisBreakdown b;
        for (int k = 0; k < 6; ++k) b.terms[k] = NAN;
        b.min_headroom = NAN;
        b.min_stage = -1; b.costed_stages = 0; b.num_stage = 0; b.reserved = 0;
        out[i] = b;
        if (stage_out)
            for (int k = 0; k < METIS_BD_FIELDS * stride; ++k) stage_out[(size_t)i * METIS_BD_FIELDS * stride + k] = NAN;
    }

    MB_HD void write(const PlanDesc &pd, int64_t i) {
        const int S = pd.S, nstage = pd.label < S ? pd.label : S;
        MetisBreakdown b;
        for (int k = 0; k < 5; ++k) b.terms[k] = tap_store.cost[k];
        b.terms[5] = T.p.batch_generator * (double)pd.batches;   // get_cost's batch generate term
        int lo = 0;
        for (int s = 1; s < S; ++s)
            if (tap_state[s] < tap_state[lo]) lo = s;
        b.min_headroom = tap_state[lo];
        b.min_stage = (int16_t)lo;
        b.costed_stages = (int16_t)nstage;
        b.num_stage = (int16_t)S;
        b.reserved = 0;
        out[i] = b;
        if (!stage_out || S > stride) return;
        double *f = stage_out + (size_t)i * METIS_BD_FIELDS * stride;
        for (int s = 0; s < S; ++s) {
            const int a = this->rank_start(s);
            f[METIS_BD_PERFORMANCE * stride + s] = w.perf[s];
            f[METIS_BD_CAPACITY * stride + s] = this->memory_capacity(a, a + this->group(s));
            f[METIS_BD_DEMAND * stride + s] = tap_demand[s];
            f[METIS_BD_STATE * stride + s] = tap_state[s];
            if (s >= nstage) continue;
            double len, pp, dpc, upd;
            this->stage_time(s, len);
            this->stage_terms(s, nstage, pp, dpc, upd);
            f[METIS_BD_EXEC_TIME * stride + s] = len;
            f[METIS_BD_DP * stride + s] = dpc;
            f[METIS_BD_UPDATE * stride + s] = upd;
            f[METIS_BD_PP * stride + s] = pp;
        }
    }

    // the requested steps of one plan (pd = the plan of picks[at])
    MB_HD void replay(const PlanDesc &pd) {
        this->run(pd, *this, (int)picks[end - 1].step);
    }
};

// HomoCostEstimator.get_cost of one UniformPlan (dp, pp, tp, mbs, gbs) with its breakdown (metis_homo_breakdown):
// terms[6], the per-stage memory sums in mem[0, stride) (NaN past pp); returns the status word of metis_homo_breakdown
MB_HD int homo_breakdown(const Tables &T, int type, const int32_t *q, double *terms, double *mem, int stride) {
    for (int k = 0; k < 6; ++k) terms[k] = NAN;
    for (int s = 0; s < stride; ++s) mem[s] = NAN;
    if (q[1] > stride) return 3;
    TraceTap tap;
    tap.demand = mem;
    tap.state = nullptr;
    double c = 0.0;
    int oom = 0;
    if (homo_cost(T, type, q[0], q[1], q[2], q[3], q[4], c, oom, &tap)) return 1;
    for (int k = 0; k < 5; ++k) terms[k] = tap.cost[k];
    terms[5] = T.p.batch_generator * (double)(q[4] / q[3] / q[0]);   // the batch generate term of homo_cost
    return oom ? 2 : 0;
}

}  // namespace metis
