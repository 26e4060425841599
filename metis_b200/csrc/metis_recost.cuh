// metis_recost.cuh - HeteroCostEstimator.get_cost of costed candidates under other bandwidth tables
// (metis_het_recost in metis_recost.cu; the test-only host build in tests/hostsim/recost_sim.cpp).
//
// Bandwidth is read only by the cost model (model/cost_estimator.py:205-232 through cluster_bandwidth.py:135-195):
// the balancer, the memory test and the strategy chain never read it, so a search under other bandwidths visits the
// same candidates with the same strategies and partitions.  A candidate is therefore re-costed from its detail row,
// without a balancer run.  The evaluator splits get_cost (metis_eval.cuh) into the part no bandwidth enters (stage
// times and their sum, max_len, fb_sync, the update term, batch_generate), computed once per candidate, and the pp and
// dp terms, computed per scenario by the same stage_terms member get_cost calls.  Plain C++, like metis_eval.cuh.
#pragma once

#include "metis_eval.cuh"

namespace metis {

template <int MAXS, int MAXL>
struct RecostEvaluator : PlanEvaluator<MAXS, MAXL> {
    using Base = PlanEvaluator<MAXS, MAXL>;
    int nstage;
    double exec, fb_sync, max_upd, bg;

    // For the bandwidth what-if (metis_het_recost), `t` must read its bandwidths through the general path
    // (t.p.uniform_bw == 0): its bw_first / bw_min hold the scenario when scenario_cost is called.  The profile
    // what-ifs (het_profile_kernel, metis_profile.cu) bind `t` to a whole scenario's tables, derived bandwidth tables
    // included.
    MB_HD RecostEvaluator(const Tables &t, Scratch<MAXS, MAXL> &s) : Base(t, s), nstage(0), exec(0), fb_sync(0), max_upd(0), bg(0) {}

    // The candidate: plan `plan` with the strategies and partition of its detail row (dp codes[S], tp codes[S],
    // partition[S+1]); then the bandwidth-independent terms.  Returns 0, or 1 when get_cost raises a KeyError.
    MB_HD int load(const PlanDesc &plan, const uint8_t *detail) {
        this->pd = plan;
        this->bs_total = this->T.p.gbs / plan.batches;
        const int S = plan.S;
        int a = 0;
        for (int s = 0; s < S; ++s) {
            this->w.gcode[s] = plan.row[s];
            this->w.tpc[s] = detail[S + s];
            this->w.rs[s] = (uint16_t)a;
            a += 1 << plan.row[s];
        }
        this->w.rs[S] = (uint16_t)a;
        for (int s = 0; s <= S; ++s) this->w.part[s] = detail[2 * S + s];
        return fixed_terms();
    }

    // get_cost (metis_eval.cuh) up to the terms bandwidth enters, in the same order
    MB_HD int fixed_terms() {
        const Tables &T = this->T;
        const PlanDesc &pd = this->pd;
        const bool one_type = T.p.num_types == 1;
        nstage = pd.label < pd.S ? pd.label : pd.S;
        if (T.p.q10_devices < T.p.total_devices && this->rank_start(nstage) > T.p.q10_devices) return 1;
        bool bad = false;
        PySum lens_sum;
        double max_len = -INFINITY;
        for (int s = 0; s < nstage; ++s) {
            double len;
            if (this->stage_time(s, len)) bad = true;
            lens_sum.add(len);
            if (len > max_len) max_len = len;
        }
        if (bad) return 1;
        max_upd = -INFINITY;
        for (int s = 0; s < nstage; ++s) {                   // the update term: stage_terms' upd reads no bandwidth
            double pp, dpc, upd;
            this->stage_terms(s, nstage, pp, dpc, upd);
            if (upd > max_upd) max_upd = upd;
        }
        const int s = nstage - 1;
        const int a = one_type ? 0 : this->rank_start(s), b = a + this->group(s);
        double v;
        if (this->fb_sync_cost(a, b, this->w.tpc[s], this->bs_total >> (this->w.gcode[s] - this->w.tpc[s]), v)) return 1;
        fb_sync = v * (double)pd.batches;
        exec = ((double)(pd.batches - 1) * max_len) + lens_sum.result();
        bg = T.p.batch_generator * (double)pd.batches;
        return 0;
    }

    // the cost under the bandwidths T holds now: get_cost's pp and dp terms, then its sum, left to right
    MB_HD double scenario_cost() const {
        double max_dp = -INFINITY, pp_cost = 0.;
        for (int s = 0; s < nstage; ++s) {
            double pp, dpc, upd;
            this->stage_terms(s, nstage, pp, dpc, upd);
            if (s < nstage - 1) pp_cost += pp;
            if (dpc > max_dp) max_dp = dpc;
        }
        return exec + fb_sync + max_upd + max_dp + pp_cost + bg;
    }
};

// One candidate of the profile what-ifs (het_profile_kernel, metis_profile.cu) under the tables `ev` is bound to:
// `cost` get_cost (NaN when it raises), `headroom` the least memory state over every stage, lowest first like the
// search's headroom (NaN when a stage's demand raises); returns the status cost code | memory code << 4, the memory
// code that of the first stage that raises.
template <int MAXS, int MAXL>
MB_HD uint8_t profile_candidate(RecostEvaluator<MAXS, MAXL> &ev, const PlanDesc &pd, const uint8_t *detail,
                                double &cost, double &headroom) {
    const int cost_code = ev.load(pd, detail) == 0 ? METIS_FATAL_NONE : METIS_FATAL_KEY_EXEC;
    cost = cost_code == METIS_FATAL_NONE ? ev.scenario_cost() : (double)NAN;
    int mem_code = METIS_FATAL_NONE;
    double m = 0.0;
    for (int s = 0; s < pd.S; ++s) {
        double demand, state;
        const int rc = ev.stage_memory(s, demand, state);
        if (rc && mem_code == METIS_FATAL_NONE) mem_code = rc;
        if (s == 0 || state < m) m = state;
    }
    headroom = mem_code == METIS_FATAL_NONE ? m : (double)NAN;
    return (uint8_t)(cost_code | mem_code << 4);
}

}  // namespace metis
