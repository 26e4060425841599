// headroom_sim.cpp - TEST-ONLY host build of the search with per-record headroom (metis_het_search_headroom): the
// evaluators of hostsim.cpp, unchanged, driven by a sink that reads the evaluator's Scratch::mstate at each emit the
// way DeviceSink does (metis_b200/csrc/metis_search.cu).  Built and loaded only by tests/test_headroom.py, with
// hostsim.cpp's flags.
#include "hostsim.cpp"

namespace {

struct HeadroomSink : HostSink {
    const double *state;             // the evaluator's Scratch::mstate
    double *headroom;                // aligned with records
    void emit(const PlanDesc &pd, int step, int nrep, double cost, const uint8_t *tpc, const uint16_t *part) {
        const int64_t slot = (int64_t)sum->num_records;
        HostSink::emit(pd, step, nrep, cost, tpc, part);
        if (slot < capacity) {
            double m = state[0];
            for (int s = 1; s < pd.S; ++s)
                if (state[s] < m) m = state[s];
            headroom[slot] = m;
        }
    }
};

}  // namespace

extern "C" {

// hostsim_het_search's schedules (mode 0 sequential, 1 first task then chain, 2 chain only) with the headroom sink
int headroom_sim_search(const MetisProblem *p, const MetisPlanSpace *sp, MetisRecord *records, double *headroom,
                        int64_t capacity, MetisSearchSummary *summary, int32_t mode) {
    if (sp->max_stage > kS || p->num_layers > kL || (kOne && p->num_types != 1) || mode < 0 || mode > 2) return -1;
    std::vector<double> dlay;
    const Tables T = host_tables(*p, dlay, mode != 0);
    memset(summary, 0, sizeof(*summary));
    summary->fatal_ordinal = ~0ULL;
    summary->best.cost = INFINITY;
    summary->best.ordinal = 0xFFFFFFFFu;
    summary->best.step = 0xFFFF;
    static thread_local Scratch<kS, kL> w;
    static thread_local CoopMail mail;
    HeadroomSink sink;
    sink.records = records; sink.capacity = capacity; sink.detail = nullptr; sink.stride = 0; sink.sum = summary;
    sink.state = w.mstate; sink.headroom = headroom;
    OneLane lanes;
    static thread_local std::vector<double> saved;
    for (int64_t ordinal = 0; ordinal < sp->num_plans; ++ordinal) {
        PlanDesc pd;
        if (!decode(*sp, ordinal, pd)) continue;
        if (mode == 0) {
            PlanEvaluator<kS, kL, Serial, kOne> ev(T, w);
            ev.run(pd, sink);
            continue;
        }
        {
            PlanEvaluator<kS, kL, Serial, kOne> probe(T, w);
            const int ok = probe.begin(pd);
            if (ok < 0) { sink.fatal(pd.ordinal, METIS_FATAL_SCRATCH, 0); continue; }
            if (ok == 0) continue;
        }
        int start = 0;
        if (mode == 1) {
            int hint = 0, resume = 1;
            if (!first_task<kS, kL, kOne>(T, w, sink, true, pd, hint, resume)) continue;
            start = resume;
            if (start == 2) saved.assign(w.perf, w.perf + pd.S);
        }
        CoopEvaluator<kS, kL, OneLane, kOne> ev(T, w, mail, lanes);
        ev.run_chain(pd, sink, start, saved.data(), 1);
    }
    return 0;
}

}  // extern "C"
