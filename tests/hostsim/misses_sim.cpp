// misses_sim.cpp - TEST-ONLY host build of the search with its out-of-memory partition attempts
// (metis_het_search_outputs): the evaluators of hostsim.cpp, unchanged, driven by a sink with the miss hook of
// MissSink (metis_b200/csrc/metis_search.cu).  Built and loaded only by tests/test_misses.py, with hostsim.cpp's flags.
#include "hostsim.cpp"

namespace {

struct MissHostSink : HostSink {
    static constexpr bool kMisses = true;
    MetisMiss *misses;
    int64_t miss_capacity;
    int call = 0;                    // set by the evaluators
    void miss(const PlanDesc &pd, int attempt, double deficit, int stage) {
        const int64_t slot = (int64_t)sum->reserved[3]++;
        if (slot < miss_capacity) {
            MetisMiss r;
            r.deficit = deficit; r.ordinal = pd.ordinal; r.key = (uint16_t)((call << 2) | attempt);
            r.stage = (uint8_t)stage; r.num_stage = (uint8_t)pd.S;
            misses[slot] = r;
        }
    }
};

}  // namespace

extern "C" {

// hostsim_het_search's schedules (mode 0 sequential, 1 first task then chain, 2 chain only, 3 chain only with the
// PAR sections reversed, 4 first task then chain replaying the first attempt) with the miss sink
int misses_sim_search(const MetisProblem *p, const MetisPlanSpace *sp, MetisRecord *records, int64_t capacity,
                      MetisMiss *misses, int64_t miss_capacity, MetisSearchSummary *summary, int32_t mode) {
    if (sp->max_stage > kS || p->num_layers > kL || (kOne && p->num_types != 1) || mode < 0 || mode > 4) return -1;
    std::vector<double> dlay;
    const Tables T = host_tables(*p, dlay, mode != 0);
    memset(summary, 0, sizeof(*summary));
    summary->fatal_ordinal = ~0ULL;
    summary->best.cost = INFINITY;
    summary->best.ordinal = 0xFFFFFFFFu;
    summary->best.step = 0xFFFF;
    static thread_local Scratch<kS, kL> w;
    static thread_local CoopMail mail;
    MissHostSink sink;
    sink.records = records; sink.capacity = capacity; sink.detail = nullptr; sink.stride = 0; sink.sum = summary;
    sink.misses = misses; sink.miss_capacity = miss_capacity;
    OneLane lanes;
    lanes.reverse = mode == 3;
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
        if (mode == 1 || mode == 4) {
            int hint = 0, resume = 1;
            if (!first_task<kS, kL, kOne>(T, w, sink, true, pd, hint, resume)) continue;
            start = resume;
            if (mode == 4 && start == 2) start = 1;           // no room in the hand-over store: replay the attempt
            if (start == 2) saved.assign(w.perf, w.perf + pd.S);
        }
        CoopEvaluator<kS, kL, OneLane, kOne> ev(T, w, mail, lanes);
        ev.run_chain(pd, sink, start, saved.data(), 1);
    }
    return 0;
}

}  // extern "C"
