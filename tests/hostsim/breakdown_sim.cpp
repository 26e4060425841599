// breakdown_sim.cpp - TEST-ONLY host build of the cost breakdown (BreakdownEvaluator and homo_breakdown of
// metis_b200/csrc/metis_trace.cuh), so that the CPU suite checks the code metis_het_breakdown / metis_homo_breakdown run.
// It is hostsim.cpp (the host build of the device evaluator, whose table and plan decoding it reuses) plus the two
// entry points below; built and loaded only by tests/test_breakdown.py, with hostsim.cpp's flags.
#include "hostsim.cpp"

extern "C" {

// metis_het_breakdown on the host: picks sorted by (ordinal, step), every run of equal ordinals replayed once
int breakdown_sim_het(const MetisProblem *p, const MetisPlanSpace *sp, const MetisRecord *picks, int64_t n,
                      MetisBreakdown *out, double *stage_out, int32_t stride) {
    std::vector<double> dlay;
    const Tables T = host_tables(*p, dlay);
    static thread_local Scratch<kS, kL> w;
    for (int64_t i = 0; i < n;) {
        int64_t end = i + 1;
        while (end < n && picks[end].ordinal == picks[i].ordinal) ++end;
        BreakdownEvaluator<kS, kL> ev(T, w, picks, i, end, out, stage_out, stride);
        for (int64_t k = i; k < end; ++k) ev.clear(k);
        PlanDesc pd;
        if (decode(*sp, picks[i].ordinal, pd)) ev.replay(pd);
        i = end;
    }
    return 0;
}

// metis_homo_breakdown on the host
int breakdown_sim_homo(const MetisProblem *p, int32_t type_id, const int32_t *plans, int64_t n, double *terms,
                       double *stage_memory, int32_t stride, int32_t *status) {
    std::vector<double> dlay;
    const Tables T = host_tables(*p, dlay);
    for (int64_t i = 0; i < n; ++i)
        status[i] = homo_breakdown(T, type_id, plans + i * 5, terms + i * 6, stage_memory + i * stride, stride);
    return 0;
}

}  // extern "C"
