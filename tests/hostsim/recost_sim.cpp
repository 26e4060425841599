// recost_sim.cpp - TEST-ONLY host build of the network what-if (RecostEvaluator of metis_b200/csrc/metis_recost.cuh),
// so that the CPU suite checks the code metis_het_recost runs.  It is hostsim.cpp (the host build of the device
// evaluator, whose table and plan decoding it reuses) plus the entry point below, walking the scenarios like
// het_recost_kernel: the bandwidth tables the evaluator reads are overwritten with each scenario in turn.  Built and
// loaded only by tests/test_recost.py, with hostsim.cpp's flags.
#include "hostsim.cpp"
#include "../../metis_b200/csrc/metis_recost.cuh"

extern "C" {

// metis_het_recost on the host: costs[j * n + i], NaN when record i's replay raises a KeyError
int recost_sim_het(const MetisProblem *p, const MetisPlanSpace *sp, const MetisRecord *records, int64_t n,
                   const uint8_t *detail, int32_t stride, const double *bandwidths, int32_t num_scenarios, double *costs) {
    std::vector<double> dlay;
    Tables T = host_tables(*p, dlay);
    const int nt = p->num_types;
    std::vector<double> bw(2 * nt);
    T.p.uniform_bw = 0;
    T.bw_first = bw.data();
    T.bw_min = bw.data() + nt;
    static thread_local Scratch<kS, kL> w;
    for (int64_t i = 0; i < n; ++i) {
        RecostEvaluator<kS, kL> ev(T, w);
        PlanDesc pd;
        bool ok = false;
        for (int j = 0; j < num_scenarios; ++j) {
            for (int t = 0; t < 2 * nt; ++t) bw[t] = bandwidths[(size_t)j * 2 * nt + t];
            if (j == 0) ok = decode(*sp, records[i].ordinal, pd) && pd.S <= kS && ev.load(pd, detail + (size_t)i * stride) == 0;
            costs[(size_t)j * n + i] = ok ? ev.scenario_cost() : NAN;
        }
    }
    return 0;
}

}  // extern "C"
