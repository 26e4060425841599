// profile_recost_sim.cpp - TEST-ONLY host build of the profile what-if (het_profile_recost_kernel of
// metis_b200/csrc/metis_profile.cu), so that the CPU suite checks the code metis_het_profile_recost runs: for every
// scenario, the tables of that scenario's problem, then RecostEvaluator::load + scenario_cost and
// PlanEvaluator::stage_memory over every stage, exactly as the kernel's loop body.  hostsim.cpp (whose table and plan
// decoding it reuses) plus the entry point below.  Built and loaded only by tests/test_profile_recost.py, with
// hostsim.cpp's flags.
#include "hostsim.cpp"
#include "../../metis_b200/csrc/metis_recost.cuh"

extern "C" {

// metis_het_profile_recost on the host: costs / headroom / status [j * n + i] under scenarios[j].  `mutant` != 0
// plants a known defect, so that the tests show they would catch it: 1 memory demand from the stage's own device type
// (METIS_FIX_Q6 set without 'Q6'), 2 the dp / update / batch terms from scenarios[0]'s model section, 3 headroom over
// the costed (label) stages only.
int profile_recost_sim_het(const MetisPlanSpace *sp, const MetisProblem *scenarios, int32_t num_scenarios,
                           const MetisRecord *records, int64_t n, const uint8_t *detail, int32_t stride, double *costs,
                           double *headroom, uint8_t *status, int32_t mutant) {
    static thread_local Scratch<kS, kL> w;
    for (int j = 0; j < num_scenarios; ++j) {
        MetisProblem p = scenarios[j];
        if (mutant == 1) p.corrected |= METIS_FIX_Q6;
        if (mutant == 2) {
            p.optimizer_time = scenarios[0].optimizer_time;
            p.batch_generator = scenarios[0].batch_generator;
            p.input_params = scenarios[0].input_params;
            p.transformer_params = scenarios[0].transformer_params;
            p.output_params = scenarios[0].output_params;
        }
        std::vector<double> dlay;
        const Tables T = host_tables(p, dlay);
        for (int64_t i = 0; i < n; ++i) {
            const size_t at = (size_t)j * n + i;
            PlanDesc pd;
            if (!decode(*sp, records[i].ordinal, pd) || pd.S > kS) {
                costs[at] = headroom[at] = NAN;
                status[at] = (uint8_t)(METIS_FATAL_SCRATCH | METIS_FATAL_SCRATCH << 4);
                continue;
            }
            RecostEvaluator<kS, kL> ev(T, w);
            const int cost_code = ev.load(pd, detail + (size_t)i * stride) == 0 ? METIS_FATAL_NONE : METIS_FATAL_KEY_EXEC;
            costs[at] = cost_code == METIS_FATAL_NONE ? ev.scenario_cost() : NAN;
            int mem_code = METIS_FATAL_NONE;
            double m = 0.0;
            const int S = mutant == 3 && pd.label < pd.S ? pd.label : pd.S;
            for (int s = 0; s < S; ++s) {
                double demand, state;
                const int rc = ev.stage_memory(s, demand, state);
                if (rc && mem_code == METIS_FATAL_NONE) mem_code = rc;
                if (s == 0 || state < m) m = state;
            }
            headroom[at] = mem_code == METIS_FATAL_NONE ? m : NAN;
            status[at] = (uint8_t)(cost_code | mem_code << 4);
        }
    }
    return 0;
}

}  // extern "C"
