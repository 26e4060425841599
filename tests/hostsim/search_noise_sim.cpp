// search_noise_sim.cpp - TEST-ONLY host build of the search what-if's draw (metis_het_search_noise_draw): noise_sim.cpp's
// draw of the profile tables plus noise_norm_kernel's norm_lc (noisy_norm, metis_noise.cuh), so that the CPU suite
// checks the code the kernels run.  Built and loaded only by tests/test_search_noise.py, with hostsim.cpp's flags.
#include "noise_sim.cpp"

extern "C" {

// Sample spec->first + s of `base` (host pointers) with its norm_lc [base->norm_len] from the source row (`norm_row`,
// its device type code and layer-computes sigma); *zero = 1 where the noisy norm total is 0 (norm_lc is then the base's)
int search_noise_sim_draw(const MetisProblem *base, const MetisNoiseSpec *spec, const double *norm_row, int32_t norm_code,
                          double norm_sigma, int32_t s, double *lc, double *lm, double *ef, double *fb, double *norm,
                          int32_t *zero) {
    noise_sim_draw(base, spec, s, lc, lm, ef, fb);
    const bool drawn = norm_sigma != 0.0 && noisy_norm(norm_row, base->norm_len, norm_sigma, spec->seed,
                                                       (uint32_t)(spec->first + s), norm_code, norm);
    if (!drawn)
        for (int i = 0; i < base->norm_len; ++i) norm[i] = base->norm_lc[i];
    *zero = norm_sigma != 0.0 && !drawn;
    return 0;
}

}  // extern "C"
