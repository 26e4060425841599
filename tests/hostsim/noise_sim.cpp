// noise_sim.cpp - TEST-ONLY host build of the profile-noise what-if's generator and reduction (metis_noise.cuh, the
// kernels of metis_b200/csrc/metis_noise.cu), so that the CPU suite checks the code the kernels run: Philox4x32-10,
// the samples' flat tables from the base problem (key_meta_kernel, noise_rows_kernel, noise_keys_kernel) and the
// per-sample best and per-candidate statistics (the two atomicMin passes in a given visit order, then
// noise_accumulate).  Built and loaded only by tests/test_profile_noise.py, with hostsim.cpp's flags.
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../metis_b200/csrc/metis_noise.cuh"
#include "../../metis_b200/csrc/metis_query.cuh"

using namespace metis;

extern "C" {

// Philox4x32-10 of n counters (4 words each) under n keys (2 words each)
int noise_sim_philox(const uint32_t *ctr, const uint32_t *key, uint32_t *out, int64_t n) {
    for (int64_t i = 0; i < n; ++i) {
        const Philox4 r = philox4x32_10(Philox4{{ctr[4 * i], ctr[4 * i + 1], ctr[4 * i + 2], ctr[4 * i + 3]}},
                                        key[2 * i], key[2 * i + 1]);
        memcpy(out + 4 * i, r.v, sizeof r.v);
    }
    return 0;
}

// Sample spec->first + s of `base` (host pointers): layer_compute / layer_memory [num_keys][lpad], exec_full and
// fb_sync [num_keys], as the draw kernels write them
int noise_sim_draw(const MetisProblem *base, const MetisNoiseSpec *spec, int32_t s, double *lc, double *lm, double *ef,
                   double *fb) {
    const MetisProblem &b = *base;
    std::vector<uint32_t> meta((size_t)b.num_keys, 0);
    const int per_type = b.num_tp * b.num_bs;
    for (int e = 0; e < b.num_types * per_type; ++e) {
        const int k = b.key_index[e];
        if (k >= 0) meta[(size_t)k] = pack_key_meta(e / per_type, (e % per_type) / b.num_bs, e % b.num_bs + 1);
    }
    const uint32_t j = (uint32_t)(spec->first + s);
    const int64_t row = (int64_t)b.num_keys * b.lpad;
    for (int64_t e = 0; e < row; ++e) {
        const uint32_t m = meta[(size_t)(e / b.lpad)], l = (uint32_t)(e % b.lpad);
        lc[e] = noisy_value(b.layer_compute[e], spec->sigma[0], spec->type_code, spec->seed, j, m, kNoiseCompute, l);
        lm[e] = noisy_value(b.layer_memory[e], spec->sigma[1], spec->type_code, spec->seed, j, m, kNoiseMemory, l);
    }
    for (int k = 0; k < b.num_keys; ++k) {
        const uint32_t m = meta[(size_t)k];
        ef[k] = spec->sigma[0][m & 0xff] == 0.0 ? b.exec_full[k] : noisy_exec_full(lc + (int64_t)k * b.lpad, b.lpad);
        fb[k] = noisy_value(b.fb_sync[k], spec->sigma[2], spec->type_code, spec->seed, j, m, kNoiseFbSync, 0);
    }
    return 0;
}

// metis_het_profile_noise_reduce of one chunk of `count` samples (cost, usable [count][n]): the candidates visited in
// the order `visit` (a permutation of 0 .. n-1) by both passes, as the atomics of the kernels may take them
int noise_sim_reduce(int32_t count, double near_factor, const double *cost, const uint8_t *usable, int64_t n,
                     const int64_t *visit, int64_t *best_pos, double *best_cost, int32_t *wins, int32_t *near,
                     int32_t *usable_count, double *regret, double *sum) {
    for (int s = 0; s < count; ++s) {
        const double *c = cost + (size_t)s * n;
        const uint8_t *u = usable + (size_t)s * n;
        uint64_t key = ~0ULL, first = ~0ULL;
        for (int64_t v = 0; v < n; ++v) {
            const int64_t i = visit[v];
            if (u[i] && cost_order_key(c[i]) < key) key = cost_order_key(c[i]);
        }
        for (int64_t v = 0; v < n; ++v) {
            const int64_t i = visit[v];
            if (u[i] && cost_order_key(c[i]) == key && (uint64_t)i < first) first = (uint64_t)i;
        }
        best_pos[s] = first == ~0ULL ? -1 : (int64_t)first;
        best_cost[s] = first == ~0ULL ? (double)NAN : c[first];
    }
    for (int64_t i = 0; i < n; ++i)
        for (int s = 0; s < count; ++s) {
            const size_t at = (size_t)s * n + i;
            noise_accumulate(usable[at] != 0, cost[at], best_pos[s] == i, best_cost[s], near_factor, wins[i], near[i],
                             usable_count[i], regret[i], sum[i]);
        }
    return 0;
}

}  // extern "C"
