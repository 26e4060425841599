// metis_noise.cuh - the seeded profile samples and the per-candidate statistics of the profile-noise what-if
// (metis_het_profile_noise_* in metis_noise.cu; the test-only host build in tests/hostsim/noise_sim.cpp).
//
// Sample j of a profile is search.noisy_profile(profile, sigma, seed, j): every entry of a key's layer-computes
// (field 1) and memory (field 2) lists and its fb_sync (field 3) multiplied by its own factor
//   f = 1.0 + s * (2.0 * u - 1.0),   u = ((r0 << 32 | r1) >> 11) * 2^-53,
// (r0, r1, r2, r3) = Philox4x32-10 (Salmon et al., SC'11, the Random123 constants) of the counter
// (j, index in the list (0 for fb_sync), bs, field << 16 | type << 8 | log2(tp)) under the key (seed lo, seed hi),
// `type` the 1-based position of the device type in utils.DeviceType.  Every step is one IEEE double operation rounded
// to nearest, written with the _rn intrinsics on the device so that no contraction to DFMA can happen.  exec_full, the
// CPython sum of a key's layer-computes, is re-summed with PySum (metis_eval.cuh), the compensated sum CPython 3.12
// runs on a list of floats.  Plain C++, like metis_eval.cuh.
#pragma once

#include "metis_eval.cuh"

namespace metis {

enum NoiseField { kNoiseCompute = 1, kNoiseMemory = 2, kNoiseFbSync = 3 };

#if defined(__CUDA_ARCH__)
MB_HD double noise_mul(double a, double b) { return __dmul_rn(a, b); }
MB_HD double noise_add(double a, double b) { return __dadd_rn(a, b); }
MB_HD double noise_sub(double a, double b) { return __dsub_rn(a, b); }
MB_HD double noise_div(double a, double b) { return __ddiv_rn(a, b); }
MB_HD uint32_t mulhi32(uint32_t a, uint32_t b) { return __umulhi(a, b); }
#else
MB_HD double noise_mul(double a, double b) { return a * b; }
MB_HD double noise_add(double a, double b) { return a + b; }
MB_HD double noise_sub(double a, double b) { return a - b; }
MB_HD double noise_div(double a, double b) { return a / b; }
MB_HD uint32_t mulhi32(uint32_t a, uint32_t b) { return (uint32_t)(((uint64_t)a * b) >> 32); }
#endif

struct Philox4 {
    uint32_t v[4];
};

// Philox4x32-10 of counter `c` under key (k0, k1)
MB_HD Philox4 philox4x32_10(Philox4 c, uint32_t k0, uint32_t k1) {
    for (int r = 0; r < 10; ++r) {
        if (r) {
            k0 += 0x9E3779B9u;
            k1 += 0xBB67AE85u;
        }
        const uint32_t lo0 = 0xD2511F53u * c.v[0], hi0 = mulhi32(0xD2511F53u, c.v[0]);
        const uint32_t lo1 = 0xCD9E8D57u * c.v[2], hi1 = mulhi32(0xCD9E8D57u, c.v[2]);
        c = Philox4{{hi1 ^ c.v[1] ^ k0, lo1, hi0 ^ c.v[3] ^ k1, lo0}};
    }
    return c;
}

// The factor of one value of sample j: `s` the sigma of its field and device type (> 0), `type` the device type's
// 1-based utils.DeviceType position, `tpl` log2 of its tp
MB_HD double noise_factor(double s, uint64_t seed, uint32_t j, uint32_t index, uint32_t bs, int field, int type,
                          int tpl) {
    const Philox4 r = philox4x32_10(Philox4{{j, index, bs, (uint32_t)(field << 16 | type << 8 | tpl)}},
                                    (uint32_t)seed, (uint32_t)(seed >> 32));
    const uint64_t bits = ((uint64_t)r.v[0] << 32 | r.v[1]) >> 11;
    const double u = noise_mul((double)bits, 0x1.0p-53);
    return noise_add(1.0, noise_mul(s, noise_sub(noise_mul(2.0, u), 1.0)));
}

// Where one profile key lives: its device type (problem order), log2(tp) and bs; packed by key_meta_kernel
MB_HD uint32_t pack_key_meta(int ti, int tpl, int bs) { return (uint32_t)ti | (uint32_t)tpl << 8 | (uint32_t)bs << 16; }

// One value of a sample's layer_compute / layer_memory row (field 1 / 2) or fb_sync (field 3, index 0): `v` scaled by
// its factor, or `v` itself when the field's sigma for the key's type is 0
MB_HD double noisy_value(double v, const double *sigma_of_field, const uint8_t *type_code, uint64_t seed, uint32_t j,
                         uint32_t meta, int field, uint32_t index) {
    const int ti = meta & 0xff;
    const double s = sigma_of_field[ti];
    if (s == 0.0) return v;
    return noise_mul(v, noise_factor(s, seed, j, index, meta >> 16, field, type_code[ti], (meta >> 8) & 0xff));
}

// exec_full of a sample's key: its layer_compute row (lpad entries; the zero padding adds nothing) summed as CPython
// sums the list
MB_HD double noisy_exec_full(const double *row, int lpad) {
    PySum s;
    for (int l = 0; l < lpad; ++l) s.add(row[l]);
    return s.result();
}

// Sample j's norm_lc, the balancer's layer weights (load_balancer.py:22-27, quirk Q3) under noisy_profile: `row` the
// n layer-computes of the profile's first-listed entry's tp1_bs1 (device type `type`, 1-based utils.DeviceType
// position, layer-computes sigma `s` > 0), each multiplied by its factor (tp 1, bs 1, field 1), then each product divided
// by their CPython sum.  Returns false, with `out` holding the products, when that sum is 0: the reference's
// ZeroDivisionError.
MB_HD bool noisy_norm(const double *row, int n, double s, uint64_t seed, uint32_t j, int type, double *out) {
    PySum total;
    for (int i = 0; i < n; ++i) {
        out[i] = noise_mul(row[i], noise_factor(s, seed, j, (uint32_t)i, 1, kNoiseCompute, type, 0));
        total.add(out[i]);
    }
    const double t = total.result();
    if (t == 0.0) return false;
    for (int i = 0; i < n; ++i) out[i] = noise_div(out[i], t);
    return true;
}

// The running per-candidate statistics of one sample: `u` whether the candidate is usable, `c` its cost, `is_best`
// whether it is the sample's best, `best_cost` the sample's best cost, `t` = 1.0 + within
MB_HD void noise_accumulate(bool u, double c, bool is_best, double best_cost, double t, int32_t &wins, int32_t &near,
                            int32_t &usable, double &regret, double &sum) {
    if (is_best) ++wins;
    if (!u) {
        regret = (double)INFINITY;
        return;
    }
    ++usable;
    sum = noise_add(sum, c);
    if (c <= noise_mul(best_cost, t)) ++near;
    const double d = noise_sub(c, best_cost);
    if (d > regret) regret = d;
}

}  // namespace metis
