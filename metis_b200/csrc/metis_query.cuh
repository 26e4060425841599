// metis_query.cuh - plan filters and group keys of searched candidates (metis_query_mark in metis_query.cu; the
// test-only host build in tests/hostsim/query_sim.cpp).
//
// A MetisPlanFilter (include/metis_b200.h) is a set of conditions on one candidate of the reference's estimate_costs
// list: its geometry (node sequence, stage count, batches), its num_repartition and, when asked for, its strategies
// (the tp codes of its detail row).  The filter selects among the candidates the search found; it does not constrain
// the search, whose strategy chain ran unconstrained.  The same function also packs the candidate's group key, the
// mixed-radix digits of the key fields, for the group-best passes.  Plain C++, like metis_eval.cuh.
#pragma once

#include "metis_eval.cuh"

namespace metis {

// What the filter and the keys read of one candidate.
struct QueryPlan {
    int ns;                  // ns_idx
    int S;                   // len(device_groups)
    int div;                 // index into MetisPlanSpace.batches (divisors of gbs, descending)
    int num_div;
    int nrep;                // num_repartition
    const uint8_t *row;      // log2(group size) per stage
    const uint8_t *tpc;      // log2(tp) per stage (the detail row's tp codes), or nullptr when not needed
};

MB_HD bool mask_bit(const uint32_t *mask, int i) { return (mask[i >> 5] >> (i & 31)) & 1u; }

// Does stage s (ranks [lo, hi) of the node sequence's placement) hold a device of a type whose tp limit its tp
// exceeds?  The types of the ranks are the runs of ns_run_type / ns_run_end (model/device_group.py:22-32).
MB_HD bool stage_over_type_limit(const MetisPlanFilter &f, int num_types, const uint8_t *run_type,
                                 const int32_t *run_end, int lo, int hi, int tpc) {
    int start = 0;
    for (int k = 0; k < num_types; ++k) {
        const int end = run_end[k];
        if (end > lo && start < hi && tpc > (int)f.type_tp_code[run_type[k]]) return true;
        start = end;
    }
    return false;
}

// The value of key field `field` (METIS_QUERY_KEY_*) of the plan, as a digit from 0: stage count - 1, batches from the
// smallest, log2 of the largest tp, num_repartition - 1.
MB_HD int key_digit(int field, const QueryPlan &q) {
    switch (field) {
        case METIS_QUERY_KEY_NS: return q.ns;
        case METIS_QUERY_KEY_STAGES: return q.S - 1;
        case METIS_QUERY_KEY_BATCHES: return q.num_div - 1 - q.div;
        case METIS_QUERY_KEY_MAX_TP: {
            int m = 0;
            for (int s = 0; s < q.S; ++s) m = q.tpc[s] > m ? q.tpc[s] : m;
            return m;
        }
        default: return q.nrep - 1;
    }
}

// PlanFilter.admits of one candidate; `group` gets its group (the mixed radix of its key digits, first key most
// significant) or METIS_QUERY_NO_GROUP when it is not admitted or a digit is outside its range.
MB_HD bool query_plan(const MetisPlanFilter &f, int num_types, const uint8_t *ns_run_type, const int32_t *ns_run_end,
                      const QueryPlan &q, uint32_t &group) {
    group = METIS_QUERY_NO_GROUP;
    bool ok = q.S >= f.min_stages && q.S <= f.max_stages && q.nrep <= f.max_repartition && mask_bit(f.ns_mask, q.ns) &&
              mask_bit(f.div_mask, q.div);
    if (ok && f.flags & METIS_QUERY_NEEDS_TP) {
        const uint8_t *run_type = ns_run_type + (size_t)q.ns * num_types;
        const int32_t *run_end = ns_run_end + (size_t)q.ns * num_types;
        const bool by_type = f.flags & METIS_QUERY_BY_TYPE;
        int lo = 0;
        for (int s = 0; s < q.S && ok; ++s) {
            const int t = q.tpc[s], hi = lo + (1 << q.row[s]);
            if (t > f.max_tp_code || (f.uniform_tp && t != q.tpc[0])) ok = false;
            else if (by_type && stage_over_type_limit(f, num_types, run_type, run_end, lo, hi, t)) ok = false;
            lo = hi;
        }
    }
    if (!ok) return false;
    uint32_t g = 0;
    for (int k = 0; k < f.num_keys; ++k) {
        const int d = key_digit(f.key_field[k], q);
        if (d < 0 || d >= f.key_range[k]) return true;      // admitted, in no group (the host sizes the ranges)
        g = g * (uint32_t)f.key_range[k] + (uint32_t)d;
    }
    if (f.num_keys > 0) group = g;
    return true;
}

// An order-preserving 64-bit image of a non-NaN double: a < b iff image(a) < image(b).  -0.0 maps to the image of
// +0.0, as the two compare equal in Python's sort.
MB_HD uint64_t cost_order_key(double x) {
    if (x == 0.0) x = 0.0;
    uint64_t u;
    memcpy(&u, &x, sizeof u);
    return (u >> 63) ? ~u : u | (1ULL << 63);
}

MB_HD double cost_from_order_key(uint64_t k) {
    const uint64_t u = (k >> 63) ? k & ~(1ULL << 63) : ~k;
    double x;
    memcpy(&x, &u, sizeof x);
    return x;
}

}  // namespace metis
