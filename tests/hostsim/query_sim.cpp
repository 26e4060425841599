// query_sim.cpp - TEST-ONLY host build of the plan queries (query_plan and the group-best passes of
// metis_b200/csrc/metis_query.cuh / metis_query.cu), so that the CPU suite checks the code metis_query_mark and
// metis_query_groups run.  It is hostsim.cpp (whose plan decoding it reuses) plus the entry points below, one loop
// iteration per device thread.  Built and loaded only by tests/test_query.py, with hostsim.cpp's flags.
#include "hostsim.cpp"
#include "../../metis_b200/csrc/metis_query.cuh"

extern "C" {

// metis_query_mark on the host (no headroom)
int query_sim_mark(const MetisProblem *p, const MetisPlanSpace *sp, const MetisPlanFilter *f, const MetisRecord *records,
                   int64_t n, const uint8_t *detail, int32_t stride, uint8_t *mask, uint32_t *group) {
    for (int64_t i = 0; i < n; ++i) {
        PlanDesc pd;
        uint32_t g = METIS_QUERY_NO_GROUP;
        bool ok = decode(*sp, records[i].ordinal, pd);
        if (ok) {
            QueryPlan q;
            q.ns = pd.ns;
            q.S = pd.S;
            q.div = (int)(pd.geo >> 56);
            q.num_div = sp->num_div;
            q.nrep = records[i].num_repartition;
            q.row = pd.row;
            q.tpc = detail ? detail + (size_t)i * stride + pd.S : nullptr;
            ok = query_plan(*f, p->num_types, p->ns_run_type, p->ns_run_end, q, g);
        }
        mask[i] = ok ? 1 : 0;
        group[i] = ok ? g : METIS_QUERY_NO_GROUP;
    }
    return 0;
}

// metis_query_groups on the host: the two passes over the candidates in the order given by `visit` (a permutation of
// 0..n-1), to show that the answer does not depend on it
int query_sim_groups(const MetisRecord *records, const uint32_t *group, int64_t n, const int64_t *visit,
                     int64_t num_groups, uint64_t *count, double *cost, int64_t *first) {
    std::vector<uint64_t> key(num_groups, ~0ULL), fst(num_groups, ~0ULL);
    for (int64_t g = 0; g < num_groups; ++g) count[g] = 0;
    for (int64_t j = 0; j < n; ++j) {
        const int64_t i = visit[j];
        const uint32_t g = group[i];
        if (g == METIS_QUERY_NO_GROUP) continue;
        ++count[g];
        const uint64_t k = cost_order_key(records[i].cost);
        if (k < key[g]) key[g] = k;
    }
    for (int64_t j = 0; j < n; ++j) {
        const int64_t i = visit[j];
        const uint32_t g = group[i];
        if (g == METIS_QUERY_NO_GROUP) continue;
        if (cost_order_key(records[i].cost) == key[g] && (uint64_t)i < fst[g]) fst[g] = (uint64_t)i;
    }
    for (int64_t g = 0; g < num_groups; ++g) {
        cost[g] = count[g] ? cost_from_order_key(key[g]) : HUGE_VAL;
        first[g] = count[g] ? (int64_t)fst[g] : -1;
    }
    return 0;
}

}  // extern "C"
