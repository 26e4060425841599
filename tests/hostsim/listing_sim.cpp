// listing_sim.cpp - test-only g++ build of the device listing (metis_comps.cuh): the routines of metis_listing.cu's
// kernels, run one composition after the other, so that the CPU suite can compare them with metis_enum_compositions.
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../metis_b200/csrc/metis_comps.cuh"

using namespace metis;

namespace {

struct Listed {
    int first_stage = 0, n = 0, gpus = 0, max_m = 0, mpl = 0;
    std::vector<int64_t> table, base, offs;
    std::vector<int32_t> first;
    std::vector<uint8_t> ngroups;
};

// the listing of the last call is kept: the tests emit many small windows of one big space
const Listed &list(int first_stage, int last_stage, int gpus, double variance, int mpl) {
    static Listed L;
    static double last_variance = -1.0;
    if (L.n && L.first_stage == first_stage && L.n == last_stage - first_stage + 1 && L.gpus == gpus && L.mpl == mpl &&
        last_variance == variance)
        return L;
    last_variance = variance;
    L.first_stage = first_stage;
    L.n = last_stage - first_stage + 1;
    L.gpus = gpus;
    L.max_m = last_stage;
    L.mpl = mpl;
    const int top = comp_top_shape(gpus);
    L.table.assign((size_t)comp_table_at(top + 2, 0, 0, gpus, L.max_m), 0);
    comp_fill_table(L.table.data(), gpus, L.max_m);
    L.first.assign(L.n, 0);
    L.base.assign(L.n + 1, 0);
    for (int i = 0; i < L.n; ++i) {
        const int S = first_stage + i;
        const int k = comp_first_shape(S, gpus, variance);
        L.first[i] = k < 0 ? 0 : k;
        L.base[i + 1] = L.base[i] + (k < 0 ? 0 : L.table[comp_table_at(k, gpus, S, gpus, L.max_m)]);
    }
    const int64_t total = L.base[L.n];
    L.offs.assign(total + 1, 0);
    L.ngroups.assign(total, 0);
    uint8_t codes[METIS_MAX_STAGES];
    CompSlice g[METIS_MAX_STAGES], tmp[METIS_MAX_STAGES];
    for (int s = 0; s < L.n; ++s)
        for (int64_t c = L.base[s]; c < L.base[s + 1]; ++c) {
            comp_unrank(L.table.data(), gpus, L.max_m, L.first[s], first_stage + s, c - L.base[s], codes);
            const int n = comp_merge(codes, first_stage + s, mpl, g, tmp);
            L.ngroups[c] = (uint8_t)n;
            L.offs[c + 1] = L.offs[c] + comp_perm_count(codes, g, n);
        }
    return L;
}

}  // namespace

extern "C" {

// rows_per_stage [n], comps_per_stage [n]; returns the most merged groups of any composition
int32_t listing_sim_stages(int32_t first_stage, int32_t last_stage, int32_t gpus, double variance, int32_t mpl,
                           int64_t *rows_per_stage, int64_t *comps_per_stage) {
    const Listed &L = list(first_stage, last_stage, gpus, variance, mpl);
    int most = 0;
    for (int s = 0; s < L.n; ++s) {
        rows_per_stage[s] = L.offs[L.base[s + 1]] - L.offs[L.base[s]];
        comps_per_stage[s] = L.base[s + 1] - L.base[s];
    }
    for (uint8_t n : L.ngroups) most = n > most ? n : most;
    return most;
}

// metis_list_window's records and pool for the ranges (stage count, first row, end row); recs == NULL: sizes only.
// sizes[0] records, sizes[1] pool bytes; returns -1 when a range holds a composition of too many groups.
int32_t listing_sim_window(int32_t first_stage, int32_t last_stage, int32_t gpus, double variance, int32_t mpl,
                           const MetisRowRange *ranges, int32_t nr, MetisCompRec *recs, uint8_t *pool, int64_t *sizes) {
    const Listed &L = list(first_stage, last_stage, gpus, variance, mpl);
    uint8_t codes[METIS_MAX_STAGES];
    CompSlice g[METIS_MAX_STAGES], tmp[METIS_MAX_STAGES];
    int64_t nrec = 0, pbytes = 0, byte = 0;
    int status = 0;
    for (int i = 0; i < nr; ++i) {
        const MetisRowRange r = ranges[i];
        const int s = r.stages - first_stage;
        const int64_t o = L.offs[L.base[s]];
        for (int64_t c = L.base[s]; c < L.base[s + 1]; ++c) {
            const int64_t f = L.offs[c] - o, perms = L.offs[c + 1] - L.offs[c];
            if (f + perms <= r.first_row || f >= r.end_row) continue;
            if (L.ngroups[c] > METIS_MAX_PERMUTE_GROUPS) { status = -1; continue; }
            comp_unrank(L.table.data(), gpus, L.max_m, L.first[s], r.stages, c - L.base[s], codes);
            const int n = comp_merge(codes, r.stages, mpl, g, tmp);
            if (recs) comp_write_pool(codes, g, n, pool + pbytes);
            nrec += comp_slice_records(f, perms, r.first_row, r.end_row, r.stages, n, byte, (uint32_t)pbytes,
                                       recs ? recs + nrec : nullptr);
            pbytes += n + r.stages;
        }
        byte += (r.end_row - r.first_row) * r.stages;
    }
    sizes[0] = nrec;
    sizes[1] = pbytes;
    return status;
}

}  // extern "C"
