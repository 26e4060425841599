// metis_comps.cuh - the compositions of a plan space, listed without walking them (SURVEY.md 8(f)-1).
//
// metis_enum.cpp lists the compositions of every stage count on the host, in the order of the reference's depth-first
// search (search_space/device_group.py:58-81), merges their groups (:7-55) and counts their multiset permutations.
// `dg_idx` is the position of a row in that list, so the order is part of the contract.  The routines below restate
// the same three steps for ONE composition, picked by its rank, so that one thread handles one composition:
//   - a table of completion counts N[k][R][m] (compositions of R GPUs into exactly m groups whose shapes are the
//     powers of two 2^k .. 2^top) turns a rank into its composition (comp_unrank);
//   - comp_merge / comp_perm_count restate merge_groups / multiset_permutation_count on (offset, length, sum) slices;
//   - comp_slice_records cuts the composition's rows inside a row range into MetisCompRec slices.
// Integer work only; shared by the CUDA kernels (metis_listing.cu) and the host test build.
#pragma once

#include <stdint.h>

#include "../../include/metis_b200.h"

#ifndef MB_HD                     // as in metis_eval.cuh, which this header does not need
#if defined(__CUDACC__)
#define MB_HD __host__ __device__ __forceinline__
#else
#define MB_HD inline
#endif
#endif

namespace metis {

// N[k][R][m] for k = 0 .. top+1, R = 0 .. gpus, m = 0 .. max_m (row-major)
MB_HD int64_t comp_table_at(int k, int R, int m, int gpus, int max_m) {
    return ((int64_t)k * (gpus + 1) + R) * (int64_t)(max_m + 1) + m;
}

MB_HD int comp_top_shape(int gpus) {         // log2 of the largest power of two <= gpus (the last shape of list_stage)
    int t = 0;
    while ((2 << t) <= gpus) ++t;
    return t;
}

// Host: fills the table.  Level top+1 holds no shape: only (0 GPUs, 0 groups) completes.  Level k either takes one
// more group of 2^k (and stays at k) or moves on to k+1 - in that order, which is list_compositions' order ("more
// of the smaller shape first").
inline void comp_fill_table(int64_t *N, int gpus, int max_m) {
    const int top = comp_top_shape(gpus);
    for (int R = 0; R <= gpus; ++R)
        for (int m = 0; m <= max_m; ++m) N[comp_table_at(top + 1, R, m, gpus, max_m)] = (R == 0 && m == 0) ? 1 : 0;
    for (int k = top; k >= 0; --k)
        for (int R = 0; R <= gpus; ++R)
            for (int m = 0; m <= max_m; ++m) {
                int64_t v = N[comp_table_at(k + 1, R, m, gpus, max_m)];
                if (R >= (1 << k) && m >= 1) v += N[comp_table_at(k, R - (1 << k), m - 1, gpus, max_m)];
                N[comp_table_at(k, R, m, gpus, max_m)] = v;
            }
}

// list_stage's first shape for `stages` stages: the smallest power of two at or above the variance floor
// (device_group.py:96-98, in the same double arithmetic); -1 when no shape is left (no composition).
inline int comp_first_shape(int stages, int gpus, double variance) {
    const int share = gpus / stages > stages / gpus ? gpus / stages : stages / gpus;
    const double floor_share = (double)share * variance;
    for (int k = 0; (1 << k) <= gpus; ++k)
        if ((double)(1 << k) >= floor_share) return k;
    return -1;
}

// Composition `idx` (0-based, list_compositions' order) of `gpus` GPUs into `stages` groups whose shapes start at
// 2^first: writes the log2 codes of its groups, non-decreasing, into codes[stages].
MB_HD void comp_unrank(const int64_t *N, int gpus, int max_m, int first, int stages, int64_t idx, uint8_t *codes) {
    const int top = comp_top_shape(gpus);
    int R = gpus, m = stages, k = first, p = 0;
    while (m > 0 && k <= top) {
        const int64_t more = (R >= (1 << k)) ? N[comp_table_at(k, R - (1 << k), m - 1, gpus, max_m)] : 0;
        if (idx < more) {
            codes[p++] = (uint8_t)k;
            R -= 1 << k;
            --m;
        } else {
            idx -= more;
            ++k;
        }
    }
}

struct CompSlice {
    uint8_t off, len;             // a merged group is a contiguous slice of the composition
    int32_t sum;                  // its devices
};

MB_HD bool comp_same(const uint8_t *codes, const CompSlice &a, const CompSlice &b) {
    if (a.len != b.len) return false;
    for (int i = 0; i < a.len; ++i)
        if (codes[a.off + i] != codes[b.off + i]) return false;
    return true;
}

MB_HD bool comp_less(const uint8_t *codes, const CompSlice &a, const CompSlice &b) {   // tuple comparison
    const int n = a.len < b.len ? a.len : b.len;
    for (int i = 0; i < n; ++i)
        if (codes[a.off + i] != codes[b.off + i]) return codes[a.off + i] < codes[b.off + i];
    return a.len < b.len;
}

// merge_groups of metis_enum.cpp (device_group.py:7-55 without the permutations) on the composition codes[stages]:
// the merged groups, sorted (utils.py:57), in g[0 .. return value).  tmp: scratch of `stages` slices.
MB_HD int comp_merge(const uint8_t *codes, int stages, int max_permute_len, CompSlice *g, CompSlice *tmp) {
    int n = stages;
    for (int i = 0; i < n; ++i) g[i] = CompSlice{(uint8_t)i, 1, 1 << codes[i]};
    int num_reduce = n - max_permute_len;
    while (num_reduce > 0) {
        const int count = n;
        const int min_size = g[0].sum;
        int num_min = count;                                   // find_num_min (:8-12)
        for (int idx = 0; idx < count; ++idx)
            if (!comp_same(codes, g[idx], g[0])) { num_min = idx + 1; break; }
        if (num_min / 2 > num_reduce) num_reduce = num_min / 2;              // :26-27
        int q = 0;
        for (int i = 0; i < count; i += 2) {                                 // :31-45
            if (num_reduce <= i / 2) {
                for (int j = i; j < count; ++j) tmp[q++] = g[j];
                break;
            }
            if (i + 1 >= count) {
                tmp[q++] = g[i];
            } else if (g[i].sum == min_size && g[i].sum == g[i + 1].sum) {
                tmp[q++] = CompSlice{g[i].off, (uint8_t)(g[i].len + g[i + 1].len), g[i].sum + g[i + 1].sum};
            } else {
                tmp[q++] = g[i];
                tmp[q++] = g[i + 1];
            }
        }
        for (int i = 0; i < q; ++i) g[i] = tmp[i];
        n = q;
        if (num_reduce == n - max_permute_len) break;                        // :48-50
        num_reduce = n - max_permute_len;
    }
    for (int i = 1; i < n; ++i) {                              // insertion sort: equal groups are identical
        const CompSlice v = g[i];
        int j = i - 1;
        while (j >= 0 && comp_less(codes, v, g[j])) { g[j + 1] = g[j]; --j; }
        g[j + 1] = v;
    }
    return n;
}

// multiset_permutation_count of metis_enum.cpp on the sorted groups: n! / prod(multiplicity!)
MB_HD int64_t comp_perm_count(const uint8_t *codes, const CompSlice *g, int n) {
    int64_t total = 1, placed = 0;
    int i = 0;
    while (i < n) {
        int j = i;
        while (j < n && comp_same(codes, g[j], g[i])) ++j;
        for (int64_t k = 1; k <= (int64_t)(j - i); ++k) total = total * (placed + k) / k;
        placed += j - i;
        i = j;
    }
    return total;
}

// The composition's pool entry (metis_enum_compositions' layout): n group lengths, then the codes of the groups in
// sorted order - n + stages bytes.
MB_HD void comp_write_pool(const uint8_t *codes, const CompSlice *g, int n, uint8_t *dst) {
    for (int i = 0; i < n; ++i) dst[i] = g[i].len;
    uint8_t *p = dst + n;
    for (int i = 0; i < n; ++i)
        for (int b = 0; b < g[i].len; ++b) *p++ = codes[g[i].off + b];
}

// The slices of one composition inside the row range [r0, r1) of its stage count.  The composition holds rows
// [first, first + perms) of the stage count's table; its slices are metis_enum_compositions' (METIS_COMP_SLICE_ROWS
// rows each from the composition's first row), cut to the range.  `range_byte` is the byte offset of row r0 in the
// window's rows.  Returns the number of slices; writes them to out[] when out is not NULL.
MB_HD int64_t comp_slice_records(int64_t first, int64_t perms, int64_t r0, int64_t r1, int stages, int num_groups,
                                 int64_t range_byte, uint32_t pool_offset, MetisCompRec *out) {
    const int64_t lo = (first > r0 ? first : r0) - first;
    const int64_t hi = (first + perms < r1 ? first + perms : r1) - first;
    if (hi <= lo) return 0;
    const int64_t slice = METIS_COMP_SLICE_ROWS;
    if (!out) return (hi - 1) / slice - lo / slice + 1;
    int64_t k = 0;
    for (int64_t s0 = lo / slice * slice; s0 < hi; s0 += slice, ++k) {
        const int64_t f = s0 > lo ? s0 : lo, e = s0 + slice < hi ? s0 + slice : hi;
        MetisCompRec r;
        r.row_offset = range_byte + (first + f - r0) * stages;
        r.pool_offset = pool_offset;
        r.stages = (uint16_t)stages;
        r.num_groups = (uint16_t)num_groups;
        r.first_row = (uint32_t)f;
        r.num_rows = (uint32_t)(e - f);
        out[k] = r;
    }
    return k;
}

}  // namespace metis
