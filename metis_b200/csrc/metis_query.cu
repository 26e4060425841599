// Plan queries of a finished search (include/metis_b200.h, metis_query_mark / metis_query_groups).
//
//   query_mark_kernel    one thread per candidate: its plan's geometry (decode_plan), the device-group row, its
//                        num_repartition and, when the filter or the keys read strategies, the tp codes of its detail
//                        row go through query_plan (metis_query.cuh); the optional headroom threshold is ANDed in.
//                        Writes a mask byte and the group.
//   group passes         a dense table of groups.  Pass 1: per group the member count and the lowest cost, atomicMin on
//                        cost_order_key; pass 2: the lowest position among the members that have that cost.  Min is
//                        exact in any order, so no schedule changes a result.  A last pass turns the keys back into
//                        costs and marks the groups that have members (compacted by metis_mask_select).
#include <cuda_runtime.h>

#include <cmath>
#include <cstdint>

#include "../../include/metis_b200.h"
#include "metis_blob.cuh"
#include "metis_internal.h"
#include "metis_query.cuh"

namespace metis {

constexpr int kQueryThreads = 256;
constexpr long long kMaxGroups = 1LL << 24;

__global__ void __launch_bounds__(kQueryThreads)
query_mark_kernel(const __grid_constant__ MetisProblem p, const __grid_constant__ MetisPlanSpace sp,
                  const __grid_constant__ MetisPlanFilter f, const MetisRecord *__restrict__ records, long long n,
                  const uint8_t *__restrict__ detail, int stride, const double *__restrict__ headroom, double x,
                  uint8_t *__restrict__ mask, uint32_t *__restrict__ group) {
    const long long i = (long long)blockIdx.x * kQueryThreads + threadIdx.x;
    if (i >= n) return;
    const MetisRecord r = records[i];
    PlanDesc pd;
    uint32_t g = METIS_QUERY_NO_GROUP;
    bool ok = decode_plan(sp, r.ordinal, pd);
    if (ok) {
        QueryPlan q;
        q.ns = pd.ns;
        q.S = pd.S;
        q.div = (int)(pd.geo >> 56);
        q.num_div = sp.num_div;
        q.nrep = r.num_repartition;
        q.row = pd.row;
        q.tpc = detail ? detail + (size_t)i * stride + pd.S : nullptr;
        ok = query_plan(f, p.num_types, p.ns_run_type, p.ns_run_end, q, g);
    }
    if (ok && headroom && !(__ldg(&headroom[i]) >= x)) ok = false;
    mask[i] = ok ? 1 : 0;
    if (group) group[i] = ok ? g : METIS_QUERY_NO_GROUP;
}

__global__ void group_init_kernel(long long G, unsigned long long *count, unsigned long long *cost_key,
                                  unsigned long long *first) {
    const long long g = (long long)blockIdx.x * kQueryThreads + threadIdx.x;
    if (g >= G) return;
    count[g] = 0;
    cost_key[g] = ~0ULL;
    first[g] = ~0ULL;
}

__global__ void __launch_bounds__(kQueryThreads)
group_min_kernel(const MetisRecord *__restrict__ records, const uint32_t *__restrict__ group, long long n,
                 unsigned long long *count, unsigned long long *cost_key) {
    const long long i = (long long)blockIdx.x * kQueryThreads + threadIdx.x;
    if (i >= n) return;
    const uint32_t g = group[i];
    if (g == METIS_QUERY_NO_GROUP) return;
    atomicAdd(&count[g], 1ULL);
    atomicMin(&cost_key[g], (unsigned long long)cost_order_key(records[i].cost));
}

__global__ void __launch_bounds__(kQueryThreads)
group_first_kernel(const MetisRecord *__restrict__ records, const uint32_t *__restrict__ group, long long n,
                   const unsigned long long *__restrict__ cost_key, unsigned long long *first) {
    const long long i = (long long)blockIdx.x * kQueryThreads + threadIdx.x;
    if (i >= n) return;
    const uint32_t g = group[i];
    if (g == METIS_QUERY_NO_GROUP) return;
    if ((unsigned long long)cost_order_key(records[i].cost) == __ldg(&cost_key[g])) atomicMin(&first[g], (unsigned long long)i);
}

__global__ void group_finish_kernel(long long G, const unsigned long long *count, unsigned long long *cost_key,
                                    unsigned long long *first, uint8_t *present) {
    const long long g = (long long)blockIdx.x * kQueryThreads + threadIdx.x;
    if (g >= G) return;
    const bool any = count[g] > 0;
    present[g] = any ? 1 : 0;
    reinterpret_cast<double *>(cost_key)[g] = any ? cost_from_order_key(cost_key[g]) : (double)HUGE_VAL;
    if (!any) first[g] = ~0ULL;                               // reads as -1 through int64
}

static unsigned blocks_of(long long n) { return (unsigned)((n + kQueryThreads - 1) / kQueryThreads); }

}  // namespace metis

using namespace metis;

extern "C" {

int metis_query_mark(const MetisProblem *problem, const MetisPlanSpace *space, const MetisPlanFilter *filter,
                     const MetisRecord *records, int64_t n, const uint8_t *detail, int32_t detail_stride,
                     const double *headroom, double min_headroom, uint8_t *mask, uint32_t *group, void *stream_) {
    if (!problem || !space || !filter || (n > 0 && (!records || !mask))) return fail_arg("metis_query_mark: NULL argument");
    if (n < 0) return fail_arg("metis_query_mark: negative number of records");
    const MetisPlanFilter &f = *filter;
    if (f.num_keys < 0 || f.num_keys > METIS_QUERY_MAX_KEYS) return fail_arg("metis_query_mark: num_keys out of range (0 .. 5)");
    bool reads_tp = f.flags & METIS_QUERY_NEEDS_TP;
    long long groups = 1;
    for (int k = 0; k < f.num_keys; ++k) {
        if (f.key_field[k] < METIS_QUERY_KEY_NS || f.key_field[k] > METIS_QUERY_KEY_NREP)
            return fail_arg("metis_query_mark: unknown key field");
        if (f.key_range[k] < 1) return fail_arg("metis_query_mark: key_range < 1");
        groups *= f.key_range[k];
        if (groups > kMaxGroups) return fail_arg("metis_query_mark: more than 2^24 groups");
        reads_tp |= f.key_field[k] == METIS_QUERY_KEY_MAX_TP;
    }
    if (f.num_keys > 0 && n > 0 && !group) return fail_arg("metis_query_mark: keys without a group output");
    if (reads_tp && n > 0 && !detail) return fail_arg("metis_query_mark: the filter or the keys read strategies: detail rows needed");
    if (reads_tp && detail_stride < 3 * space->max_stage + 1)
        return fail_arg("metis_query_mark: detail_stride too small (3 * max_stage + 1)");
    if (headroom && !std::isfinite(min_headroom)) return fail_arg("metis_query_mark: min_headroom must be finite");
    if (problem->num_types < 1 || problem->num_types > METIS_MAX_TYPES || space->num_div > 256)
        return fail_arg("metis_query_mark: problem out of range");
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (n > 0)
        query_mark_kernel<<<blocks_of(n), kQueryThreads, 0, stream>>>(*problem, *space, f, records, n,
                                                                      reads_tp ? detail : nullptr, detail_stride,
                                                                      headroom, min_headroom, mask, group);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? METIS_OK : fail_cuda(e, "query_mark_kernel");
}

int metis_query_groups(const MetisRecord *records, const uint32_t *group, int64_t n, int64_t num_groups,
                       uint64_t *count, double *cost, int64_t *first, uint8_t *present, void *stream_) {
    if (n < 0) return fail_arg("metis_query_groups: negative number of records");
    if (num_groups < 1 || num_groups > kMaxGroups) return fail_arg("metis_query_groups: num_groups out of range (1 .. 2^24)");
    if (!count || !cost || !first || !present || (n > 0 && (!records || !group)))
        return fail_arg("metis_query_groups: NULL argument");
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    auto *cnt = reinterpret_cast<unsigned long long *>(count);
    auto *key = reinterpret_cast<unsigned long long *>(cost);
    auto *fst = reinterpret_cast<unsigned long long *>(first);
    group_init_kernel<<<blocks_of(num_groups), kQueryThreads, 0, stream>>>(num_groups, cnt, key, fst);
    if (n > 0) {
        group_min_kernel<<<blocks_of(n), kQueryThreads, 0, stream>>>(records, group, n, cnt, key);
        group_first_kernel<<<blocks_of(n), kQueryThreads, 0, stream>>>(records, group, n, key, fst);
    }
    group_finish_kernel<<<blocks_of(num_groups), kQueryThreads, 0, stream>>>(num_groups, cnt, key, fst, present);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? METIS_OK : fail_cuda(e, "group kernels");
}

}  // extern "C"
