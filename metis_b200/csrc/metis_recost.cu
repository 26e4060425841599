// Network what-if of a finished search (include/metis_b200.h, metis_het_recost / metis_recost_regret).
//
//   het_recost_kernel   one thread per costed candidate: the strategies and partition of its detail row and the
//                       device groups of its plan, the bandwidth-independent terms of get_cost once
//                       (RecostEvaluator, metis_recost.cuh), then the pp / dp terms and the sum under every scenario.
//                       The scenarios are walked by the whole block in step: each one's bandwidth tables are loaded
//                       into shared memory, where the block's Tables descriptor points, and read by the general
//                       (non-uniform) path of stage_terms.
//   regret              best[j] = min_i costs[j][i], regret[i] = max_j (costs[j][i] - best[j]), two-level like
//                       metis_select.cu: a min per (tile, scenario), one block per scenario over its tiles, then one
//                       pass over the candidates.  Min and max are exact, so the order of the reductions does not
//                       change a bit.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdint>

#include "../../include/metis_b200.h"
#include "metis_blob.cuh"
#include "metis_internal.h"
#include "metis_recost.cuh"

namespace metis {

constexpr int kRecostThreads = 128;
constexpr int kMaxS = METIS_MAX_STAGES, kMaxL = METIS_MAX_LAYERS;
constexpr int kRegThreads = 256, kRegItems = 8;
constexpr long long kRegTile = (long long)kRegThreads * kRegItems;
constexpr int kRegScan = 1024;

__global__ void __launch_bounds__(kRecostThreads)
het_recost_kernel(const __grid_constant__ MetisProblem p, const __grid_constant__ MetisPlanSpace sp,
                  const __grid_constant__ BlobLayout lay, const uint8_t *__restrict__ blob,
                  const MetisRecord *__restrict__ records, long long n, const uint8_t *__restrict__ detail, int stride,
                  const double *__restrict__ bandwidths, int num_scenarios, double *costs) {
    __shared__ Tables s_T;
    __shared__ double s_bw[2 * METIS_MAX_TYPES];
    const int nt = p.num_types;
    if (threadIdx.x == 0) {
        s_T = make_tables(p, lay, blob);
        s_T.p.uniform_bw = 0;                                 // the general path: bw_of_node_range / dp_bandwidth
        s_T.bw_first = s_bw;
        s_T.bw_min = s_bw + nt;
    }
    const long long i = (long long)blockIdx.x * kRecostThreads + threadIdx.x;
    Scratch<kMaxS, kMaxL> w;
    RecostEvaluator<kMaxS, kMaxL> ev(s_T, w);
    bool ok = false;
    for (int j = 0; j < num_scenarios; ++j) {
        __syncthreads();                                      // the previous scenario's tables are no longer read
        for (int t = threadIdx.x; t < 2 * nt; t += kRecostThreads) s_bw[t] = bandwidths[(size_t)j * 2 * nt + t];
        __syncthreads();
        if (i >= n) continue;
        if (j == 0) {
            PlanDesc pd;
            ok = decode_plan(sp, records[i].ordinal, pd) && pd.S <= kMaxS && ev.load(pd, detail + (size_t)i * stride) == 0;
        }
        costs[(size_t)j * n + i] = ok ? ev.scenario_cost() : (double)NAN;
    }
}

__device__ __forceinline__ double warp_min(double v) {
    for (int d = 16; d > 0; d >>= 1) v = fmin(v, __shfl_xor_sync(0xFFFFFFFFu, v, d));
    return v;
}

// min of a block's values, on thread 0
__device__ __forceinline__ double block_min(double v) {
    __shared__ double s_warp[32];
    v = warp_min(v);
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (lane == 0) s_warp[wid] = v;
    __syncthreads();
    if (threadIdx.x == 0)
        for (int k = 1; k < (int)(blockDim.x >> 5); ++k) v = fmin(v, s_warp[k]);
    return v;
}

// tile_min[j * ntiles + tile] = min of scenario j's costs over the tile (grid: tiles x scenarios)
__global__ void __launch_bounds__(kRegThreads) tile_min_kernel(const double *costs, long long n, double *tile_min) {
    const long long ntiles = gridDim.x;
    const double *row = costs + (size_t)blockIdx.y * n;
    const long long first = blockIdx.x * kRegTile + threadIdx.x;
    double m = HUGE_VAL;
#pragma unroll
    for (int k = 0; k < kRegItems; ++k) {                     // coalesced: item k of the tile's threads are adjacent
        const long long at = first + (long long)k * kRegThreads;
        if (at < n) m = fmin(m, __ldg(&row[at]));
    }
    m = block_min(m);
    if (threadIdx.x == 0) tile_min[(size_t)blockIdx.y * ntiles + blockIdx.x] = m;
}

// best[j] = min over scenario j's tiles (one block per scenario)
__global__ void __launch_bounds__(kRegScan) best_kernel(const double *tile_min, long long ntiles, double *best) {
    const double *row = tile_min + (size_t)blockIdx.x * ntiles;
    double m = HUGE_VAL;
    for (long long t = threadIdx.x; t < ntiles; t += kRegScan) m = fmin(m, row[t]);
    m = block_min(m);
    if (threadIdx.x == 0) best[blockIdx.x] = m;
}

// regret[i] = max_j (costs[j][i] - best[j])
__global__ void __launch_bounds__(kRegThreads) regret_kernel(const double *costs, int num_scenarios, long long n,
                                                              const double *best, double *regret) {
    const long long first = blockIdx.x * kRegTile + threadIdx.x;
#pragma unroll
    for (int k = 0; k < kRegItems; ++k) {
        const long long at = first + (long long)k * kRegThreads;
        if (at >= n) break;
        double r = -HUGE_VAL;
        for (int j = 0; j < num_scenarios; ++j) r = fmax(r, __ldg(&costs[(size_t)j * n + at]) - __ldg(&best[j]));
        regret[at] = r;
    }
}

static long long regret_tiles(int64_t n) { return n > 0 ? (n + kRegTile - 1) / kRegTile : 1; }

}  // namespace metis

using namespace metis;

extern "C" {

int metis_het_recost(const MetisProblem *problem, const MetisPlanSpace *space, const MetisRecord *records, int64_t n,
                     const uint8_t *detail, int32_t detail_stride, const double *bandwidths, int32_t num_scenarios,
                     double *costs, void *workspace, int64_t workspace_bytes, void *stream_) {
    if (!problem || !space || !workspace || (n > 0 && (!records || !detail || !bandwidths || !costs)))
        return fail_arg("metis_het_recost: NULL argument");
    if (n < 0) return fail_arg("metis_het_recost: negative number of records");
    if (num_scenarios < 1) return fail_arg("metis_het_recost: num_scenarios < 1");
    if (detail_stride < 3 * space->max_stage + 1) return fail_arg("metis_het_recost: detail_stride too small (3 * max_stage + 1)");
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    BlobLayout lay;
    const uint8_t *blob = nullptr;
    const int rc = stage_replay_tables(problem, workspace, workspace_bytes, stream, lay, blob);
    if (rc) return rc;
    if (n > 0) {
        const unsigned nb = (unsigned)((n + kRecostThreads - 1) / kRecostThreads);
        het_recost_kernel<<<nb, kRecostThreads, 0, stream>>>(*problem, *space, lay, blob, records, n, detail,
                                                             detail_stride, bandwidths, num_scenarios, costs);
    }
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? METIS_OK : fail_cuda(e, "het_recost_kernel");
}

int64_t metis_recost_regret_workspace_bytes(int32_t num_scenarios, int64_t n) {
    if (num_scenarios < 1 || n < 0) return METIS_E_ARG;
    return 256 + (int64_t)num_scenarios * regret_tiles(n) * 8;
}

int metis_recost_regret(const double *costs, int32_t num_scenarios, int64_t n, double *best, double *regret,
                        void *workspace, int64_t workspace_bytes, void *stream_) {
    if (n < 0) return fail_arg("metis_recost_regret: negative number of candidates");
    if (num_scenarios < 1 || num_scenarios > 65535) return fail_arg("metis_recost_regret: num_scenarios out of range (1 .. 65535)");
    if (!best || !workspace || (n > 0 && (!costs || !regret))) return fail_arg("metis_recost_regret: NULL argument");
    if (workspace_bytes < metis_recost_regret_workspace_bytes(num_scenarios, n)) return METIS_E_CAPACITY;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    double *tile_min = reinterpret_cast<double *>(align_workspace(workspace));
    const long long nt = regret_tiles(n);                     // one empty tile when n == 0: best[j] = +inf
    tile_min_kernel<<<dim3((unsigned)nt, (unsigned)num_scenarios), kRegThreads, 0, stream>>>(costs, n, tile_min);
    best_kernel<<<(unsigned)num_scenarios, kRegScan, 0, stream>>>(tile_min, nt, best);
    if (n > 0) regret_kernel<<<(unsigned)nt, kRegThreads, 0, stream>>>(costs, num_scenarios, n, best, regret);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? METIS_OK : fail_cuda(e, "regret kernels");
}

}  // extern "C"
