// Ordering of the candidate records on the device (SURVEY.md 8(f)-2).
//
// metis_het_search appends its 16-byte records in completion order.  The reference's list
// `estimate_costs` (cost_het_cluster.py:44) is in (inter-stage plan, chain step) order and its ranked
// listing is `sorted(estimate_costs, key=cost)` (cost_het_cluster.py:76) - a STABLE sort, so equal costs keep
// their estimate_costs order.  Both orders are produced here by one cooperative kernel: a stable
// least-significant-digit radix sort, 8 bits per pass, over the key
//     (ordinal : 32, step : 16)                       6 passes  -> estimate_costs order
//     then the order-preserving image of the fp64 cost  8 passes  -> ranked order (ties keep position order)
// Each warp owns a contiguous chunk of the array: it counts its digits, a grid-wide scan turns the
// counts into global offsets, and the warp scatters its chunk in order (ranks inside a 32-element tile
// from __match_any_sync), which is what keeps every pass stable.  Passes whose digit is the same for all
// records (high bytes of small ordinals, steps < 256, shared exponent bytes) are detected after the
// count and skipped.  The work is byte shuffling bound by HBM/L2 bandwidth; for the 2.7e5 records of
// BASELINE configs[2] it is tens of microseconds per pass.
#include <cooperative_groups.h>
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>

#include "../../include/metis_b200.h"
#include "metis_internal.h"

namespace cg = cooperative_groups;

namespace metis {

constexpr int kRankThreads = 256;
constexpr int kRankWarps = kRankThreads / 32;

struct RankArgs {
    uint4 *a, *b;             // records (16 B each): a = caller's array, b = scratch
    uint32_t *ia, *ib;        // original index travelling with each record
    long long n;
    unsigned int *hist;       // [256][warps]
    unsigned int *bintot;     // [256]
    int pass_begin, pass_end; // passes 0-5 sort by position, 6-13 by cost
    uint32_t *perm_out;       // optional
};

__device__ __forceinline__ unsigned int digit_of(const uint4 &r, int pass) {
    // r.x, r.y = cost bits (lo, hi); r.z = ordinal; r.w = step | num_repartition << 16 | num_stage << 24
    if (pass < 6) {
        const unsigned long long pos = ((unsigned long long)r.z << 16) | (r.w & 0xFFFFu);
        return (unsigned int)(pos >> (8 * pass)) & 0xFFu;
    }
    unsigned long long u = ((unsigned long long)r.y << 32) | r.x;
    u ^= (u >> 63) ? ~0ULL : 0x8000000000000000ULL;      // total order of the doubles (no NaN reaches here)
    return (unsigned int)(u >> (8 * (pass - 6))) & 0xFFu;
}

__global__ void __launch_bounds__(kRankThreads) rank_records_kernel(RankArgs q) {
    cg::grid_group grid = cg::this_grid();
    __shared__ unsigned int bins[kRankWarps][256];
    __shared__ unsigned int sbase[256];
    __shared__ unsigned int sscan[kRankWarps];
    __shared__ int s_skip;
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const long long nwarps = (long long)gridDim.x * kRankWarps;
    const long long gw = (long long)blockIdx.x * kRankWarps + wib;
    const long long n = q.n;
    long long chunk = (n + nwarps - 1) / nwarps;
    chunk = (chunk + 31) / 32 * 32;
    const long long lo = gw * chunk < n ? gw * chunk : n;
    const long long hi = lo + chunk < n ? lo + chunk : n;
    const unsigned full = 0xFFFFFFFFu;
    const unsigned lt = (1u << lane) - 1u;

    for (long long i = (long long)blockIdx.x * kRankThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kRankThreads)
        q.ia[i] = (uint32_t)i;
    uint4 *src = q.a, *dst = q.b;
    uint32_t *isrc = q.ia, *idst = q.ib;
    grid.sync();

    for (int pass = q.pass_begin; pass < q.pass_end; ++pass) {
        // ---- count -------------------------------------------------------------------------------
        for (int d = lane; d < 256; d += 32) bins[wib][d] = 0;
        __syncwarp();
        for (long long t = lo; t < hi; t += 32) {
            const long long i = t + lane;
            const int d = i < hi ? (int)digit_of(src[i], pass) : -1;
            const unsigned peers = __match_any_sync(full, d);
            if (d >= 0 && lane == __ffs(peers) - 1) bins[wib][d] += __popc(peers);
            __syncwarp();
        }
        for (int d = lane; d < 256; d += 32) q.hist[(long long)d * nwarps + gw] = bins[wib][d];
        grid.sync();
        // ---- scan: rows (one digit over all warps), then the 256 digit totals -----------------------
        for (long long d = gw; d < 256; d += nwarps) {
            unsigned int *row = q.hist + d * nwarps;
            unsigned int run = 0;
            for (long long c = 0; c < nwarps; c += 32) {
                const unsigned int v = c + lane < nwarps ? row[c + lane] : 0;
                unsigned int inc = v;
                for (int o = 1; o < 32; o <<= 1) {
                    const unsigned int up = __shfl_up_sync(full, inc, o);
                    if (lane >= o) inc += up;
                }
                if (c + lane < nwarps) row[c + lane] = run + inc - v;
                run += __shfl_sync(full, inc, 31);
            }
            if (lane == 0) q.bintot[d] = run;
        }
        grid.sync();
        {
            const unsigned int v = threadIdx.x < 256 ? *(volatile unsigned int *)&q.bintot[threadIdx.x] : 0;
            if (threadIdx.x == 0) s_skip = 0;
            __syncthreads();
            if (threadIdx.x < 256 && (long long)v == n) s_skip = 1;        // every record has this digit
            unsigned int inc = v;
            for (int o = 1; o < 32; o <<= 1) {
                const unsigned int up = __shfl_up_sync(full, inc, o);
                if (lane >= o) inc += up;
            }
            if (lane == 31) sscan[wib] = inc;
            __syncthreads();
            unsigned int before = 0;
            for (int k = 0; k < wib; ++k) before += sscan[k];
            if (threadIdx.x < 256) sbase[threadIdx.x] = before + inc - v;
            __syncthreads();
        }
        if (s_skip) { __syncthreads(); continue; }              // same decision in every block: nothing to move
        // ---- scatter, chunk order preserved ----------------------------------------------------------
        for (int d = lane; d < 256; d += 32) bins[wib][d] = sbase[d] + q.hist[(long long)d * nwarps + gw];
        __syncwarp();
        for (long long t = lo; t < hi; t += 32) {
            const long long i = t + lane;
            uint4 r = make_uint4(0, 0, 0, 0);
            uint32_t id = 0;
            int d = -1;
            if (i < hi) { r = src[i]; id = isrc[i]; d = (int)digit_of(r, pass); }
            const unsigned peers = __match_any_sync(full, d);
            unsigned int base = 0;
            if (d >= 0) base = bins[wib][d];
            __syncwarp();
            if (d >= 0) {
                if (lane == __ffs(peers) - 1) bins[wib][d] = base + __popc(peers);
                const unsigned int to = base + __popc(peers & lt);
                dst[to] = r;
                idst[to] = id;
            }
            __syncwarp();
        }
        { uint4 *t = src; src = dst; dst = t; }
        { uint32_t *t = isrc; isrc = idst; idst = t; }
        grid.sync();
    }
    // ---- results into the caller's arrays ----------------------------------------------------------------
    for (long long i = (long long)blockIdx.x * kRankThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kRankThreads) {
        if (src != q.a) q.a[i] = src[i];
        if (q.perm_out) q.perm_out[i] = isrc[i];
    }
}

static int rank_grid(int *blocks) {
    int dev = 0, sms = 0, per_sm = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, rank_records_kernel, kRankThreads, 0);
    if (e != cudaSuccess) return fail_cuda(e, "rank_records_kernel occupancy");
    if (per_sm < 1) return fail_arg("rank_records_kernel does not fit on this device");
    if (per_sm > 2) per_sm = 2;                 // 2 blocks x 8 warps per SM are plenty for a bandwidth-light pass
    *blocks = sms * per_sm;
    return METIS_OK;
}

}  // namespace metis

using namespace metis;

extern "C" {

// upper bound on the warps of the cooperative grid (H100 SXM: 132 SMs x 2 blocks x 8 warps = 2112)
static const int64_t kRankMaxWarps = 8192;

int64_t metis_sort_workspace_bytes(int64_t n) {
    if (n < 0) return METIS_E_ARG;
    return 512 + n * 16 + 2 * n * 4 + 256 * kRankMaxWarps * 4 + 256 * 4 + 512;
}

int metis_sort_records(MetisRecord *records, int64_t n, int32_t mode, uint32_t *perm_out, void *workspace,
                       int64_t workspace_bytes, void *stream_) {
    if (n < 0 || (n > 0 && !records) || !workspace) return fail_arg("metis_sort_records: bad argument");
    if (mode < METIS_SORT_POSITION || mode > METIS_SORT_BY_COST_STABLE) return fail_arg("metis_sort_records: unknown mode");
    if (n >= 0xFFFFFFF0LL) return fail_arg("metis_sort_records: more than 2^32 records");
    if (workspace_bytes < metis_sort_workspace_bytes(n)) return METIS_E_CAPACITY;
    if (n == 0) return METIS_OK;
    int blocks = 0;
    const int rc = rank_grid(&blocks);
    if (rc) return rc;
    if ((int64_t)blocks * kRankWarps > kRankMaxWarps) blocks = (int)(kRankMaxWarps / kRankWarps);
    uint8_t *p = align_workspace(workspace);
    RankArgs q;
    q.a = reinterpret_cast<uint4 *>(records);
    q.b = reinterpret_cast<uint4 *>(p);            p += n * 16;
    q.ia = reinterpret_cast<uint32_t *>(p);        p += n * 4;
    q.ib = reinterpret_cast<uint32_t *>(p);        p += n * 4;
    p = align_workspace(p);
    q.hist = reinterpret_cast<unsigned int *>(p);  p += 256 * (int64_t)blocks * kRankWarps * 4;
    q.bintot = reinterpret_cast<unsigned int *>(p);
    q.n = n;
    q.pass_begin = mode == METIS_SORT_BY_COST_STABLE ? 6 : 0;
    q.pass_end = mode == METIS_SORT_POSITION ? 6 : 14;
    q.perm_out = perm_out;
    void *args[] = {&q};
    cudaError_t e = cudaLaunchCooperativeKernel((const void *)rank_records_kernel, dim3((unsigned)blocks), dim3(kRankThreads),
                                                args, 0, static_cast<cudaStream_t>(stream_));
    if (e != cudaSuccess) return fail_cuda(e, "rank_records_kernel");
    return METIS_OK;
}

}  // extern "C"
