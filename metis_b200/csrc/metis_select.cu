// Headroom-constrained views of the ranked candidate list (include/metis_b200.h, metis_headroom_select /
// metis_headroom_front).
//
// Both walk the ranked list - the stable cost permutation of metis_sort_records - in tiles of kTile entries, each
// thread owning kItems consecutive ones, and are two-level: a per-tile pass, one block that scans the per-tile
// values, then a per-tile pass that adds the tile's carry-in.
//
//   select  stable stream compaction of the entries whose headroom is >= the threshold: count per tile, exclusive sum
//           over the tiles, scatter in ranked order.  Tiles that start at or past the k-th hit write nothing.
//   front   an entry is a "record" when its headroom is strictly above every headroom before it in ranked order
//           (exclusive prefix max: tile maxima, a max-scan over the tiles, then each tile's own scan from its carry-in).
//           Ranked order is cost ascending, estimate_costs order within equal costs, so the records are the entries no
//           earlier one weakly dominates, and the first of any equal (cost, headroom) pair.  Within a run of equal
//           costs the records climb, and only the run's last record (its first maximum) is on the front; the others
//           have a later entry of the same cost and more headroom.  So the front is a second compaction over the
//           compacted records: keep record t when record t + 1 has another cost.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdint>

#include "../../include/metis_b200.h"
#include "metis_internal.h"

namespace metis {

constexpr int kSelThreads = 256, kItems = 8;
constexpr long long kTile = (long long)kSelThreads * kItems;
constexpr int kScanThreads = 1024;
constexpr double kNegInf = -HUGE_VAL;

// block-wide exclusive scan of one value per thread (sum or max), and the block's total; all threads call it
template <class T, class Op>
__device__ __forceinline__ T block_exclusive(T v, T identity, Op op, T &total) {
    __shared__ T s_warp[32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
    T inc = v;
    for (int o = 1; o < 32; o <<= 1) {
        const T up = __shfl_up_sync(0xFFFFFFFFu, inc, o);
        if (lane >= o) inc = op(inc, up);
    }
    if (lane == 31) s_warp[wid] = inc;
    __syncthreads();
    T before = identity, all = identity;
    for (int k = 0; k < nw; ++k) {
        if (k < wid) before = op(before, s_warp[k]);
        all = op(all, s_warp[k]);
    }
    T excl = __shfl_up_sync(0xFFFFFFFFu, inc, 1);
    if (lane == 0) excl = identity;
    __syncthreads();                                          // s_warp is reused by the next call
    total = all;
    return op(before, excl);
}

struct SumOp { __device__ unsigned long long operator()(unsigned long long a, unsigned long long b) const { return a + b; } };
struct MaxOp { __device__ double operator()(double a, double b) const { return b > a ? b : a; } };

// ---- stream compaction: which entries (flag) and what is written for them (value) -----------------------------------
struct SelectItems {                 // ranked entries with headroom >= x -> their positions
    const double *headroom;
    const uint32_t *rank;
    double x;
    __device__ bool flag(long long i) const { return __ldg(&headroom[__ldg(&rank[i])]) >= x; }
    __device__ uint32_t value(long long i) const { return __ldg(&rank[i]); }
};

struct RecordItems {                 // ranked entries marked by record_flags_kernel -> their ranked index
    const uint8_t *flags;
    __device__ bool flag(long long i) const { return flags[i] != 0; }
    __device__ uint32_t value(long long i) const { return (uint32_t)i; }
};

struct LastOfRunItems {              // record t (of *m) whose successor has another cost -> its position
    const MetisRecord *records;
    const uint32_t *rank;
    const uint32_t *recs;            // ranked indices of the records
    const unsigned long long *m;
    __device__ double cost(long long t) const { return records[rank[recs[t]]].cost; }
    __device__ bool flag(long long t) const {
        const long long n = (long long)*m;
        return t < n && (t + 1 == n || cost(t + 1) != cost(t));
    }
    __device__ uint32_t value(long long t) const { return rank[recs[t]]; }
};

struct MaskItems {                   // entries whose order[i] (i without an order) is marked -> order[i]
    const uint8_t *mask;
    const uint32_t *order;
    __device__ uint32_t at(long long i) const { return order ? __ldg(&order[i]) : (uint32_t)i; }
    __device__ bool flag(long long i) const { return __ldg(&mask[at(i)]) != 0; }
    __device__ uint32_t value(long long i) const { return at(i); }
};

template <class F>
__global__ void __launch_bounds__(kSelThreads) count_kernel(F f, long long n, unsigned long long *tile_count) {
    const long long first = blockIdx.x * kTile + (long long)threadIdx.x * kItems;
    unsigned long long c = 0;
#pragma unroll
    for (int j = 0; j < kItems; ++j)
        if (first + j < n && f.flag(first + j)) ++c;
    unsigned long long total;
    block_exclusive(c, 0ULL, SumOp(), total);
    if (threadIdx.x == 0) tile_count[blockIdx.x] = total;
}

// one block: exclusive sum (in place) over the tiles; the sum of all into *total
__global__ void __launch_bounds__(kScanThreads) scan_sum_kernel(unsigned long long *v, long long ntiles,
                                                                unsigned long long *total) {
    unsigned long long carry = 0;
    for (long long b = 0; b < ntiles; b += kScanThreads) {
        const long long i = b + threadIdx.x;
        const unsigned long long x = i < ntiles ? v[i] : 0ULL;
        unsigned long long all;
        const unsigned long long e = block_exclusive(x, 0ULL, SumOp(), all);
        if (i < ntiles) v[i] = carry + e;
        carry += all;
    }
    if (threadIdx.x == 0) *total = carry;
}

// entries of a tile in order, after the base of the tile; entries at or past `limit` are not written
template <class F>
__global__ void __launch_bounds__(kSelThreads) scatter_kernel(F f, long long n, const unsigned long long *tile_base,
                                                               uint32_t *out, long long limit) {
    const unsigned long long base = tile_base[blockIdx.x];
    if ((long long)base >= limit) return;                    // whole block: no __syncthreads skipped by a part of it
    const long long first = blockIdx.x * kTile + (long long)threadIdx.x * kItems;
    bool hit[kItems];
    unsigned long long c = 0;
#pragma unroll
    for (int j = 0; j < kItems; ++j) {
        hit[j] = first + j < n && f.flag(first + j);
        c += hit[j] ? 1 : 0;
    }
    unsigned long long total;
    unsigned long long at = base + block_exclusive(c, 0ULL, SumOp(), total);
#pragma unroll
    for (int j = 0; j < kItems; ++j)
        if (hit[j]) {
            if ((long long)at < limit) out[at] = f.value(first + j);
            ++at;
        }
}

// ---- prefix max of the headroom in ranked order ---------------------------------------------------------------------
__device__ __forceinline__ double ranked_headroom(const double *headroom, const uint32_t *rank, long long i) {
    return __ldg(&headroom[__ldg(&rank[i])]);
}

__global__ void __launch_bounds__(kSelThreads) tile_max_kernel(const double *headroom, const uint32_t *rank, long long n,
                                                                double *tile_max) {
    const long long first = blockIdx.x * kTile + (long long)threadIdx.x * kItems;
    double m = kNegInf;
#pragma unroll
    for (int j = 0; j < kItems; ++j)
        if (first + j < n) m = fmax(m, ranked_headroom(headroom, rank, first + j));
    double total;
    block_exclusive(m, kNegInf, MaxOp(), total);
    if (threadIdx.x == 0) tile_max[blockIdx.x] = total;
}

// one block: exclusive max (in place) over the tiles, from -inf
__global__ void __launch_bounds__(kScanThreads) scan_max_kernel(double *v, long long ntiles) {
    double carry = kNegInf;
    for (long long b = 0; b < ntiles; b += kScanThreads) {
        const long long i = b + threadIdx.x;
        const double x = i < ntiles ? v[i] : kNegInf;
        double all;
        const double e = block_exclusive(x, kNegInf, MaxOp(), all);
        if (i < ntiles) v[i] = fmax(carry, e);
        carry = fmax(carry, all);
    }
}

// flags[i] = 1 when entry i's headroom is above every earlier one's (tile_in: the max over the tiles before)
__global__ void __launch_bounds__(kSelThreads) record_flags_kernel(const double *headroom, const uint32_t *rank,
                                                                    long long n, const double *tile_in, uint8_t *flags) {
    const long long first = blockIdx.x * kTile + (long long)threadIdx.x * kItems;
    double h[kItems];
    double m = kNegInf;
#pragma unroll
    for (int j = 0; j < kItems; ++j) {
        h[j] = first + j < n ? ranked_headroom(headroom, rank, first + j) : kNegInf;
        m = fmax(m, h[j]);
    }
    double total;
    double carry = fmax(tile_in[blockIdx.x], block_exclusive(m, kNegInf, MaxOp(), total));
#pragma unroll
    for (int j = 0; j < kItems; ++j)
        if (first + j < n) {
            flags[first + j] = h[j] > carry ? 1 : 0;
            carry = fmax(carry, h[j]);
        }
}

struct SelectWorkspace {
    unsigned long long *tile_count;  // per tile: count, then base
    double *tile_max;                // per tile: max, then the max before it
    unsigned long long *totals;      // [0] records of the front's first pass, [1] the answer's count
    uint8_t *flags;                  // n
    uint32_t *recs;                  // n
};

static long long num_tiles(int64_t n) { return n > 0 ? (n + kTile - 1) / kTile : 1; }

static SelectWorkspace carve_select(void *ws, int64_t n) {
    uint8_t *p = align_workspace(ws);
    const long long nt = num_tiles(n);
    SelectWorkspace w;
    w.tile_count = reinterpret_cast<unsigned long long *>(p); p += align256(nt * 8);
    w.tile_max = reinterpret_cast<double *>(p);               p += align256(nt * 8);
    w.totals = reinterpret_cast<unsigned long long *>(p);     p += 256;
    w.flags = p;                                              p += align256(n);
    w.recs = reinterpret_cast<uint32_t *>(p);
    return w;
}

template <class F>
static int compact(const F &f, long long n, const SelectWorkspace &w, unsigned long long *total, uint32_t *out,
                   long long limit, cudaStream_t stream) {
    const long long nt = num_tiles(n);
    count_kernel<<<(unsigned)nt, kSelThreads, 0, stream>>>(f, n, w.tile_count);
    scan_sum_kernel<<<1, kScanThreads, 0, stream>>>(w.tile_count, nt, total);
    if (limit > 0) scatter_kernel<<<(unsigned)nt, kSelThreads, 0, stream>>>(f, n, w.tile_count, out, limit);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? METIS_OK : fail_cuda(e, "headroom compaction kernels");
}

static int check_select_args(const void *headroom, const uint32_t *rank, int64_t n, const uint64_t *count,
                             const void *workspace, int64_t workspace_bytes) {
    if (n < 0 || n > 0xFFFFFFFFLL) return fail_arg("metis_headroom: n out of range (0 .. 2^32 - 1)");
    if ((n > 0 && (!headroom || !rank)) || !count || !workspace) return fail_arg("metis_headroom: NULL argument");
    if (workspace_bytes < metis_headroom_workspace_bytes(n)) return METIS_E_CAPACITY;
    return METIS_OK;
}

static int send_count(const unsigned long long *d_count, uint64_t *count, cudaStream_t stream) {
    const cudaError_t e = cudaMemcpyAsync(count, d_count, sizeof(uint64_t), cudaMemcpyDeviceToHost, stream);
    return e == cudaSuccess ? METIS_OK : fail_cuda(e, "copy headroom count");
}

}  // namespace metis

using namespace metis;

extern "C" {

int64_t metis_headroom_workspace_bytes(int64_t n) {
    if (n < 0) return METIS_E_ARG;
    return 256 + 2 * align256(num_tiles(n) * 8) + 256 + align256(n) + n * 4;
}

int metis_headroom_select(const double *headroom, const uint32_t *rank, int64_t n, double min_headroom, int64_t k,
                          uint32_t *out, uint64_t *count, void *workspace, int64_t workspace_bytes, void *stream_) {
    int rc = check_select_args(headroom, rank, n, count, workspace, workspace_bytes);
    if (rc) return rc;
    if (!std::isfinite(min_headroom)) return fail_arg("metis_headroom_select: min_headroom must be finite");
    if (k < 0 || (k > 0 && !out)) return fail_arg("metis_headroom_select: bad k / out");
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    const SelectWorkspace w = carve_select(workspace, n);
    rc = compact(SelectItems{headroom, rank, min_headroom}, n, w, w.totals + 1, out, k < n ? k : n, stream);
    return rc ? rc : send_count(w.totals + 1, count, stream);
}

int metis_headroom_front(const MetisRecord *records, const double *headroom, const uint32_t *rank, int64_t n,
                         uint32_t *out, uint64_t *count, void *workspace, int64_t workspace_bytes, void *stream_) {
    int rc = check_select_args(headroom, rank, n, count, workspace, workspace_bytes);
    if (rc) return rc;
    if (n > 0 && (!records || !out)) return fail_arg("metis_headroom_front: NULL argument");
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    const SelectWorkspace w = carve_select(workspace, n);
    const long long nt = num_tiles(n);
    if (n > 0) {
        tile_max_kernel<<<(unsigned)nt, kSelThreads, 0, stream>>>(headroom, rank, n, w.tile_max);
        scan_max_kernel<<<1, kScanThreads, 0, stream>>>(w.tile_max, nt);
        record_flags_kernel<<<(unsigned)nt, kSelThreads, 0, stream>>>(headroom, rank, n, w.tile_max, w.flags);
    }
    rc = compact(RecordItems{w.flags}, n, w, w.totals, w.recs, n, stream);
    if (rc) return rc;
    rc = compact(LastOfRunItems{records, rank, w.recs, w.totals}, n, w, w.totals + 1, out, n, stream);
    return rc ? rc : send_count(w.totals + 1, count, stream);
}

int metis_mask_select(const uint8_t *mask, const uint32_t *order, int64_t n, int64_t k, uint32_t *out, uint64_t *count,
                      void *workspace, int64_t workspace_bytes, void *stream_) {
    if (n < 0 || n > 0xFFFFFFFFLL) return fail_arg("metis_mask_select: n out of range (0 .. 2^32 - 1)");
    if ((n > 0 && !mask) || !count || !workspace) return fail_arg("metis_mask_select: NULL argument");
    if (k < 0 || (k > 0 && !out)) return fail_arg("metis_mask_select: bad k / out");
    if (workspace_bytes < metis_headroom_workspace_bytes(n)) return METIS_E_CAPACITY;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    const SelectWorkspace w = carve_select(workspace, n);
    const int rc = compact(MaskItems{mask, order}, n, w, w.totals + 1, out, k < n ? k : n, stream);
    return rc ? rc : send_count(w.totals + 1, count, stream);
}

}  // extern "C"
