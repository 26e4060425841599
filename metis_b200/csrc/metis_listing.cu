// metis_listing.cu - device-side listing of a plan space's compositions (C ABI: metis_list_*, include/metis_b200.h).
//
// metis_enum_compositions lists every composition on the host and keeps them all; at 512 GPUs that is millions of
// heap vectors and seconds per call.  Here the host only builds the table of completion counts (metis_comps.cuh, a
// few MB) and the GPU does the rest:
//   list_comps_kernel     one thread per composition: unrank, merge, count its permutations
//   scan_*_kernel         prefix sums (int64) of the counts: row offsets per composition, record / pool offsets of a
//                         window
//   window_*_kernel       the records and pool of a window's row ranges: count, scan, write
// The rows themselves are written afterwards by het_rows_kernel (metis_generate_rows), unchanged.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <vector>

#include "metis_comps.cuh"
#include "metis_internal.h"

namespace metis {
namespace {

constexpr int kListThreads = 128;
constexpr int kListBlocks = 2048;                     // grid-stride kernels: enough blocks to fill an H100
constexpr int kScanThreads = 256, kScanItems = 8, kScanTile = kScanThreads * kScanItems;

// workspace header (int64 slots)
enum { H_ITEMS = 0, H_NREC, H_POOL, H_STATUS, H_MAX_GROUPS, H_SIZES, H_SIZES1, H_SIZES2, H_MAX_GROUPS32, H_WORDS = 32 };

struct Layout {
    int n = 0, max_m = 0, gpus = 0;
    int64_t total = 0;            // compositions of all stage counts
    int64_t items = 0;            // bound on (range, composition) pairs of one window
    size_t table = 0, first = 0, base = 0, offs = 0, ngroups = 0, rows = 0, ranges = 0, rlo = 0, ritem = 0, rbyte = 0,
           irec = 0, ipool = 0, partials = 0, bytes = 0;
};

int64_t scan_blocks(int64_t n) { return (n + kScanTile - 1) / kScanTile; }

// the counting table, the first shape and first composition of every stage count, and the workspace layout
int plan_listing(const MetisListing *l, std::vector<int64_t> &table, std::vector<int32_t> &first,
                 std::vector<int64_t> &base, Layout &lay) {
    if (!l) return fail_arg("listing is NULL");
    if (l->first_stage < 1 || l->last_stage < l->first_stage || l->last_stage > METIS_MAX_STAGES)
        return fail_arg("stage counts out of range (1 .. METIS_MAX_STAGES)");
    if (l->num_gpus < 1 || l->num_gpus > 8192) return fail_arg("num_gpus out of range (1 .. 8192)");
    if (l->max_permute_len < 1 || l->max_ranges < 1) return fail_arg("max_permute_len / max_ranges must be positive");
    lay.n = l->last_stage - l->first_stage + 1;
    lay.max_m = l->last_stage;
    lay.gpus = l->num_gpus;
    const int top = comp_top_shape(l->num_gpus);
    table.assign((size_t)comp_table_at(top + 2, 0, 0, lay.gpus, lay.max_m), 0);
    comp_fill_table(table.data(), lay.gpus, lay.max_m);
    first.assign(lay.n, 0);
    base.assign(lay.n + 1, 0);
    for (int i = 0; i < lay.n; ++i) {
        const int S = l->first_stage + i;
        first[i] = comp_first_shape(S, l->num_gpus, l->variance);
        const int64_t comps = first[i] < 0 ? 0 : table[comp_table_at(first[i], lay.gpus, S, lay.gpus, lay.max_m)];
        if (first[i] < 0) first[i] = 0;
        base[i + 1] = base[i] + comps;
    }
    lay.total = base[lay.n];
    lay.items = lay.total + l->max_ranges;
    const int64_t scan_max = (lay.items > lay.total ? lay.items : lay.total) + 1;
    size_t o = align256(H_WORDS * 8);
    lay.table = o;    o = align256(o + table.size() * 8);
    lay.first = o;    o = align256(o + first.size() * 4);
    lay.base = o;     o = align256(o + base.size() * 8);
    lay.offs = o;     o = align256(o + (size_t)(lay.total + 1) * 8);
    lay.ngroups = o;  o = align256(o + (size_t)lay.total + 1);
    lay.rows = o;     o = align256(o + (size_t)lay.n * 8);
    lay.ranges = o;   o = align256(o + (size_t)l->max_ranges * sizeof(MetisRowRange));
    lay.rlo = o;      o = align256(o + (size_t)l->max_ranges * 8);
    lay.ritem = o;    o = align256(o + (size_t)(l->max_ranges + 1) * 8);
    lay.rbyte = o;    o = align256(o + (size_t)l->max_ranges * 8);
    lay.irec = o;     o = align256(o + (size_t)(lay.items + 1) * 8);
    lay.ipool = o;    o = align256(o + (size_t)(lay.items + 1) * 8);
    lay.partials = o; o = align256(o + (size_t)(scan_blocks(scan_max) + 1) * 8);
    lay.bytes = o;
    return METIS_OK;
}

template <class T> T *at(void *ws, size_t off) { return reinterpret_cast<T *>(static_cast<uint8_t *>(ws) + off); }

// ---- prefix sums: in place, inclusive, over a[0 .. n) with n = *n_dev (n_dev != NULL) or n_host ----------------------
__global__ void __launch_bounds__(kScanThreads)
scan_tiles_kernel(int64_t *a, const int64_t *n_dev, int64_t n_host, int64_t *partials) {
    __shared__ int64_t sh[kScanThreads];
    const int64_t n = n_dev ? *n_dev : n_host;
    const int64_t t0 = (int64_t)blockIdx.x * kScanTile + (int64_t)threadIdx.x * kScanItems;
    int64_t v[kScanItems], sum = 0;
    for (int k = 0; k < kScanItems; ++k) {
        sum += (t0 + k < n) ? a[t0 + k] : 0;
        v[k] = sum;
    }
    sh[threadIdx.x] = sum;
    __syncthreads();
    for (int d = 1; d < kScanThreads; d <<= 1) {               // Hillis-Steele over the thread sums
        const int64_t add = threadIdx.x >= (unsigned)d ? sh[threadIdx.x - d] : 0;
        __syncthreads();
        sh[threadIdx.x] += add;
        __syncthreads();
    }
    const int64_t before = threadIdx.x ? sh[threadIdx.x - 1] : 0;
    for (int k = 0; k < kScanItems; ++k)
        if (t0 + k < n) a[t0 + k] = v[k] + before;
    if (threadIdx.x == kScanThreads - 1) partials[blockIdx.x] = sh[kScanThreads - 1];
}

__global__ void __launch_bounds__(1024) scan_partials_kernel(int64_t *partials, int64_t nb) {   // -> exclusive
    __shared__ int64_t sh[1024];
    const int64_t chunk = (nb + 1023) / 1024, lo = threadIdx.x * chunk, hi = lo + chunk < nb ? lo + chunk : nb;
    int64_t sum = 0;
    for (int64_t i = lo; i < hi; ++i) sum += partials[i];
    sh[threadIdx.x] = sum;
    __syncthreads();
    for (int d = 1; d < 1024; d <<= 1) {
        const int64_t add = threadIdx.x >= (unsigned)d ? sh[threadIdx.x - d] : 0;
        __syncthreads();
        sh[threadIdx.x] += add;
        __syncthreads();
    }
    int64_t run = threadIdx.x ? sh[threadIdx.x - 1] : 0;
    for (int64_t i = lo; i < hi; ++i) {
        const int64_t x = partials[i];
        partials[i] = run;
        run += x;
    }
}

__global__ void __launch_bounds__(kScanThreads)
scan_add_kernel(int64_t *a, const int64_t *n_dev, int64_t n_host, const int64_t *partials) {
    const int64_t n = n_dev ? *n_dev : n_host;
    const int64_t add = partials[blockIdx.x];
    const int64_t t0 = (int64_t)blockIdx.x * kScanTile;
    for (int k = threadIdx.x; k < kScanTile; k += kScanThreads)
        if (t0 + k < n) a[t0 + k] += add;
}

int scan(int64_t *a, const int64_t *n_dev, int64_t n_bound, int64_t *partials, cudaStream_t st) {
    const int64_t nb = scan_blocks(n_bound);
    if (nb == 0) return METIS_OK;
    if (nb > 0x7FFFFFFFLL) return fail_arg("too many items for one scan");
    scan_tiles_kernel<<<(unsigned)nb, kScanThreads, 0, st>>>(a, n_dev, n_bound, partials);
    scan_partials_kernel<<<1, 1024, 0, st>>>(partials, nb);
    scan_add_kernel<<<(unsigned)nb, kScanThreads, 0, st>>>(a, n_dev, n_bound, partials);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? METIS_OK : fail_cuda(e, "scan kernels");
}

// ---- listing -------------------------------------------------------------------------------------------------------
struct ListArgs {
    const int64_t *N;
    const int32_t *first;         // first shape of each stage count
    const int64_t *base;          // first composition of each stage count (n + 1 entries)
    int64_t *offs;                // [total + 1]: permutations of c at c + 1; after the scan, the rows before c
    uint8_t *ngroups;
    int n, first_stage, gpus, max_m, mpl;
    int64_t total;
};

__device__ int stage_of(const int64_t *base, int n, int64_t c) {     // base[s] <= c < base[s + 1]
    int lo = 0, hi = n;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (base[mid] <= c) lo = mid; else hi = mid;
    }
    return lo;
}

__global__ void __launch_bounds__(kListThreads) list_comps_kernel(ListArgs a, unsigned long long *hdr) {
    uint8_t codes[METIS_MAX_STAGES];
    CompSlice g[METIS_MAX_STAGES], tmp[METIS_MAX_STAGES];
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < a.total; c += (int64_t)gridDim.x * blockDim.x) {
        const int s = stage_of(a.base, a.n, c);
        const int S = a.first_stage + s;
        comp_unrank(a.N, a.gpus, a.max_m, a.first[s], S, c - a.base[s], codes);
        const int n = comp_merge(codes, S, a.mpl, g, tmp);
        a.offs[c + 1] = comp_perm_count(codes, g, n);
        a.ngroups[c] = (uint8_t)n;                             // n <= S <= METIS_MAX_STAGES
        atomicMax(&hdr[H_MAX_GROUPS], (unsigned long long)n);
    }
}

__global__ void stage_rows_kernel(const int64_t *base, const int64_t *offs, int n, int64_t *rows, int64_t *hdr) {
    for (int s = threadIdx.x; s < n; s += blockDim.x) rows[s] = offs[base[s + 1]] - offs[base[s]];
    if (threadIdx.x == 0) reinterpret_cast<int32_t *>(hdr + H_MAX_GROUPS32)[0] = (int32_t)hdr[H_MAX_GROUPS];
}

// ---- one window ----------------------------------------------------------------------------------------------------
struct WindowArgs {
    ListArgs l;
    const MetisRowRange *ranges;
    int nr;
    int64_t *rlo, *ritem, *rbyte;  // per range: first composition, first item (nr + 1), byte offset in the window
    int64_t *irec, *ipool;         // per item (+1): records / pool bytes, scanned into offsets
    int64_t items_bound;
};

// one thread: the compositions each range overlaps, and where the range's rows start in the window
__global__ void window_ranges_kernel(WindowArgs w, int64_t *hdr) {
    int64_t item = 0, bytes = 0;
    for (int i = 0; i < w.nr; ++i) {
        const MetisRowRange r = w.ranges[i];
        const int s = r.stages - w.l.first_stage;
        int64_t lo = 0, hi = 0;
        bool ok = s >= 0 && s < w.l.n && r.first_row >= 0 && r.end_row >= r.first_row;
        if (ok) {
            const int64_t b = w.l.base[s], e = w.l.base[s + 1], o = w.l.offs[b];
            ok = r.end_row <= w.l.offs[e] - o;
            int64_t x = b, y = e;                              // first c with rows end (offs[c + 1] - o) > first_row
            while (x < y) { const int64_t m = (x + y) >> 1; if (w.l.offs[m + 1] - o > r.first_row) y = m; else x = m + 1; }
            lo = x;
            x = lo; y = e;                                     // first c with rows start (offs[c] - o) >= end_row
            while (x < y) { const int64_t m = (x + y) >> 1; if (w.l.offs[m] - o >= r.end_row) y = m; else x = m + 1; }
            hi = r.end_row > r.first_row ? x : lo;
        }
        if (!ok) { hdr[H_STATUS] |= 1; lo = hi = 0; }
        w.rlo[i] = lo;
        w.ritem[i] = item;
        w.rbyte[i] = bytes;
        item += hi - lo;
        if (ok) bytes += (r.end_row - r.first_row) * r.stages;
    }
    w.ritem[w.nr] = item;
    hdr[H_ITEMS] = item;
    w.irec[0] = w.ipool[0] = 0;
}

__device__ int range_of(const int64_t *ritem, int nr, int64_t item) {    // ritem[i] <= item < ritem[i + 1]
    int lo = 0, hi = nr;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (ritem[mid] <= item) lo = mid; else hi = mid;
    }
    return lo;
}

__global__ void __launch_bounds__(kListThreads) window_count_kernel(WindowArgs w, unsigned long long *hdr) {
    const int64_t items = (int64_t)hdr[H_ITEMS];
    for (int64_t it = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; it < items; it += (int64_t)gridDim.x * blockDim.x) {
        const int i = range_of(w.ritem, w.nr, it);
        const MetisRowRange r = w.ranges[i];
        const int s = r.stages - w.l.first_stage;
        const int64_t c = w.rlo[i] + (it - w.ritem[i]);
        const int n = w.l.ngroups[c];
        int64_t recs = 0, pool = 0;
        if (n > METIS_MAX_PERMUTE_GROUPS) {
            atomicOr(&hdr[H_STATUS], 2ull);
        } else {
            const int64_t o = w.l.offs[w.l.base[s]];
            recs = comp_slice_records(w.l.offs[c] - o, w.l.offs[c + 1] - w.l.offs[c], r.first_row, r.end_row, r.stages,
                                      n, 0, 0, nullptr);
            pool = n + r.stages;
        }
        w.irec[it + 1] = recs;
        w.ipool[it + 1] = pool;
    }
}

__global__ void window_totals_kernel(WindowArgs w, int64_t *hdr, int64_t recs_capacity, int64_t pool_capacity,
                                     int writing) {
    const int64_t items = hdr[H_ITEMS];
    hdr[H_NREC] = w.irec[items];
    hdr[H_POOL] = w.ipool[items];
    if (writing && (w.irec[items] > recs_capacity || w.ipool[items] > pool_capacity)) hdr[H_STATUS] |= 4;
    hdr[H_SIZES] = hdr[H_NREC];
    hdr[H_SIZES1] = hdr[H_POOL];
    hdr[H_SIZES2] = hdr[H_STATUS];
}

__global__ void __launch_bounds__(kListThreads)
window_write_kernel(WindowArgs w, const int64_t *hdr, MetisCompRec *recs, uint8_t *pool) {
    if (hdr[H_STATUS] & 4) return;
    const int64_t items = hdr[H_ITEMS];
    uint8_t codes[METIS_MAX_STAGES];
    CompSlice g[METIS_MAX_STAGES], tmp[METIS_MAX_STAGES];
    for (int64_t it = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; it < items; it += (int64_t)gridDim.x * blockDim.x) {
        const int i = range_of(w.ritem, w.nr, it);
        const MetisRowRange r = w.ranges[i];
        const int s = r.stages - w.l.first_stage;
        const int64_t c = w.rlo[i] + (it - w.ritem[i]);
        if (w.l.ngroups[c] > METIS_MAX_PERMUTE_GROUPS) continue;          // reported (status bit 1), never written
        comp_unrank(w.l.N, w.l.gpus, w.l.max_m, w.l.first[s], r.stages, c - w.l.base[s], codes);
        const int n = comp_merge(codes, r.stages, w.l.mpl, g, tmp);
        const int64_t at = w.ipool[it];
        comp_write_pool(codes, g, n, pool + at);
        const int64_t o = w.l.offs[w.l.base[s]];
        comp_slice_records(w.l.offs[c] - o, w.l.offs[c + 1] - w.l.offs[c], r.first_row, r.end_row, r.stages, n,
                           w.rbyte[i], (uint32_t)at, recs + w.irec[it]);
    }
}

ListArgs list_args(void *ws, const Layout &lay, const MetisListing *l) {
    ListArgs a;
    a.N = at<int64_t>(ws, lay.table);
    a.first = at<int32_t>(ws, lay.first);
    a.base = at<int64_t>(ws, lay.base);
    a.offs = at<int64_t>(ws, lay.offs);
    a.ngroups = at<uint8_t>(ws, lay.ngroups);
    a.n = lay.n;
    a.first_stage = l->first_stage;
    a.gpus = lay.gpus;
    a.max_m = lay.max_m;
    a.mpl = l->max_permute_len;
    a.total = lay.total;
    return a;
}

unsigned grid_for(int64_t n) {
    const int64_t b = (n + kListThreads - 1) / kListThreads;
    return (unsigned)(b < 1 ? 1 : (b > kListBlocks ? kListBlocks : b));
}

}  // namespace
}  // namespace metis

using namespace metis;

extern "C" {

int64_t metis_list_workspace_bytes(const MetisListing *listing, int64_t *comps_per_stage) {
    std::vector<int64_t> table, base;
    std::vector<int32_t> first;
    Layout lay;
    const int rc = plan_listing(listing, table, first, base, lay);
    if (rc) return rc;
    if (comps_per_stage)
        for (int i = 0; i < lay.n; ++i) comps_per_stage[i] = base[i + 1] - base[i];
    return (int64_t)lay.bytes;
}

int metis_list_stages(const MetisListing *listing, void *workspace, int64_t workspace_bytes, int64_t *rows_per_stage,
                      int32_t *max_groups, void *stream_) {
    std::vector<int64_t> table, base;
    std::vector<int32_t> first;
    Layout lay;
    const int rc = plan_listing(listing, table, first, base, lay);
    if (rc) return rc;
    if (!workspace || !rows_per_stage || !max_groups) return fail_arg("NULL argument");
    if (workspace_bytes < (int64_t)lay.bytes) return fail_arg("workspace too small (metis_list_workspace_bytes)");
    cudaStream_t st = static_cast<cudaStream_t>(stream_);
    // the host vectors die on return: cudaMemcpyAsync from pageable memory has staged them by then
    cudaError_t e = cudaMemsetAsync(workspace, 0, H_WORDS * 8, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(at<void>(workspace, lay.table), table.data(), table.size() * 8, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(at<void>(workspace, lay.first), first.data(), first.size() * 4, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(at<void>(workspace, lay.base), base.data(), base.size() * 8, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(at<void>(workspace, lay.offs), 0, 8, st);
    if (e != cudaSuccess) return fail_cuda(e, "listing tables");
    const ListArgs a = list_args(workspace, lay, listing);
    unsigned long long *hdr = at<unsigned long long>(workspace, 0);
    if (lay.total > 0) list_comps_kernel<<<grid_for(lay.total), kListThreads, 0, st>>>(a, hdr);
    e = cudaGetLastError();
    if (e != cudaSuccess) return fail_cuda(e, "list_comps_kernel");
    int r = scan(a.offs + 1, nullptr, lay.total, at<int64_t>(workspace, lay.partials), st);
    if (r) return r;
    int64_t *rows = at<int64_t>(workspace, lay.rows);
    stage_rows_kernel<<<1, 128, 0, st>>>(a.base, a.offs, lay.n, rows, at<int64_t>(workspace, 0));
    e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpyAsync(rows_per_stage, rows, (size_t)lay.n * 8, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess)
        e = cudaMemcpyAsync(max_groups, at<int64_t>(workspace, 0) + H_MAX_GROUPS32, 4, cudaMemcpyDeviceToHost, st);
    return e == cudaSuccess ? METIS_OK : fail_cuda(e, "stage_rows_kernel");
}

int metis_list_window(const MetisListing *listing, void *workspace, int64_t workspace_bytes, const MetisRowRange *ranges,
                      int32_t num_ranges, MetisCompRec *recs, int64_t recs_capacity, uint8_t *pool,
                      int64_t pool_capacity, int64_t *sizes, void *stream_) {
    std::vector<int64_t> table, base;
    std::vector<int32_t> first;
    Layout lay;
    const int rc = plan_listing(listing, table, first, base, lay);
    if (rc) return rc;
    if (!workspace || !sizes || (num_ranges > 0 && !ranges)) return fail_arg("NULL argument");
    if (num_ranges < 0 || num_ranges > listing->max_ranges) return fail_arg("num_ranges out of range (0 .. max_ranges)");
    if (workspace_bytes < (int64_t)lay.bytes) return fail_arg("workspace too small (metis_list_workspace_bytes)");
    const int writing = recs != nullptr;
    if (writing && (!pool || recs_capacity < 0 || pool_capacity < 0)) return fail_arg("recs without pool");
    cudaStream_t st = static_cast<cudaStream_t>(stream_);
    WindowArgs w;
    w.l = list_args(workspace, lay, listing);
    w.ranges = at<MetisRowRange>(workspace, lay.ranges);
    w.nr = num_ranges;
    w.rlo = at<int64_t>(workspace, lay.rlo);
    w.ritem = at<int64_t>(workspace, lay.ritem);
    w.rbyte = at<int64_t>(workspace, lay.rbyte);
    w.irec = at<int64_t>(workspace, lay.irec);
    w.ipool = at<int64_t>(workspace, lay.ipool);
    w.items_bound = lay.items;
    int64_t *hdr = at<int64_t>(workspace, 0);
    cudaError_t e = cudaMemsetAsync(hdr + H_STATUS, 0, 8, st);
    if (e == cudaSuccess && num_ranges > 0)
        e = cudaMemcpyAsync(at<void>(workspace, lay.ranges), ranges, (size_t)num_ranges * sizeof(MetisRowRange),
                            cudaMemcpyHostToDevice, st);
    if (e != cudaSuccess) return fail_cuda(e, "window ranges");
    window_ranges_kernel<<<1, 1, 0, st>>>(w, hdr);
    window_count_kernel<<<grid_for(lay.items), kListThreads, 0, st>>>(w, reinterpret_cast<unsigned long long *>(hdr));
    e = cudaGetLastError();
    if (e != cudaSuccess) return fail_cuda(e, "window_count_kernel");
    int r = scan(w.irec + 1, hdr + H_ITEMS, lay.items, at<int64_t>(workspace, lay.partials), st);
    if (!r) r = scan(w.ipool + 1, hdr + H_ITEMS, lay.items, at<int64_t>(workspace, lay.partials), st);
    if (r) return r;
    window_totals_kernel<<<1, 1, 0, st>>>(w, hdr, recs_capacity, pool_capacity, writing);
    if (writing) window_write_kernel<<<grid_for(lay.items), kListThreads, 0, st>>>(w, hdr, recs, pool);
    e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpyAsync(sizes, hdr + H_SIZES, 24, cudaMemcpyDeviceToHost, st);
    return e == cudaSuccess ? METIS_OK : fail_cuda(e, "window kernels");
}

}  // extern "C"
