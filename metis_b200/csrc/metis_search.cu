// metis_search.cu - sm_90a kernels + C ABI of libmetis_b200.so (see include/metis_b200.h).
//
// Kernel map (SURVEY.md section 8a):
//   het_rows_kernel       a3/a4: device-group rows of every composition, in the reference's visiting order
//                         (metis_rows.cuh; once per plan space, not per search)
//   pack_tables_kernel    flattens the profile tables into one 16 B-aligned blob (+ norm_lc/7, derived tables)
//   range_sums_kernel     sum(row[a:b]) of every profile row and slice, as CPython adds it up (looked up by a5..a16)
//   het_admit_kernel      a2: ordinal -> plan, plans without a valid strategy dropped, survivors listed with a
//                         chain-length hint
//   het_scatter_kernel    counting sort of the list: by stage count (bulk round next) or by hint (chain kernel only)
//   het_first_kernel      a5..a16, bulk round: first partition attempt of every listed plan, one plan per thread,
//                         lanes re-joined explicitly (policy Lockstep, metis_eval.cuh); plans that run out of memory
//                         are re-weighted and handed to the chain kernel
//   het_order_kernel      those continuations by hint, longest expected chain first
//   het_chain_kernel      a5..a16: one warp per plan walks the whole strategy chain (metis_coop.cuh);
//                         both evaluation kernels stage the tables into shared memory by one TMA bulk copy
//                         (cp.async.bulk + mbarrier) per block, write a 16 B record per costed candidate and
//                         reduce their best candidate by warp shuffles + shared memory
//   het_finalize_kernel   grid argmin over the per-block bests, counters -> summary
//   het_detail_kernel     replays chosen (ordinal, step) candidates to materialise strategies/partition
//   het_trace_kernel      replays plans and records what the reference prints (metis_trace.cuh)
//   homo_cost_kernel      a17: one thread per UniformPlan
//   layer_balance_kernel  a10 alone, for unit parity
//   (rank_records_kernel, the stable record sort, lives in metis_rank.cu)
//
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -fmad=false (no FMA contraction: parity).
#include <cuda_runtime.h>
#include <cooperative_groups.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "metis_eval.cuh"
#include "metis_coop.cuh"
#include "metis_warp.cuh"
#include "metis_trace.cuh"
#include "metis_rows.cuh"

namespace cg = cooperative_groups;

namespace metis {

// bulk-round block shape: 256 threads, >= 3 blocks/SM, i.e. at most 80 registers (3 x 256 x 80 fits the 64 Ki
// registers of an H100 SM); the other choices were 128 x 6 and 256 x 4
#ifndef METIS_THREADS
#define METIS_THREADS 256
#endif
#ifndef METIS_MIN_BLOCKS
#define METIS_MIN_BLOCKS 3
#endif
// instantiations for more than 64 stages: 80 registers cost some spills and buy a third block per SM; single-type
// clusters take a fourth one at 64 registers (more spills, more warps), mixed-type ones keep three
#ifndef METIS_MIN_BLOCKS_BIG
#define METIS_MIN_BLOCKS_BIG METIS_MIN_BLOCKS
#endif
#ifndef METIS_MIN_BLOCKS_BIG_ONE
#define METIS_MIN_BLOCKS_BIG_ONE (METIS_MIN_BLOCKS + 1)
#endif
constexpr int kThreads = METIS_THREADS;
constexpr int kMaxS = METIS_MAX_STAGES;
constexpr int kMaxL = METIS_MAX_LAYERS;
constexpr int kSmemBlobMax = 160 * 1024;

static thread_local char g_err[256] = "";
static thread_local cudaEvent_t g_ev_before = nullptr, g_ev_after = nullptr;

static int cuda_fail(cudaError_t e, const char *what) {
    snprintf(g_err, sizeof(g_err), "%s: %s", what, cudaGetErrorString(e));
    return METIS_E_CUDA;
}
static int arg_fail(const char *what) {
    snprintf(g_err, sizeof(g_err), "%s", what);
    return METIS_E_ARG;
}
int fail_cuda(cudaError_t e, const char *what) { return cuda_fail(e, what); }   // metis_internal.h
int fail_arg(const char *what) { return arg_fail(what); }

struct BlobLayout {
    uint32_t total;               // bytes staged into shared memory
    uint32_t key, lc, mem, exec_full, fb, norm, derived, tmem, bwf, bwm, runt, rune, q10e;
    uint32_t rsum, rsum_bytes;    // range-sum tables (Tables::rsum): behind the staged part, read from L2
};

static uint32_t align16(uint32_t v) { return (v + 15u) & ~15u; }

static BlobLayout make_layout(const MetisProblem &p) {
    BlobLayout l;
    uint32_t o = 0;
    const uint32_t nkey = (uint32_t)p.num_types * p.num_tp * p.num_bs;
    l.key = o;       o = align16(o + nkey * 2);
    l.lc = o;        o = align16(o + (uint32_t)p.num_keys * p.lpad * 8);
    l.mem = o;       o = align16(o + (uint32_t)p.num_keys * p.lpad * 8);
    l.exec_full = o; o = align16(o + (uint32_t)p.num_keys * 8);
    l.fb = o;        o = align16(o + (uint32_t)p.num_keys * 8);
    l.norm = o;      o = align16(o + (uint32_t)p.norm_len * 8);
    l.derived = o;   o = align16(o + (uint32_t)derived_layout(p).total * 8);
    l.tmem = o;      o = align16(o + (uint32_t)p.num_types * 8);
    l.bwf = o;       o = align16(o + (uint32_t)p.num_types * 8);
    l.bwm = o;       o = align16(o + (uint32_t)p.num_types * 8);
    l.runt = o;      o = align16(o + (uint32_t)p.num_node_sequences * p.num_types);
    l.rune = o;      o = align16(o + (uint32_t)p.num_node_sequences * p.num_types * 4);
    l.q10e = o;      o = align16(o + (uint32_t)p.num_node_sequences * p.num_types * 4);
    l.total = o;
    const uint64_t n = (uint64_t)p.num_layers + 1;
    l.rsum = (o + 127u) & ~127u;
    l.rsum_bytes = (uint32_t)((uint64_t)(2 * p.num_keys + 1) * n * n * 8);    // <= 2 * 255 keys... checked in check_problem
    return l;
}

// `base`: the staged tables (shared or global memory); `gblob`: the blob in global memory when its range-sum tables
// were filled for this launch (search kernels), else nullptr
__device__ __forceinline__ Tables make_tables(const MetisProblem &p, const BlobLayout &l, const uint8_t *base,
                                              const uint8_t *gblob = nullptr) {
    Tables T;
    T.p = p;
    T.rsum = gblob ? reinterpret_cast<const double *>(gblob + l.rsum) : nullptr;
    T.key_index = reinterpret_cast<const int16_t *>(base + l.key);
    T.lc = reinterpret_cast<const double *>(base + l.lc);
    T.mem = reinterpret_cast<const double *>(base + l.mem);
    T.exec_full = reinterpret_cast<const double *>(base + l.exec_full);
    T.fb_sync = reinterpret_cast<const double *>(base + l.fb);
    T.norm_lc = reinterpret_cast<const double *>(base + l.norm);
    bind_derived(T, reinterpret_cast<const double *>(base + l.derived));
    T.type_memory = reinterpret_cast<const double *>(base + l.tmem);
    T.bw_first = reinterpret_cast<const double *>(base + l.bwf);
    T.bw_min = reinterpret_cast<const double *>(base + l.bwm);
    T.run_type = base + l.runt;
    T.run_end = reinterpret_cast<const int32_t *>(base + l.rune);
    T.q10_end = reinterpret_cast<const int32_t *>(base + l.q10e);
    return T;
}

__device__ __forceinline__ void copy_bytes(uint8_t *dst, const void *src, uint32_t n, uint32_t tid, uint32_t nthr) {
    const uint8_t *s = static_cast<const uint8_t *>(src);
    for (uint32_t i = tid; i < n; i += nthr) dst[i] = s[i];
}

__global__ void pack_tables_kernel(MetisProblem p, BlobLayout l, uint8_t *blob) {
    const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x, nthr = gridDim.x * blockDim.x;
    const uint32_t nkey = (uint32_t)p.num_types * p.num_tp * p.num_bs;
    copy_bytes(blob + l.key, p.key_index, nkey * 2, tid, nthr);
    copy_bytes(blob + l.lc, p.layer_compute, (uint32_t)p.num_keys * p.lpad * 8, tid, nthr);
    copy_bytes(blob + l.mem, p.layer_memory, (uint32_t)p.num_keys * p.lpad * 8, tid, nthr);
    copy_bytes(blob + l.exec_full, p.exec_full, (uint32_t)p.num_keys * 8, tid, nthr);
    copy_bytes(blob + l.fb, p.fb_sync, (uint32_t)p.num_keys * 8, tid, nthr);
    copy_bytes(blob + l.norm, p.norm_lc, (uint32_t)p.norm_len * 8, tid, nthr);
    copy_bytes(blob + l.tmem, p.type_memory, (uint32_t)p.num_types * 8, tid, nthr);
    copy_bytes(blob + l.bwf, p.type_bw_first, (uint32_t)p.num_types * 8, tid, nthr);
    copy_bytes(blob + l.bwm, p.type_bw_min, (uint32_t)p.num_types * 8, tid, nthr);
    copy_bytes(blob + l.runt, p.ns_run_type, (uint32_t)p.num_node_sequences * p.num_types, tid, nthr);
    copy_bytes(blob + l.rune, p.ns_run_end, (uint32_t)p.num_node_sequences * p.num_types * 4, tid, nthr);
    copy_bytes(blob + l.q10e, p.ns_q10_end, (uint32_t)p.num_node_sequences * p.num_types * 4, tid, nthr);
    // derived tables: each entry is one IEEE operation of the reference, evaluated once per launch
    double *derived = reinterpret_cast<double *>(blob + l.derived);
    const DerivedLayout d = derived_layout(p);
    for (uint32_t i = tid; i < (uint32_t)d.total; i += nthr)
        derived[i] = derive_entry(p, d, p.norm_lc, p.exec_full, p.type_bw_first, (int)i);
}

// Range-sum tables (metis_eval.cuh, fill_range_sums): one thread per (row, first layer) adds the row up once and
// stores the sum of every slice that starts there; neighbouring threads write neighbouring addresses.
__global__ void __launch_bounds__(128)
range_sums_kernel(MetisProblem p, BlobLayout l, uint8_t *blob) {
    const int L = p.num_layers;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)range_sum_tables(p) * L) return;
    const int t = (int)(i / L), a = (int)(i % L);
    const double *row = range_sum_row(p, t, p.layer_memory, p.layer_compute, p.norm_lc);
    if (!row) return;
    const size_t n = (size_t)L + 1;
    fill_range_sums(row, L, a, reinterpret_cast<double *>(blob + l.rsum) + (size_t)t * n * n);
}

// ---- TMA 1-D bulk copy global -> shared, completion on an mbarrier --------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ void stage_blob_tma(uint8_t *smem, const uint8_t *blob, uint32_t bytes, uint64_t *mbar) {
    const uint32_t bar = smem_u32(mbar);
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar) : "memory");
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
        constexpr uint32_t kChunk = 32768;
        for (uint32_t off = 0; off < bytes; off += kChunk) {
            const uint32_t n = (bytes - off < kChunk) ? bytes - off : kChunk;
            asm volatile(
                "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                ::"r"(smem_u32(smem + off)), "l"(blob + off), "r"(n), "r"(bar)
                : "memory");
        }
    }
    uint32_t done = 0;
    while (!done) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(bar)
            : "memory");
    }
}

// ---- ordinal -> plan ---------------------------------------------------------------------------
__device__ __forceinline__ int find_block(const MetisPlanSpace &sp, int64_t ordinal) {
    int lo = 0, hi = sp.num_blocks - 1;
    while (lo < hi) {                                         // last block with first_ordinal <= ordinal
        const int mid = (lo + hi + 1) >> 1;
        if (__ldg(&sp.blocks[mid].first_ordinal) <= ordinal) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// `hint` >= 0: a block known to start at or before `ordinal` (the warp's first plan); blocks are walked
// forward from it, so the 32 consecutive plans of a warp cost one binary search instead of 32.
__device__ __forceinline__ bool decode_plan(const MetisPlanSpace &sp, int64_t ordinal, PlanDesc &pd, int hint = -1) {
    if (ordinal < 0 || ordinal >= sp.num_plans) return false;
    int lo;
    if (hint >= 0) {
        lo = hint;
        while (lo + 1 < sp.num_blocks && __ldg(&sp.blocks[lo + 1].first_ordinal) <= ordinal) ++lo;
    } else {
        lo = find_block(sp, ordinal);
    }
    const MetisPlanBlock b = sp.blocks[lo];
    const int64_t rel = ordinal - b.first_ordinal;
    const int64_t row = rel / sp.num_div;
    const int div = (int)(rel - row * sp.num_div);
    pd.ordinal = (uint32_t)ordinal;
    pd.ns = b.ns_idx;
    pd.S = b.num_stage;
    pd.label = b.label_stage;
    pd.batches = __ldg(&sp.batches[div]);
    const int64_t off = b.rows_offset + row * b.num_stage;
    pd.row = sp.rows + off;
    pd.geo = pack_geo(off, b.num_stage, b.label_stage, b.ns_idx, div);
    return true;
}

// task list entry -> plan (no block search: the geometry word was stored at admission)
__device__ __forceinline__ void decode_task(const MetisPlanSpace &sp, uint64_t hdr, uint64_t geo, PlanDesc &pd) {
    pd.ordinal = (uint32_t)hdr;
    pd.geo = geo;
    pd.row = sp.rows + (geo & 0xFFFFFFFFULL);
    pd.S = (int)((geo >> 32) & 0xFF) + 1;
    pd.label = (int)((geo >> 40) & 0xFF) + 1;
    pd.ns = (int)((geo >> 48) & 0xFF);
    pd.batches = __ldg(&sp.batches[(geo >> 56) & 0xFF]);
}

__device__ __forceinline__ bool rec_less(double c0, uint32_t o0, uint32_t s0, double c1, uint32_t o1, uint32_t s1) {
    if (c0 < c1) return true;
    if (c0 > c1) return false;
    if (o0 != o1) return o0 < o1;
    return s0 < s1;
}

struct DeviceOut {
    MetisRecord *records;
    long long capacity;
    uint8_t *detail;
    int detail_stride;
    unsigned long long *counters;   // [0] records [1] partition calls [2] balancer runs [3] keyerrors [4] fatal key
    MetisRecord *block_best;
};

struct DeviceSink {
    const DeviceOut &o;
    unsigned int n_part, n_run, n_key;
    double best_cost;
    uint32_t best_ord, best_step, best_meta;
    bool leader;                    // chain kernel: only lane 0 of the warp produces side effects
    __device__ DeviceSink(const DeviceOut &out)
        : o(out), n_part(0), n_run(0), n_key(0), best_cost(INFINITY), best_ord(0xFFFFFFFFu), best_step(0xFFFFu),
          best_meta(0), leader(true) {}
    __device__ void phase(int) {}
    __device__ void partition_call() { n_part += leader ? 1u : 0u; }
    __device__ void balancer_run() { n_run += leader ? 1u : 0u; }
    __device__ void keyerror() { n_key += leader ? 1u : 0u; }
    // lowest ordinal wins; among several fatal conditions of one plan the earliest (first raised) is kept by the
    // caller order: a plan reports at most one fatal condition (its evaluation stops there)
    __device__ void fatal(uint32_t ordinal, int code, uint32_t aux) {
        if (!leader) return;
        const unsigned long long key = ((unsigned long long)ordinal << 32) | ((unsigned long long)(code & 0xFF) << 24) |
                                       (unsigned long long)(((aux >> 16) & 0xFF) << 16) | (aux & 0xFFFF);
        atomicMin(&o.counters[4], key);
    }
    __device__ void emit(const PlanDesc &pd, int step, int nrep, double cost, const uint8_t *tpc, const uint16_t *part) {
        if (!leader) return;
        const unsigned long long slot = atomicAdd(&o.counters[0], 1ULL);
        if ((long long)slot < o.capacity) {
            MetisRecord r;
            r.cost = cost; r.ordinal = pd.ordinal; r.step = (uint16_t)step;
            r.num_repartition = (uint8_t)nrep; r.num_stage = (uint8_t)pd.S;
            o.records[slot] = r;
            if (o.detail) {
                uint8_t *d = o.detail + (size_t)slot * o.detail_stride;
                for (int s = 0; s < pd.S; ++s) { d[s] = (uint8_t)(pd.row[s] - tpc[s]); d[pd.S + s] = tpc[s]; }
                for (int s = 0; s <= pd.S; ++s) d[2 * pd.S + s] = (uint8_t)part[s];
            }
        }
        if (rec_less(cost, pd.ordinal, (uint32_t)step, best_cost, best_ord, best_step)) {
            best_cost = cost; best_ord = pd.ordinal; best_step = (uint32_t)step;
            best_meta = ((uint32_t)nrep << 8) | (uint32_t)pd.S;
        }
    }
};

// End of a search kernel: counters (warp reduce, one atomic per warp) and the block's best candidate:
// argmin (cost, ordinal, step) by __shfl_xor_sync inside the warp, then across the warps through shared memory.
__device__ __forceinline__ void finish_block(const DeviceSink &sink, const DeviceOut &out, int slot) {
    __shared__ double s_cost[32];
    __shared__ uint32_t s_ord[32], s_step[32], s_meta[32];
    const unsigned full = 0xFFFFFFFFu;
    const unsigned np = __reduce_add_sync(full, sink.n_part);
    const unsigned nr = __reduce_add_sync(full, sink.n_run);
    const unsigned nk = __reduce_add_sync(full, sink.n_key);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) {
        if (np) atomicAdd(&out.counters[1], (unsigned long long)np);
        if (nr) atomicAdd(&out.counters[2], (unsigned long long)nr);
        if (nk) atomicAdd(&out.counters[3], (unsigned long long)nk);
    }
    double c = sink.best_cost;
    uint32_t o = sink.best_ord, st = sink.best_step, mt = sink.best_meta;
    for (int d = 16; d > 0; d >>= 1) {
        const double c2 = __shfl_xor_sync(full, c, d);
        const uint32_t o2 = __shfl_xor_sync(full, o, d), s2 = __shfl_xor_sync(full, st, d),
                       m2 = __shfl_xor_sync(full, mt, d);
        if (rec_less(c2, o2, s2, c, o, st)) { c = c2; o = o2; st = s2; mt = m2; }
    }
    if (lane == 0) { s_cost[warp] = c; s_ord[warp] = o; s_step[warp] = st; s_meta[warp] = mt; }
    __syncthreads();
    if (threadIdx.x == 0) {
        const int nw = (blockDim.x + 31) >> 5;
        for (int wi = 1; wi < nw; ++wi)
            if (rec_less(s_cost[wi], s_ord[wi], s_step[wi], c, o, st)) { c = s_cost[wi]; o = s_ord[wi]; st = s_step[wi]; mt = s_meta[wi]; }
        MetisRecord r;
        r.cost = c; r.ordinal = o; r.step = (uint16_t)st; r.num_repartition = (uint8_t)(mt >> 8); r.num_stage = (uint8_t)mt;
        out.block_best[slot] = r;
    }
}

// ---- the search, four kernels on one stream (DESIGN.md section 4) ---------------------------------------
//   het_admit_kernel    one thread per inter-stage plan: decode, first strategy that can be valid, drop the plans
//                       that have none (78 % at BASELINE configs[2]); survivors -> list A + histogram of stage counts
//   het_scatter_kernel  counting sort of list A by stage count, longest first -> list B
//   het_first_kernel    bulk round: first partition attempt of every listed plan, one plan per thread, 32 plans of
//                       equal stage count per warp in lockstep; plans that run out of memory -> list C
//   het_chain_kernel    one warp per plan: the whole strategy chain, depth first (metis_coop.cuh), over list C -
//                       or over list B when the list is too short to fill the bulk round
// List entry: (ordinal, flags, geometry word); flags bit 0 = first attempt already counted by the bulk round.
struct SearchLists {
    uint4 *a, *b;                 // list C reuses the storage of list A
    unsigned int *ctl;            // [0] admitted [1] bulk fetch cursor [2] continuations [3] chain fetch cursor
                                  // [16..16+128) histogram by stage count, [160+16..) scatter cursors
    long long bulk_min;           // lists shorter than this skip the bulk round
    // hand-over of the bulk round's failed first attempts (CoopEvaluator::kRetry): the re-weighted stage performance of
    // continuation c, stage s, at perf[s * save_cap + c] for c < save_cap (later continuations replay the attempt);
    // src[i] = c of the i-th entry of list B after het_order_kernel
    double *perf;
    unsigned int *src;
    unsigned int save_cap;
};
// list entry flags: bit 0 = first attempt counted by the bulk round, bits 1-2 = CoopEvaluator::Start, bits 8-14 = hint
constexpr int kCtlHist = 16, kCtlCursor = 16 + 160;
constexpr int kCtlHist2 = 512, kCtlCursor2 = 512 + 160;   // ordering of the continuations by chain hint
constexpr int kCtlHist3 = 832, kCtlCursor3 = 832 + 160;   // ordering of the admitted plans by chain hint (no bulk round)
constexpr unsigned kHintMax = 127;

__device__ __forceinline__ uint4 make_entry(uint32_t ordinal, uint32_t flags, uint64_t geo) {
    return make_uint4(ordinal, flags, (uint32_t)geo, (uint32_t)(geo >> 32));
}
__device__ __forceinline__ void decode_entry(const MetisPlanSpace &sp, const uint4 e, PlanDesc &pd) {
    decode_task(sp, (uint64_t)e.x, ((uint64_t)e.w << 32) | e.z, pd);
}

__global__ void __launch_bounds__(256)
het_admit_kernel(const __grid_constant__ MetisPlanSpace sp, const MetisShard sh, const long long slots,
                 const int gbs, const int max_bs, const int max_tp, const SearchLists ls) {
    const int lane = threadIdx.x & 31;
    const long long b0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) & ~31LL;   // the warp's first slot
    if (b0 >= slots) return;
    // tiles are multiples of 32, so a warp's 32 plans are consecutive ordinals
    const long long first = ((b0 / sh.tile) * sh.world + sh.rank) * sh.tile + (b0 % sh.tile);
    int hint = 0;
    if (lane == 0 && first < sp.num_plans) hint = find_block(sp, first);
    hint = __shfl_sync(0xFFFFFFFFu, hint, 0);
    PlanDesc pd;
    int halvings = 0;
    bool ok = b0 + lane < slots && decode_plan(sp, first + lane, pd, hint);
    if (ok) {
        // PlanEvaluator::begin: tp_s = max(1, group_s / B), B = 2^floor(log2(gbs // batches)); the plan has a
        // valid strategy iff that one is valid (search_space/plan.py:238-249)
        const int bs_total = gbs / pd.batches;
        const int lb = 31 - __clz(bs_total > 0 ? bs_total : 1);
        const int ltp = 31 - __clz(max_tp > 0 ? max_tp : 1), lbs = 31 - __clz(max_bs > 0 ? max_bs : 1);
        if (bs_total <= 0) ok = false;
        for (int s = 0; ok && s < pd.S; ++s) {
            const int g = __ldg(&pd.row[s]);
            const int t = g > lb ? g - lb : 0;
            const int mbs = bs_total >> (g - t);
            if (mbs == 0 || mbs > max_bs || (1 << t) > max_tp) ok = false;
            else {                                           // PlanEvaluator::halvings (scheduling hint)
                const int lm = 31 - __clz(mbs);
                int room = g - t;
                room = min(room, min(ltp - t, lbs - lm));
                if (room > 0) halvings += room;
            }
        }
    }
    const unsigned full = 0xFFFFFFFFu;
    const unsigned m = __ballot_sync(full, ok);
    if (m == 0) return;
    const int leader = __ffs(m) - 1;
    unsigned int base = 0;
    if (lane == leader) base = atomicAdd(&ls.ctl[0], (unsigned int)__popc(m));
    base = __shfl_sync(full, base, leader);
    const int k = ok ? pd.S - 1 : -1;
    const unsigned peers = __match_any_sync(full, k);        // neighbours mostly share the stage count
    const unsigned key = (unsigned)halvings > kHintMax ? kHintMax : (unsigned)halvings;
    const unsigned peers3 = __match_any_sync(full, ok ? (int)key : -1);
    if (ok) {
        ls.a[base + __popc(m & ((1u << lane) - 1u))] = make_entry(pd.ordinal, key << 8, pd.geo);
        if (lane == __ffs(peers) - 1) atomicAdd(&ls.ctl[kCtlHist + k], (unsigned int)__popc(peers));
        if (lane == __ffs(peers3) - 1) atomicAdd(&ls.ctl[kCtlHist3 + key], (unsigned int)__popc(peers3));
    }
}

__global__ void __launch_bounds__(256)
het_scatter_kernel(const SearchLists ls) {
    __shared__ unsigned int s_base[160];
    const unsigned int n = ls.ctl[0];
    // bulk round next: by stage count, longest first (equal trip counts inside a warp, long batches early).  Chain
    // kernel alone: by chain hint, longest expected chain first - the chain kernel walks a plan's whole chain on one
    // warp, so the long ones must start early (LPT order; see het_order_kernel for the same after a bulk round)
    const bool bulk = (long long)n >= ls.bulk_min;
    const int hist = bulk ? kCtlHist : kCtlHist3, cursor = bulk ? kCtlCursor : kCtlCursor3;
    if (threadIdx.x == 0) {
        unsigned int acc = 0;
        for (int k = 127; k >= 0; --k) { s_base[k] = acc; acc += ls.ctl[hist + k]; }
    }
    __syncthreads();
    const long long span = (long long)gridDim.x * blockDim.x;
    const long long upto = (((long long)n + 31) / 32) * 32;
    for (long long pos = (long long)blockIdx.x * blockDim.x + threadIdx.x; pos < upto; pos += span) {
        const bool live = pos < (long long)n;
        uint4 e = make_uint4(0, 0, 0, 0);
        if (live) e = ls.a[pos];
        // geometry bits 32..39 = S - 1; flag bits 8..14 = chain hint
        const int k = !live ? -1 : bulk ? (int)(e.w & 0xFF) : (int)((e.y >> 8) & 0x7F);
        const unsigned int peers = __match_any_sync(0xFFFFFFFFu, k);
        const int leader = __ffs(peers) - 1, me = threadIdx.x & 31;
        unsigned int at = 0;
        if (live && me == leader) at = atomicAdd(&ls.ctl[cursor + k], (unsigned int)__popc(peers));
        at = __shfl_sync(0xFFFFFFFFu, at, leader);
        if (live) ls.b[(long long)s_base[k] + at + __popc(peers & ((1u << me) - 1u))] = e;
    }
}

template <int MAXS, int MAXL, bool ONE>
__global__ void __launch_bounds__(kThreads, (MAXS <= 64 ? METIS_MIN_BLOCKS : ONE ? METIS_MIN_BLOCKS_BIG_ONE : METIS_MIN_BLOCKS_BIG))
het_first_kernel(const __grid_constant__ MetisProblem p, const __grid_constant__ MetisPlanSpace sp,
                 const __grid_constant__ BlobLayout lay, const uint8_t *__restrict__ blob, const int use_smem,
                 const __grid_constant__ DeviceOut out, const SearchLists ls, const int best_slot) {
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ uint64_t mbar;
    DeviceSink sink(out);
    const unsigned int n = ls.ctl[0];
    if ((long long)n >= ls.bulk_min) {
        const uint8_t *base = blob;
        if (use_smem) {
            stage_blob_tma(smem, blob, lay.total, &mbar);
            base = smem;
        }
        const Tables T = make_tables(p, lay, base, blob);
        Scratch<MAXS, MAXL> w;
        const int lane = threadIdx.x & 31;
        for (;;) {                                           // batches of 32 plans, longest stage counts first
            unsigned int fetched = 0;
            if (lane == 0) fetched = atomicAdd(&ls.ctl[1], 1u);
            const long long b0 = 32LL * __shfl_sync(0xFFFFFFFFu, fetched, 0);
            if (b0 >= (long long)n) break;
            const long long pos = b0 + lane;
            PlanDesc pd;
            const bool has = pos < (long long)n;
            uint4 e = make_uint4(0, 0, 0, 0);
            if (has) { e = ls.b[pos]; decode_entry(sp, e, pd); }
            int hint = 0, start = 1;                         // CoopEvaluator::kReplay unless first_task says more
            const bool cont = first_task<MAXS, MAXL, ONE, Lockstep>(T, w, sink, has, pd, hint, start);
            const unsigned m = __ballot_sync(0xFFFFFFFFu, cont);
            if (m) {
                const int leader = __ffs(m) - 1;
                unsigned int at = 0;
                if (lane == leader) at = atomicAdd(&ls.ctl[2], (unsigned int)__popc(m));
                at = __shfl_sync(0xFFFFFFFFu, at, leader);
                if (cont) {
                    const unsigned key = hint < 0 ? 0u : (hint > 127 ? 127u : (unsigned)hint);
                    const unsigned int c = at + __popc(m & ((1u << lane) - 1u));
                    if (start == 2) {                        // kRetry: hand the re-weighted performance over
                        if (c < ls.save_cap) {
                            for (int s = 0; s < pd.S; ++s) ls.perf[(size_t)s * ls.save_cap + c] = w.perf[s];
                        } else start = 1;                    // no room: the chain kernel replays the attempt
                    }
                    e.y = 1u | ((unsigned)start << 1) | (key << 8);
                    ls.a[c] = e;
                    atomicAdd(&ls.ctl[kCtlHist2 + key], 1u);
                }
            }
        }
    }
    finish_block(sink, out, best_slot + blockIdx.x);
}

// Continuations of the bulk round (list C, in the storage of list A) -> list B, longest expected chain first: the
// chain kernel walks a plan's whole chain on one warp, so the long ones must start early (LPT order).
__global__ void __launch_bounds__(256)
het_order_kernel(const SearchLists ls) {
    __shared__ unsigned int s_base[128];
    if ((long long)ls.ctl[0] < ls.bulk_min) return;          // no bulk round: list B already holds the work
    const unsigned int n = ls.ctl[2];
    if (threadIdx.x == 0) {
        unsigned int acc = 0;
        for (int k = 127; k >= 0; --k) { s_base[k] = acc; acc += ls.ctl[kCtlHist2 + k]; }
    }
    __syncthreads();
    const long long span = (long long)gridDim.x * blockDim.x;
    for (long long pos = (long long)blockIdx.x * blockDim.x + threadIdx.x; pos < (long long)n; pos += span) {
        const uint4 e = ls.a[pos];
        const unsigned key = (e.y >> 8) & 0x7Fu;
        const unsigned int to = s_base[key] + atomicAdd(&ls.ctl[kCtlCursor2 + key], 1u);
        ls.b[to] = e;
        ls.src[to] = (unsigned int)pos;                      // where its saved stage performance lives
    }
}

template <int MAXS, int MAXL>
struct alignas(16) ChainScratch {
    Scratch<MAXS, MAXL> w;
    CoopMail mail;
};

// 64 registers per thread: 32 resident warps per SM in blocks of 16 warps (tables staged once per block)
template <int MAXS, int MAXL, bool ONE>
__global__ void __launch_bounds__(512, 2)
het_chain_kernel(const __grid_constant__ MetisProblem p, const __grid_constant__ MetisPlanSpace sp,
                 const __grid_constant__ BlobLayout lay, const uint8_t *__restrict__ blob, const int use_smem,
                 const unsigned int scratch_off, const __grid_constant__ DeviceOut out, const SearchLists ls,
                 const int best_slot) {
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ uint64_t mbar;
    const uint8_t *base = blob;
    if (use_smem) {
        stage_blob_tma(smem, blob, lay.total, &mbar);
        base = smem;
    }
    const Tables T = make_tables(p, lay, base, blob);
    DeviceSink sink(out);
    const int lane = threadIdx.x & 31;
    sink.leader = lane == 0;
    ChainScratch<MAXS, MAXL> *cs = reinterpret_cast<ChainScratch<MAXS, MAXL> *>(smem + scratch_off) + (threadIdx.x >> 5);
    const unsigned int n_adm = ls.ctl[0];
    const bool bulk = (long long)n_adm >= ls.bulk_min;
    const uint4 *list = ls.b;                                // sorted: by chain hint after a bulk round, else by stage count
    const unsigned int n = bulk ? ls.ctl[2] : n_adm;
    WarpCoop lanes;
    CoopEvaluator<MAXS, MAXL, WarpCoop, ONE> ev(T, cs->w, cs->mail, lanes);
    for (;;) {
        unsigned int i = 0;
        if (lane == 0) i = atomicAdd(&ls.ctl[3], 1u);
        i = __shfl_sync(0xFFFFFFFFu, i, 0);
        if (i >= n) break;
        const uint4 e = __ldcg(&list[i]);
        PlanDesc pd;
        decode_entry(sp, e, pd);
        lanes.mark(1);
        // flags: not touched by a bulk round -> kFresh; else what first_task decided (kReplay / kRetry / kAdvance)
        const int start = (e.y & 1u) ? (int)((e.y >> 1) & 3u) : 0;
        const double *perf = nullptr;
        if (start == 2) perf = ls.perf + __ldcg(&ls.src[i]);
        ev.run_chain(pd, sink, start, perf, (size_t)ls.save_cap);
        lanes.mark(0);
    }
    while (WarpCoop::block_or(0)) {}                         // out of work: answer the others' gates until all are done
    sink.leader = true;                                      // lanes 1-31 carry empty counters / bests
    if (lane != 0) { sink.n_part = sink.n_run = sink.n_key = 0; }
    finish_block(sink, out, best_slot + blockIdx.x);
}

__global__ void het_finalize_kernel(const MetisRecord *block_best, int nblocks, const unsigned long long *counters,
                                    const unsigned int *ctl, unsigned long long instantiation, MetisSearchSummary *summary) {
    __shared__ double s_cost[32];
    __shared__ uint32_t s_ord[32], s_step[32], s_meta[32];
    double c = INFINITY;
    uint32_t o = 0xFFFFFFFFu, st = 0xFFFFu, mt = 0;
    for (int i = threadIdx.x; i < nblocks; i += blockDim.x) {
        const MetisRecord r = block_best[i];
        if (rec_less(r.cost, r.ordinal, r.step, c, o, st)) {
            c = r.cost; o = r.ordinal; st = r.step; mt = ((uint32_t)r.num_repartition << 8) | r.num_stage;
        }
    }
    const unsigned full = 0xFFFFFFFFu;
    for (int d = 16; d > 0; d >>= 1) {
        const double c2 = __shfl_xor_sync(full, c, d);
        const uint32_t o2 = __shfl_xor_sync(full, o, d), s2 = __shfl_xor_sync(full, st, d),
                       m2 = __shfl_xor_sync(full, mt, d);
        if (rec_less(c2, o2, s2, c, o, st)) { c = c2; o = o2; st = s2; mt = m2; }
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) { s_cost[warp] = c; s_ord[warp] = o; s_step[warp] = st; s_meta[warp] = mt; }
    __syncthreads();
    if (threadIdx.x == 0) {
        const int nw = (blockDim.x + 31) / 32;
        for (int wi = 1; wi < nw; ++wi)
            if (rec_less(s_cost[wi], s_ord[wi], s_step[wi], c, o, st)) { c = s_cost[wi]; o = s_ord[wi]; st = s_step[wi]; mt = s_meta[wi]; }
        MetisSearchSummary s;
        memset(&s, 0, sizeof(s));
        s.num_records = counters[0];
        s.num_partition_calls = counters[1];
        s.num_balancer_runs = counters[2];
        s.num_keyerror = counters[3];
        const unsigned long long fk = counters[4];
        if (fk == 0xFFFFFFFFFFFFFFFFULL) { s.fatal_ordinal = 0xFFFFFFFFFFFFFFFFULL; s.fatal_code = 0; s.fatal_aux = 0; }
        else { s.fatal_ordinal = fk >> 32; s.fatal_code = (uint32_t)((fk >> 24) & 0xFF); s.fatal_aux = (uint32_t)(fk & 0xFFFFFF); }
        s.best.cost = c; s.best.ordinal = o; s.best.step = (uint16_t)st;
        s.best.num_repartition = (uint8_t)(mt >> 8); s.best.num_stage = (uint8_t)mt;
        s.reserved[0] = ctl[0];                                          // plans admitted
        s.reserved[1] = ctl[2];                                          // plans handed to the chain kernel by the bulk round
        s.reserved[2] = instantiation;                                   // MAXS | MAXL << 16 | ONE << 32 of the kernels
        *summary = s;
    }
}

// replays single candidates: writes dp code, tp code, partition for (ordinal, step)
struct DetailSink {
    uint8_t *dst;
    int want_step;
    __device__ void phase(int) {}
    __device__ void partition_call() {}
    __device__ void balancer_run() {}
    __device__ void keyerror() {}
    __device__ void fatal(uint32_t, int, uint32_t) {}
    __device__ void emit(const PlanDesc &pd, int step, int, double, const uint8_t *tpc, const uint16_t *part) {
        if (step != want_step) return;
        for (int s = 0; s < pd.S; ++s) { dst[s] = (uint8_t)(pd.row[s] - tpc[s]); dst[pd.S + s] = tpc[s]; }
        for (int s = 0; s <= pd.S; ++s) dst[2 * pd.S + s] = (uint8_t)part[s];
    }
};

template <int MAXS, int MAXL>
__global__ void __launch_bounds__(kThreads)
het_detail_kernel(const __grid_constant__ MetisProblem p, const __grid_constant__ MetisPlanSpace sp,
                  const __grid_constant__ BlobLayout lay, const uint8_t *__restrict__ blob,
                  const MetisRecord *__restrict__ picks, long long n, uint8_t *detail, int stride) {
    const Tables T = make_tables(p, lay, blob);
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    PlanDesc pd;
    if (!decode_plan(sp, picks[i].ordinal, pd)) return;
    DetailSink sink{detail + (size_t)i * stride, (int)picks[i].step};
    Scratch<MAXS, MAXL> w;
    PlanEvaluator<MAXS, MAXL> ev(T, w);
    ev.run(pd, sink, (int)picks[i].step);
}

// verbose transcript: one thread replays one plan and records what the reference prints (metis_trace.cuh)
__global__ void __launch_bounds__(64)
het_trace_kernel(const __grid_constant__ MetisProblem p, const __grid_constant__ MetisPlanSpace sp,
                 const __grid_constant__ BlobLayout lay, const uint8_t *__restrict__ blob,
                 const uint32_t *__restrict__ ordinals, long long n, uint64_t *trace, int words) {
    const Tables T = make_tables(p, lay, blob);
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    TraceOut out(trace + (size_t)i * words, words);
    PlanDesc pd;
    if (decode_plan(sp, ordinals[i], pd)) {
        Scratch<kMaxS, kMaxL> w;
        TraceEvaluator<kMaxS, kMaxL> ev(T, w, out);
        ev.run_traced(pd);
    }
    out.finish();
}

__global__ void __launch_bounds__(kThreads)
homo_cost_kernel(const __grid_constant__ MetisProblem p, const __grid_constant__ BlobLayout lay,
                 const uint8_t *__restrict__ blob, int type_id, const int32_t *__restrict__ plans, long long n,
                 double *cost, int32_t *status) {
    const Tables T = make_tables(p, lay, blob);
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    const int32_t *q = plans + i * 5;
    double c = 0.0;
    int oom = 0;
    const int rc = homo_cost(T, type_id, q[0], q[1], q[2], q[3], q[4], c, oom);
    cost[i] = rc ? NAN : c;
    status[i] = rc ? 1 : (oom ? 2 : 0);
}

template <int MAXS, int MAXL>
__global__ void __launch_bounds__(kThreads)
layer_balance_kernel(const double *__restrict__ capa, const int32_t *__restrict__ num_stage, long long n, int stride,
                     const double *__restrict__ lc, const double *__restrict__ dlay, int norm_len, int num_layers,
                     uint16_t *partition) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    Tables T;
    memset(&T, 0, sizeof(T));
    T.p.num_layers = num_layers;
    T.p.norm_len = norm_len;
    T.norm_lc = lc;
    T.dlay = dlay;
    Scratch<MAXS, MAXL> w;
    const int S = num_stage[i];
    uint16_t *out = partition + i * (stride + 1);
    if (S < 1 || S > MAXS || num_layers > MAXL) { out[0] = 0xFFFF; return; }
    for (int s = 0; s < S; ++s) w.perf[s] = capa[i * stride + s];
    const int rc = balance_run<MAXS, MAXL>(T, S, w, Serial());
    if (rc) { out[0] = 0xFFFF; return; }
    for (int s = 0; s <= S; ++s) out[s] = w.part[s];
}

// SURVEY.md 8(f)-1: one warp per record = a slice of <= 64 permutations of one composition.  The walk (metis_rows.cuh) is sequential - every permutation is one
// node of a linked list moved to the front of the previous one - so the leader lane advances it, on a state kept
// in shared memory; writing a row out is not: group by group, the lanes copy the codes (coalesced byte stores).
constexpr int kRowWarps = 8;
__global__ void __launch_bounds__(kRowWarps * 32)
het_rows_kernel(const MetisCompRec *__restrict__ recs, long long ncomp, const uint8_t *__restrict__ pool,
                uint8_t *__restrict__ rows) {
    __shared__ CompWalk s_walk[kRowWarps];
    __shared__ uint8_t s_pool[kRowWarps][METIS_MAX_PERMUTE_GROUPS + METIS_MAX_STAGES];
    const unsigned full = 0xFFFFFFFFu;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const long long c = (long long)blockIdx.x * kRowWarps + wid;
    if (c >= ncomp) return;                                   // whole warps leave together
    const MetisCompRec rec = recs[c];
    const int stages = rec.stages, n = rec.num_groups;
    if (stages > METIS_MAX_STAGES || n > METIS_MAX_PERMUTE_GROUPS) return;   // refused on the host
    for (int p = lane; p < n + stages; p += 32) s_pool[wid][p] = pool[rec.pool_offset + p];
    __syncwarp();
    CompWalk &cw = s_walk[wid];
    MetisCompRec local = rec;
    local.pool_offset = 0;
    if (lane == 0) {
        cw.init(local, s_pool[wid]);
        for (uint32_t skip = 0; skip < rec.first_row; ++skip) cw.advance();   // to the first permutation of the slice
    }
    uint8_t *dst = rows + rec.row_offset;
    for (uint32_t r = 0;;) {
        __syncwarp();                                         // the list as the leader left it
        int at = 0;
        for (int h = cw.head; h >= 0; h = cw.nxt[h]) {        // every lane walks the (short) list
            const int len = cw.len[h], off = cw.off[h];
            for (int b = lane; b < len; b += 32) dst[at + b] = cw.codes[off + b];
            at += len;
        }
        __syncwarp();
        if (++r >= rec.num_rows) break;                       // warp-uniform
        int more = 0;
        if (lane == 0) more = cw.advance() ? 1 : 0;
        if (!__shfl_sync(full, more, 0)) break;
        dst += stages;
    }
}

__global__ void divide_by_seven_kernel(const double *lc, int n, double *out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = lc[i] / 7.0;
}

static int check_problem(const MetisProblem *p) {
    if (!p) return arg_fail("problem is NULL");
    if (p->num_types < 1 || p->num_types > METIS_MAX_TYPES) return arg_fail("num_types out of range");
    // detail rows keep layer_partition entries in one byte: the last boundary (num_layers) must fit
    if (p->num_layers < 1 || p->num_layers > METIS_MAX_LAYERS || p->num_layers > 255)
        return arg_fail("num_layers out of range (1 .. 255)");
    if (p->lpad < p->num_layers) return arg_fail("lpad < num_layers");
    if (p->num_keys < 1 || p->num_tp < 1 || p->num_bs < 1 || p->norm_len < 1) return arg_fail("empty profile tables");
    if (p->devices_per_node < 1 || p->total_devices < 1 || p->q10_devices < 1) return arg_fail("empty cluster");
    return METIS_OK;
}

}  // namespace metis

using namespace metis;

extern "C" {

const char *metis_last_error(void) { return g_err; }
int metis_abi_version(void) { return METIS_ABI_VERSION; }
#ifdef METIS_PROFILE_PHASES
int metis_debug_marks(long long *out32, int reset) {
    long long zero[64] = {0};
    if (out32) cudaMemcpyFromSymbol(out32, g_mark_acc, sizeof(zero));      // caller provides 64 entries
    if (reset) cudaMemcpyToSymbol(g_mark_acc, zero, sizeof(zero));
    return 0;
}
#endif
void metis_set_profile_events(void *before_kernel, void *after_kernel) {
    g_ev_before = static_cast<cudaEvent_t>(before_kernel);
    g_ev_after = static_cast<cudaEvent_t>(after_kernel);
}

static int64_t shard_plan_slots(int64_t num_plans, const MetisShard *sh) {
    const int64_t tile = sh->tile, world = sh->world;
    const int64_t rounds = (num_plans + tile * world - 1) / (tile * world);
    return rounds * tile;
}

constexpr int64_t kFixedWs = 16384;                // summary + counters + list control words
constexpr int64_t kMaxBlocks = 4096;               // per-block best records (bulk round + chain kernel)

static int env_int(const char *name, int lo, int hi, int dflt) {
    const char *e = getenv(name);
    if (!e || !*e) return dflt;
    char *end = nullptr;
    const long v = strtol(e, &end, 10);
    if (end == e || *end != '\0' || v < lo || v > hi) return dflt;     // malformed or out of range: ignored
    return (int)v;
}

// continuations of the bulk round whose re-weighted stage performance is kept for the chain kernel (the others replay
// their first attempt): a quarter of the plans, at most 128 Ki (METIS_SAVE_SLOTS: test knob for the replay path)
static int64_t save_slots(int64_t cap) {
    const int forced = env_int("METIS_SAVE_SLOTS", 1, 1 << 20, 0);
    if (forced) return forced;
    return cap / 4 < 131072 ? (cap / 4 > 0 ? cap / 4 : 1) : 131072;
}

int64_t metis_het_workspace_bytes(const MetisProblem *problem, int64_t num_plans, int32_t max_stage) {
    if (check_problem(problem)) return METIS_E_ARG;
    if (num_plans < 0) return METIS_E_ARG;
    const BlobLayout lay = make_layout(*problem);
    const int64_t cap = (num_plans + 127) & ~(int64_t)127;      // worst case: every plan of the shard is admitted
    const int64_t stages = max_stage < 1 ? 1 : (max_stage > METIS_MAX_STAGES ? METIS_MAX_STAGES : max_stage);
    return 256 + kFixedWs + (int64_t)lay.rsum + (int64_t)align16(lay.rsum_bytes) + kMaxBlocks * (int64_t)sizeof(MetisRecord) +
           2 * cap * (int64_t)sizeof(uint4) + cap * 4 + save_slots(cap) * stages * 8 + 1024;
}

struct Workspace {
    MetisSearchSummary *summary;
    unsigned long long *counters;
    unsigned int *ctl;
    uint8_t *blob;
    MetisRecord *block_best;
    uint8_t *lists;
};

static Workspace carve(void *ws, const BlobLayout &lay) {
    uint8_t *b = static_cast<uint8_t *>(ws);
    uintptr_t a = (reinterpret_cast<uintptr_t>(b) + 127) & ~(uintptr_t)127;
    b = reinterpret_cast<uint8_t *>(a);
    Workspace w;
    w.summary = reinterpret_cast<MetisSearchSummary *>(b);
    w.counters = reinterpret_cast<unsigned long long *>(b + 1024);
    w.ctl = reinterpret_cast<unsigned int *>(b + 2048);
    w.blob = b + kFixedWs;
    w.block_best = reinterpret_cast<MetisRecord *>(b + kFixedWs + lay.rsum + align16(lay.rsum_bytes));
    w.lists = reinterpret_cast<uint8_t *>(w.block_best + kMaxBlocks);
    return w;
}


}  // extern "C"

// Launch configuration of one search: which instantiation, how the tables are staged, block shapes.
template <int MAXS, int MAXL, bool ONE>
static int launch_search(const MetisProblem &p_arg, const MetisPlanSpace &s_arg, const MetisShard &sh,
                         const BlobLayout &lay, const Workspace &ws, const DeviceOut &out, int64_t slots,
                         cudaStream_t stream) {
    cudaError_t e;
    int dev = 0, sms = 0, smem_optin = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaDeviceGetAttribute(&smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    if (sms < 1 || smem_optin < 48 * 1024) return cuda_fail(cudaErrorInvalidDevice, "device attributes");
    const int blob_max = env_int("METIS_SMEM_BLOB_MAX", 0, kSmemBlobMax, kSmemBlobMax);   // larger tables stay in global memory
    const unsigned int blob_pad = (lay.total + 127u) & ~127u;

    SearchLists ls;
    const int64_t cap = (slots + 127) & ~(int64_t)127;
    ls.a = reinterpret_cast<uint4 *>(ws.lists);
    ls.b = ls.a + cap;
    ls.ctl = ws.ctl;
    ls.src = reinterpret_cast<unsigned int *>(ls.b + cap);
    ls.perf = reinterpret_cast<double *>(ls.src + cap);     // cap is a multiple of 128: 8-byte aligned
    ls.save_cap = (unsigned int)save_slots(cap);

    // ---- chain kernel: warps per block chosen so that tables + per-warp scratch fill the SM with warps ----
    auto chain = het_chain_kernel<MAXS, MAXL, ONE>;
    const size_t per_warp = sizeof(ChainScratch<MAXS, MAXL>);
    int chain_smem_tables = (int)lay.total <= blob_max;
    int chain_threads = 0, chain_per_sm = 0;
    size_t chain_dyn = 0;
    unsigned int chain_off = 0;
    const int forced = env_int("METIS_CHAIN_THREADS", 32, 512, 0);
    for (int pass = 0; pass < 2 && chain_threads == 0; ++pass) {       // second pass: tables in global memory
        int best_warps = 0;
        for (int threads = 64; threads <= 512; threads *= 2) {
            if (forced && threads != ((forced + 31) & ~31)) continue;
            const unsigned int off = chain_smem_tables ? blob_pad : 0u;
            const size_t dyn = off + (size_t)(threads / 32) * per_warp;
            if (dyn > (size_t)smem_optin) continue;
            if (dyn > 48 * 1024) {
                e = cudaFuncSetAttribute(chain, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn);
                if (e != cudaSuccess) { cudaGetLastError(); continue; }
            }
            int per_sm = 0;
            e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, chain, threads, dyn);
            if (e != cudaSuccess || per_sm < 1) { cudaGetLastError(); continue; }
            const int warps = per_sm * threads / 32;
            if (warps > best_warps) { best_warps = warps; chain_threads = threads; chain_per_sm = per_sm; chain_dyn = dyn; chain_off = off; }
        }
        if (chain_threads == 0) chain_smem_tables = 0;
    }
    if (chain_threads == 0) return arg_fail("chain kernel does not fit this device (shared memory)");
    if (chain_dyn > 48 * 1024) {
        e = cudaFuncSetAttribute(chain, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)chain_dyn);
        if (e != cudaSuccess) return cuda_fail(e, "cudaFuncSetAttribute(chain)");
    }
    int64_t chain_grid = (int64_t)sms * chain_per_sm;

    // ---- bulk round ----
    auto first = het_first_kernel<MAXS, MAXL, ONE>;
    int first_smem_tables = (int)lay.total <= blob_max && blob_pad <= (unsigned int)smem_optin;
    size_t first_dyn = first_smem_tables ? blob_pad : 0;
    if (first_dyn > 48 * 1024) {
        e = cudaFuncSetAttribute(first, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)first_dyn);
        if (e != cudaSuccess) { cudaGetLastError(); first_smem_tables = 0; first_dyn = 0; }
    }
    int first_per_sm = 0;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&first_per_sm, first, kThreads, first_dyn);
    if (e != cudaSuccess || first_per_sm < 1) return cuda_fail(e, "occupancy query (bulk round)");
    int64_t first_grid = (int64_t)sms * first_per_sm;
    if (first_grid + chain_grid > kMaxBlocks) return arg_fail("grid exceeds the per-block best table");

    // MetisShard.reserved: minimum list length for the bulk round (0 = default: 12 lists' worth of chain warps)
    ls.bulk_min = sh.reserved > 0 ? (long long)sh.reserved : 12LL * chain_grid * (chain_threads / 32);

    if (g_ev_before) cudaEventRecord(g_ev_before, stream);
    if (slots > 0) {
        const int64_t admit_blocks = (slots + 255) / 256;
        if (admit_blocks > 0x7FFFFFFFLL) return arg_fail("too many plans for one launch");
        het_admit_kernel<<<(unsigned)admit_blocks, 256, 0, stream>>>(s_arg, sh, (long long)slots, p_arg.gbs, p_arg.max_bs,
                                                                     p_arg.max_tp, ls);
        int64_t scatter_blocks = (slots + 255) / 256;
        if (scatter_blocks > 8LL * sms) scatter_blocks = 8LL * sms;
        het_scatter_kernel<<<(unsigned)scatter_blocks, 256, 0, stream>>>(ls);
        first<<<(unsigned)first_grid, kThreads, first_dyn, stream>>>(p_arg, s_arg, lay, ws.blob, first_smem_tables, out, ls, 0);
        het_order_kernel<<<(unsigned)(2 * sms), 256, 0, stream>>>(ls);
        chain<<<(unsigned)chain_grid, chain_threads, chain_dyn, stream>>>(p_arg, s_arg, lay, ws.blob, chain_smem_tables,
                                                                         chain_off, out, ls, (int)first_grid);
        e = cudaGetLastError();
        if (e != cudaSuccess) return cuda_fail(e, "search kernels");
    }
    if (g_ev_after) cudaEventRecord(g_ev_after, stream);
    g_ev_before = g_ev_after = nullptr;
    const unsigned long long instantiation = (unsigned long long)MAXS | (unsigned long long)MAXL << 16 |
                                             (unsigned long long)ONE << 32;
    het_finalize_kernel<<<1, 256, 0, stream>>>(ws.block_best, (int)(slots > 0 ? first_grid + chain_grid : 0), ws.counters,
                                               ws.ctl, instantiation, ws.summary);
    e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, "het_finalize_kernel");
    return METIS_OK;
}

extern "C" {

int metis_het_search(const MetisProblem *problem, const MetisPlanSpace *space, const MetisShard *shard,
                     MetisRecord *records, int64_t capacity, uint8_t *detail, int32_t detail_stride,
                     void *workspace, int64_t workspace_bytes, MetisSearchSummary *summary, void *stream_) {
    int rc = check_problem(problem);
    if (rc) return rc;
    if (!space || !shard || !workspace || !summary) return arg_fail("NULL argument");
    if (shard->world < 1 || shard->rank < 0 || shard->rank >= shard->world || shard->tile < 32 || shard->tile % 32)
        return arg_fail("bad shard (tile must be a positive multiple of 32)");
    if (space->num_plans > 0xFFFFFFF0LL) return arg_fail("more than 2^32 plans");
    if (space->max_stage < 1 || space->max_stage > METIS_MAX_STAGES) return arg_fail("max_stage out of range (METIS_MAX_STAGES)");
    if (space->num_div < 1 || space->num_div > 256) return arg_fail("more than 256 divisors of gbs");
    // the geometry word of a list entry keeps ns_idx in 8 bits and the byte offset of the row in 32
    if (problem->num_node_sequences < 1 || problem->num_node_sequences > 256)
        return arg_fail("more than 256 node sequences (geometry word)");
    if (space->rows_bytes < 0 || space->rows_bytes > 0xFFFFFFFFLL) return arg_fail("row tables must be smaller than 4 GiB (geometry word)");
    if (detail && detail_stride < 3 * space->max_stage + 1) return arg_fail("detail_stride too small (3 * max_stage + 1)");
    if (capacity < 0 || (capacity > 0 && !records)) return arg_fail("records/capacity mismatch");
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    const BlobLayout lay = make_layout(*problem);
    const int64_t slots = shard_plan_slots(space->num_plans, shard);
    const int64_t need = metis_het_workspace_bytes(problem, slots, space->max_stage);
    if (workspace_bytes < need) { snprintf(g_err, sizeof(g_err), "workspace too small: need %lld", (long long)need); return METIS_E_CAPACITY; }
    const Workspace ws = carve(workspace, lay);

    cudaError_t e;
    e = cudaMemsetAsync(ws.counters, 0, kFixedWs - 1024, stream);   // counters, list control words
    if (e != cudaSuccess) return cuda_fail(e, "memset counters");
    e = cudaMemsetAsync(ws.counters + 4, 0xFF, sizeof(unsigned long long), stream);
    if (e != cudaSuccess) return cuda_fail(e, "memset fatal key");
    pack_tables_kernel<<<8, 256, 0, stream>>>(*problem, lay, ws.blob);
    {
        const long long nthr = (long long)range_sum_tables(*problem) * problem->num_layers;
        range_sums_kernel<<<(unsigned)((nthr + 127) / 128), 128, 0, stream>>>(*problem, lay, ws.blob);
    }
    e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, "pack_tables_kernel");

    DeviceOut out;
    out.records = records; out.capacity = capacity; out.detail = detail; out.detail_stride = detail_stride;
    out.counters = ws.counters; out.block_best = ws.block_best;
    // three instantiations: per-warp scratch of the chain kernel (and per-thread scratch of the bulk round)
    // sized for S <= 64 / L <= 128, S <= 96 / L <= 128, and the compiled limits
    // ... each once for single-type clusters (no mixed-type code at all) and once for the general case
    const bool one = problem->num_types == 1;
    if (space->max_stage <= 64 && problem->num_layers <= 128)
        rc = one ? launch_search<64, 128, true>(*problem, *space, *shard, lay, ws, out, slots, stream)
                 : launch_search<64, 128, false>(*problem, *space, *shard, lay, ws, out, slots, stream);
    else if (space->max_stage <= 96 && problem->num_layers <= 128)
        rc = one ? launch_search<96, 128, true>(*problem, *space, *shard, lay, ws, out, slots, stream)
                 : launch_search<96, 128, false>(*problem, *space, *shard, lay, ws, out, slots, stream);
    else
        rc = one ? launch_search<kMaxS, kMaxL, true>(*problem, *space, *shard, lay, ws, out, slots, stream)
                 : launch_search<kMaxS, kMaxL, false>(*problem, *space, *shard, lay, ws, out, slots, stream);
    if (rc) return rc;
    e = cudaMemcpyAsync(summary, ws.summary, sizeof(MetisSearchSummary), cudaMemcpyDeviceToHost, stream);
    if (e != cudaSuccess) return cuda_fail(e, "copy summary");
    return METIS_OK;
}

int metis_het_detail(const MetisProblem *problem, const MetisPlanSpace *space, const MetisRecord *picks, int64_t n,
                     uint8_t *detail, int32_t detail_stride, void *workspace, int64_t workspace_bytes, void *stream_) {
    int rc = check_problem(problem);
    if (rc) return rc;
    if (!space || !picks || !detail || !workspace) return arg_fail("NULL argument");
    if (detail_stride < 3 * space->max_stage + 1) return arg_fail("detail_stride too small (3 * max_stage + 1)");
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    const BlobLayout lay = make_layout(*problem);
    if (workspace_bytes < 256 + kFixedWs + (int64_t)align16(lay.total)) return METIS_E_CAPACITY;
    const Workspace ws = carve(workspace, lay);
    pack_tables_kernel<<<8, 256, 0, stream>>>(*problem, lay, ws.blob);
    if (n > 0) {
        const unsigned nb = (unsigned)((n + kThreads - 1) / kThreads);
        het_detail_kernel<kMaxS, kMaxL><<<nb, kThreads, 0, stream>>>(*problem, *space, lay, ws.blob, picks, n, detail,
                                                                     detail_stride);
    }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, "het_detail_kernel");
    return METIS_OK;
}

int metis_het_trace(const MetisProblem *problem, const MetisPlanSpace *space, const uint32_t *ordinals, int64_t n,
                    uint64_t *trace, int32_t words_per_plan, void *workspace, int64_t workspace_bytes, void *stream_) {
    int rc = check_problem(problem);
    if (rc) return rc;
    if (!space || !ordinals || !trace || !workspace) return arg_fail("NULL argument");
    if (words_per_plan < 64) return arg_fail("words_per_plan too small");
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    const BlobLayout lay = make_layout(*problem);
    if (workspace_bytes < 256 + kFixedWs + (int64_t)align16(lay.total)) return METIS_E_CAPACITY;
    const Workspace ws = carve(workspace, lay);
    pack_tables_kernel<<<8, 256, 0, stream>>>(*problem, lay, ws.blob);
    if (n > 0) {
        const unsigned nb = (unsigned)((n + 63) / 64);
        het_trace_kernel<<<nb, 64, 0, stream>>>(*problem, *space, lay, ws.blob, ordinals, n, trace, words_per_plan);
    }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, "het_trace_kernel");
    return METIS_OK;
}

int metis_generate_rows(const MetisCompRec *recs, int64_t num_comps, const uint8_t *pool, uint8_t *rows, void *stream_) {
    if (num_comps < 0 || (num_comps > 0 && (!recs || !pool || !rows))) return arg_fail("NULL argument");
    if (num_comps > 0) {
        const int64_t nb = (num_comps + kRowWarps - 1) / kRowWarps;
        if (nb > 0x7FFFFFFFLL) return arg_fail("too many compositions for one launch");
        het_rows_kernel<<<(unsigned)nb, kRowWarps * 32, 0, static_cast<cudaStream_t>(stream_)>>>(recs, (long long)num_comps, pool, rows);
    }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, "het_rows_kernel");
    return METIS_OK;
}

int metis_homo_cost(const MetisProblem *problem, int32_t type_id, const int32_t *plans, int64_t n, double *cost,
                    int32_t *status, void *workspace, int64_t workspace_bytes, void *stream_) {
    int rc = check_problem(problem);
    if (rc) return rc;
    if (!plans || !cost || !status || !workspace) return arg_fail("NULL argument");
    if (type_id < 0 || type_id >= problem->num_types) return arg_fail("type_id out of range");
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    const BlobLayout lay = make_layout(*problem);
    if (workspace_bytes < 256 + kFixedWs + (int64_t)align16(lay.total)) return METIS_E_CAPACITY;
    const Workspace ws = carve(workspace, lay);
    pack_tables_kernel<<<8, 256, 0, stream>>>(*problem, lay, ws.blob);
    if (n > 0) {
        const unsigned nb = (unsigned)((n + kThreads - 1) / kThreads);
        homo_cost_kernel<<<nb, kThreads, 0, stream>>>(*problem, lay, ws.blob, type_id, plans, n, cost, status);
    }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, "homo_cost_kernel");
    return METIS_OK;
}

int metis_layer_balance(const double *capa, const int32_t *num_stage, int64_t n, int32_t stride, const double *lc,
                        int32_t norm_len, int32_t num_layers, uint16_t *partition, void *workspace,
                        int64_t workspace_bytes, void *stream_) {
    if (!capa || !num_stage || !lc || !partition || !workspace) return arg_fail("NULL argument");
    if (stride < 1 || stride > METIS_MAX_STAGES) return arg_fail("stride out of range");
    if (num_layers < 1 || num_layers > METIS_MAX_LAYERS || norm_len < 1) return arg_fail("layers out of range");
    if (workspace_bytes < (int64_t)norm_len * 8 + 256) return METIS_E_CAPACITY;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    double *dlay = reinterpret_cast<double *>((reinterpret_cast<uintptr_t>(workspace) + 127) & ~(uintptr_t)127);
    divide_by_seven_kernel<<<(norm_len + 127) / 128, 128, 0, stream>>>(lc, norm_len, dlay);
    if (n > 0) {
        const unsigned nb = (unsigned)((n + kThreads - 1) / kThreads);
        layer_balance_kernel<kMaxS, kMaxL><<<nb, kThreads, 0, stream>>>(capa, num_stage, n, stride, lc, dlay, norm_len,
                                                                        num_layers, partition);
    }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, "layer_balance_kernel");
    return METIS_OK;
}

}  // extern "C"
