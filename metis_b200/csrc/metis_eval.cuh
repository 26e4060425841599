// metis_eval.cuh - per-plan evaluator of the Metis plan-search hot path.
//
// One *thread* evaluates one inter-stage plan (SURVEY.md section 8a rows a5-a16):
// the intra-stage strategy chain, the layer load balancer with its memory
// feasibility loop and the hetero cost model, all in IEEE binary64 in the
// reference's evaluation order (compile with -fmad=false: no FMA contraction).
//
// The code is plain C++ (no CUDA intrinsics) so that tests/hostsim can compile
// the very same source with g++ for CPU-side debugging of the device logic.
// That shim lives in tests/ and is never loaded by the metis_b200 package.
//
// Reference citations (paths relative to the reference root) are given at each
// function.  State is kept compact instead of the reference's per-sub-layer
// lists; see DESIGN.md "Load balancer on device" for why each step is equivalent.
#pragma once

#include <stdint.h>
#include <string.h>
#include <math.h>

#include "../../include/metis_b200.h"

#if defined(__CUDACC__)
#define MB_HD __host__ __device__ __forceinline__
#define MB_HD_NOINLINE __host__ __device__ __noinline__
#else
#define MB_HD inline
#define MB_HD_NOINLINE inline
#endif

namespace metis {

// Task-list words are read with ld.global.cg (L2 only): in the barrier-free latency mode another SM may have
// rewritten a neighbouring slot of the same 128-byte line a moment ago, and an L1 copy of that line fetched
// by a different warp of this SM could be stale (L1 is not coherent; every task is read exactly once anyway).
template <class V>
MB_HD V list_load(const V *p) {
#if defined(__CUDA_ARCH__)
    return __ldcg(p);
#else
    return *p;
#endif
}

constexpr int kH = 7;                 // hallucination (model/load_balancer.py:183)
constexpr double kMemCoef = 5.0;      // mem_coef (model/load_balancer.py:31)
constexpr uint8_t kDropped = 0xFF;    // real layer kept by no stage (quirk Q5)

// Tables as seen by the evaluator (pointers into shared or global memory).
struct Tables {
    MetisProblem p;
    const int16_t *key_index;
    const double *lc;          // [num_keys][lpad]
    const double *mem;         // [num_keys][lpad]
    const double *exec_full;   // [num_keys]
    const double *fb_sync;     // [num_keys]
    const double *norm_lc;     // [norm_len]
    const double *type_memory, *bw_first, *bw_min;
    const uint8_t *run_type;   // [ns][num_types]
    const int32_t *run_end;    // [ns][num_types]  type runs of the true rank -> device map (model/device_group.py:22-32)
    const int32_t *q10_end;    // [ns][num_types]  type runs of the rank list built with node 0's GPU count (quirk Q10):
                               //                  load_balancer.py:109-119 (ranks) and cluster_bandwidth.py:158-167 (nodes)
    // derived once per launch (derive_tables): every entry is the result of the same single IEEE
    // operation the reference performs, so looking it up is bit-identical to recomputing it
    const double *dlay;        // [norm_len] norm_lc[r] / 7              (load_balancer.py:190-193)
    const double *inv_exec;    // [num_keys] 1. / sum(layer-computes)    (model/device_group.py:80)
    const double *ratio;       // [num_layers+1] n / num_layers          (cost_estimator.py:146)
    const double *dpk;         // [kDpk] 2*(dp-1) / (dp * (bw*2^20)), dp = 2^i, uniform bandwidth only (:40-41)
    const double *pp_hidden;   // [num_bs+1] mbs*seq*hidden / (bw*2^20), uniform bandwidth only (:45-47)
    const double *pp_vocab;    // [num_bs+1][num_tp] (mbs*seq*vocab / tp) / (bw*2^20)
    // not a reference value: running sum of the sub-layer demands, psub[j] = dlay[0/7] + .. + dlay[(j-1)/7], used only
    // to PREDICT where a stage's forward fill ends (metis_coop.cuh); every prediction is verified exactly
    const double *psub;        // [7 * num_layers + 1] (empty when norm_len < num_layers)
    const double *dsub;        // [7 * num_layers] demand of every sub-layer, dsub[j] = dlay[j / 7] (the same bits)
    // range sums (fill_range_sums below): rsum[(t * n + b) * n + a] = sum(row_t[a:b]) as CPython adds it up, n =
    // num_layers + 1; rows t: layer_memory of key t, then layer_compute of key t - num_keys, then norm_lc.  Every
    // stage of every candidate needs such a sum (memory demand, execution time, compute left after the vote); the
    // search kernels look them up, the other kernels (rsum == nullptr) add the slice up.
    const double *rsum;
};

constexpr int kDpk = 16;

// Sizes (in doubles) of the derived tables, in the order derive_tables fills them.
struct DerivedLayout {
    int dlay, inv_exec, ratio, dpk, pp_hidden, pp_vocab, psub, dsub, total;
};

MB_HD DerivedLayout derived_layout(const MetisProblem &p) {
    DerivedLayout d;
    int o = 0;
    d.dlay = o; o += p.norm_len;
    d.inv_exec = o; o += p.num_keys;
    d.ratio = o; o += p.num_layers + 1;
    d.dpk = o; o += kDpk;
    d.pp_hidden = o; o += p.num_bs + 1;
    d.pp_vocab = o; o += (p.num_bs + 1) * p.num_tp;
    d.psub = o; o += (p.norm_len >= p.num_layers) ? kH * p.num_layers + 1 : 0;
    d.dsub = o; o += (p.norm_len >= p.num_layers) ? kH * p.num_layers : 0;
    d.total = o;
    return d;
}

// One entry of the derived tables (index i of the flat array laid out by derived_layout).
MB_HD double derive_entry(const MetisProblem &p, const DerivedLayout &d, const double *norm_lc,
                          const double *exec_full, const double *bw_first, int i) {
    if (i < d.inv_exec) return norm_lc[i - d.dlay] / 7.0;
    if (i < d.ratio) return 1. / exec_full[i - d.inv_exec];
    if (i < d.dpk) return (double)(i - d.ratio) / (double)p.num_layers;
    const double bw = bw_first[0] * 1048576.0;
    if (i < d.pp_hidden) {
        const int dp = 1 << (i - d.dpk);
        return (double)(2 * (dp - 1)) / ((double)dp * bw);
    }
    if (i < d.pp_vocab) return (double)((int64_t)(i - d.pp_hidden) * p.sequence_length * p.hidden_size) / bw;
    if (i >= d.dsub) return norm_lc[(i - d.dsub) / kH] / 7.0;      // expand_lc_demand (load_balancer.py:189-193)
    if (i >= d.psub) {                                       // predictor table (see Tables::psub): whole layers + a share
        const int j = i - d.psub, r = j / kH;
        double acc = 0.0;
        for (int t = 0; t < r; ++t) acc += norm_lc[t];
        return r < p.norm_len ? acc + norm_lc[r] * ((double)(j - r * kH) / 7.0) : acc;
    }
    const int e = i - d.pp_vocab;
    const int mbs = e / p.num_tp, tpc = e - mbs * p.num_tp;
    return ((double)((int64_t)mbs * p.sequence_length * p.vocab_size) / (double)(1 << tpc)) / bw;
}

MB_HD void bind_derived(Tables &T, const double *base) {
    const DerivedLayout d = derived_layout(T.p);
    T.dlay = base + d.dlay;
    T.inv_exec = base + d.inv_exec;
    T.ratio = base + d.ratio;
    T.dpk = base + d.dpk;
    T.pp_hidden = base + d.pp_hidden;
    T.pp_vocab = base + d.pp_vocab;
    T.psub = base + d.psub;
    T.dsub = base + d.dsub;
}

// One inter-stage plan (search_space/plan.py:21-29).
struct PlanDesc {
    uint32_t ordinal;
    int ns;            // ns_idx
    int S;             // len(device_groups)
    int label;         // InterStagePlan.num_stage as emitted (quirk Q1)
    int batches;
    const uint8_t *row;  // log2(group size) per stage
    uint64_t geo;        // packed geometry (pack_geo) carried through the task lists
};

// rows byte offset (32) | S-1 (8) | label-1 (8) | ns (8) | divisor index (8)
MB_HD uint64_t pack_geo(int64_t row_offset, int S, int label, int ns, int div) {
    return (uint64_t)(row_offset & 0xFFFFFFFFLL) | ((uint64_t)((S - 1) & 0xFF) << 32) | ((uint64_t)((label - 1) & 0xFF) << 40) |
           ((uint64_t)(ns & 0xFF) << 48) | ((uint64_t)(div & 0xFF) << 56);
}

// Paths of the layer balancer that the inputs decide (balance_run below, CoopEvaluator::balance_coop in
// metis_coop.cuh).  The balancer tells its lane policy which ones a run takes (x.note); the policies of the product
// ignore it, the test-only device build (tests/devsim) records it so that a test can show that its inputs reach them.
enum BalancerPath {
    kPathVerifyFailed = 0,   // coop: a predicted forward interval did not verify, the leader re-ran the forward pass
    kPathSeqForward = 1,     // coop: fewer than 4 stages, the forward pass ran sequentially without a prediction
    kPathIrregular = 2,      // a stage's forward interval is empty (coop: the leader places the skipped sub-layers)
    kPathMiddle = 3,         // sub-layers are left between the forward and backward passes (the middle block)
    kPathFirstGe = 4,        // coop: a prediction missed its 32-entry window and searched the whole table
    kPathTail = 5,           // the forward pass ran into the reserved last 8 sub-layers with stages to spare
};

// Execution policies.  `Serial`: one thread owns the task (host, replay kernel, and the throughput
// mode of the search kernel where the 32 lanes of a warp hold 32 different tasks).  A cooperative
// policy (metis_search.cu: WarpLanes) has all lanes of a warp work on ONE task whose scratch lives in
// shared memory: loops over independent elements are strided over the lanes (lane()/width(), then
// sync()), everything else is executed redundantly by every lane on identical data.
struct Serial {
    static constexpr bool kUniform = false;
    MB_HD int lane() const { return 0; }
    MB_HD int width() const { return 1; }
    MB_HD void sync() const {}
    // combine per-lane partial results: largest v, lowest index among equals / largest v
    MB_HD void argmax_first(double &, int &) const {}
    MB_HD double max_all(double v) const { return v; }
    MB_HD bool any(bool p) const { return p; }
    MB_HD void mark(int) const {}              // profiling hook (cooperative mode, profiling build)
    MB_HD void note(int) const {}              // balancer path taken (BalancerPath; recorded by tests/devsim only)
    // lockstep hooks (see Lockstep below): nothing to do when a thread works alone
    MB_HD void converge() const {}
    MB_HD void rejoin(bool) {}
};
#if defined(__CUDACC__)
// `Lockstep`: the bulk round of the search (metis_search.cu, het_first_kernel) - the 32 lanes of a warp hold 32
// different plans of equal stage count and should execute the same instruction stream.  Data-dependent branches
// let lanes drift apart and the hardware only re-joins them at the post-dominator of the branch, which an error
// exit deep inside a loop pushes to the end of the function (measured: 6 of 32 lanes active per instruction on a
// 128-GPU space).  converge() re-joins the lanes that hold a plan at points every one of them reaches exactly once;
// rejoin(p) is called by ALL 32 lanes between the phases and makes the lanes with p == true the group from there on.
struct Lockstep : Serial {
    unsigned mask;
    __device__ Lockstep() : mask(0xFFFFFFFFu) {}
    __device__ void converge() const { __syncwarp(mask); }
    __device__ void rejoin(bool p) { mask = __ballot_sync(0xFFFFFFFFu, p); }
};
#endif
struct SerialUniform : Serial {           // tests: the code paths of the cooperative mode, one lane
    static constexpr bool kUniform = true;
};

constexpr uint64_t kOnes = 0x0101010101010101ULL;

constexpr uint16_t kBroke = 0x8000;   // stage closed because a sub-layer did not fit (that sub-layer is skipped)
constexpr uint16_t kTaken = 0x4000;   // that skipped sub-layer was taken by the backward pass
constexpr uint16_t kPos = 0x3FFF;

// Per-plan scratch (one per thread; indexed with lane-uniform indices wherever the algorithm
// allows, so that the per-thread arrays are accessed coalesced across the warp).
template <int MAXS, int MAXL>
struct Scratch {
    double perf[MAXS];     // stage compute performance of the current attempt (sc_capa_bak)
    double capa[MAXS];     // working capacities / scratch
    double mstate[MAXS];   // memory_state of the last partition_layer call / scratch in adjust
    double extra[MAXS];    // additional_alloc_sc_capa / memory demand
    uint16_t fe[MAXS];     // end of the stage's forward interval in sub-layers | kBroke | kTaken
    uint16_t first[MAXS], lastl[MAXS], cnt[MAXS];   // real layers owned by each stage
    uint16_t part[MAXS + 1];
    uint16_t rs[MAXS + 1]; // first rank of each stage (prefix sum of the group sizes)
    uint8_t gcode[MAXS];   // log2(device group size)
    uint8_t tpc[MAXS];     // log2(tp)
    uint8_t lstk[MAXS];    // stage on which the skipped sub-layer of stage s was placed
    uint8_t got[MAXS];     // stage received a leftover sub-layer
    uint64_t ownerw[MAXL / 8 + 1];   // byte r = stage owning real layer r after the vote (kDropped = none)
    uint64_t subw[MAXL];   // per real layer: byte q = stage of sub-layer 7r+q (below the backward tail); the chain
                           // evaluator keeps the stages of the middle block here instead (byte j - k, up to 7 * MAXL)
};

// ---------------------------------------------------------------------------
// CPython >= 3.12 builtin sum() over a float slice x[a:b] (Neumaier; see oracle fsum)
// ---------------------------------------------------------------------------
MB_HD double py_sum_range(const double *x, int a, int b) {
    if (a >= b) return 0.0;
    double f = 0.0 + x[a];
    double c = 0.0;
    for (int i = a + 1; i < b; ++i) {
        const double v = x[i];
        const double t = f + v;
        if (fabs(f) >= fabs(v)) c += (f - t) + v;
        else c += (v - t) + f;
        f = t;
    }
    if (c != 0.0 && isfinite(c)) f += c;
    return f;
}

// The same, kept out of line and rolled: the cooperative mode is instruction-fetch bound
// (stall_no_instruction is its top stall), so it trades unrolling for code size.
MB_HD_NOINLINE double py_sum_range_compact(const double *x, int a, int b) {
    if (a >= b) return 0.0;
    double f = 0.0 + x[a];
    double c = 0.0;
#pragma unroll 1
    for (int i = a + 1; i < b; ++i) {
        const double v = x[i];
        const double t = f + v;
        if (fabs(f) >= fabs(v)) c += (f - t) + v;
        else c += (v - t) + f;
        f = t;
    }
    if (c != 0.0 && isfinite(c)) f += c;
    return f;
}

template <class X>
MB_HD double sum_range(const double *x, int a, int b) {
    if constexpr (X::kUniform) return py_sum_range_compact(x, a, b);
    else return py_sum_range(x, a, b);
}

// CPython's sum(row[a:b]) for every b in (a, L] in one pass: the running (f, c) of the compensated sum do not depend
// on where the slice ends, only the final `f + c` does.  out[b * n + a], n = L + 1 (entries with b <= a unused).
MB_HD void fill_range_sums(const double *row, int L, int a, double *out) {
    const int n = L + 1;
    double f = 0.0 + row[a];
    double c = 0.0;
    out[(size_t)(a + 1) * n + a] = f;
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
    for (int i = a + 1; i < L; ++i) {
        const double v = row[i];
        const double t = f + v;
        if (fabs(f) >= fabs(v)) c += (f - t) + v;
        else c += (v - t) + f;
        f = t;
        out[(size_t)(i + 1) * n + a] = (c != 0.0 && isfinite(c)) ? f + c : f;
    }
}
MB_HD int range_sum_tables(const MetisProblem &p) { return 2 * p.num_keys + 1; }
MB_HD const double *range_sum_row(const MetisProblem &p, int t, const double *mem, const double *lc, const double *norm) {
    if (t < p.num_keys) return mem + (size_t)t * p.lpad;
    if (t < 2 * p.num_keys) return lc + (size_t)(t - p.num_keys) * p.lpad;
    return p.norm_len >= p.num_layers ? norm : nullptr;     // shorter norm_lc: the search aborts before using it
}

enum RangeTable { kRangeMem = 0, kRangeLc = 1, kRangeNorm = 2 };
// sum(row[a:b]) of one of the three table families; `row` is the same row in T.mem / T.lc / T.norm_lc
template <class X>
MB_HD double range_sum(const Tables &T, int family, int key, const double *row, int a, int b) {
    if (a >= b) return 0.0;
    if (T.rsum && b <= T.p.num_layers) {
        const int n = T.p.num_layers + 1;
        const int t = family == kRangeMem ? key : family == kRangeLc ? T.p.num_keys + key : 2 * T.p.num_keys;
#if defined(__CUDA_ARCH__)
        return __ldg(&T.rsum[((size_t)t * n + b) * n + a]);
#else
        return T.rsum[((size_t)t * n + b) * n + a];
#endif
    }
    return sum_range<X>(row, a, b);
}

// Running form of the same sum for values produced on the fly.
struct PySum {
    double f, c;
    int n;
    MB_HD PySum() : f(0.0), c(0.0), n(0) {}
    MB_HD void add(double v) {
        if (n == 0) { f = 0.0 + v; }
        else {
            const double t = f + v;
            if (fabs(f) >= fabs(v)) c += (f - t) + v;
            else c += (v - t) + f;
            f = t;
        }
        ++n;
    }
    MB_HD double result() const {
        double r = f;
        if (c != 0.0 && isfinite(c)) r += c;
        return r;
    }
};

// 2^-k as a double (k >= 0): dividing by tp = 2^k and multiplying by this round identically.
MB_HD double pow2_neg(int k) {
    const uint64_t bits = (uint64_t)(1023 - k) << 52;
    double d;
    memcpy(&d, &bits, sizeof(d));
    return d;
}

MB_HD int type_of_rank(const Tables &T, int ns, int rank) {
    const int nt = T.p.num_types;
    const int32_t *end = T.run_end + ns * nt;
    const uint8_t *typ = T.run_type + ns * nt;
#pragma unroll 1
    for (int k = 0; k < nt; ++k)
        if (rank < end[k]) return typ[k];
    return typ[nt - 1];
}

// device type at position `idx` of the Q10 rank list (callers check idx < T.p.q10_devices)
MB_HD int type_of_q10(const Tables &T, int ns, int idx) {
    const int nt = T.p.num_types;
    const int32_t *end = T.q10_end + ns * nt;
    const uint8_t *typ = T.run_type + ns * nt;
#pragma unroll 1
    for (int k = 0; k < nt; ++k)
        if (idx < end[k]) return typ[k];
    return typ[nt - 1];
}

MB_HD int key_of(const Tables &T, int type, int tpc, int bs) {
    if (tpc >= T.p.num_tp || bs < 1 || bs > T.p.num_bs) return -1;
    return T.key_index[(type * T.p.num_tp + tpc) * T.p.num_bs + (bs - 1)];
}

// ---------------------------------------------------------------------------
// LayerComputeBalancer.run  (model/load_balancer.py:197-207, passes :216-364)
// in : w.perf[0..S) = sc_capa (kept as sc_capa_bak), out: w.part[0..S], w.cnt
// returns METIS_FATAL_* (0 = ok)
//
// Written for lockstep execution by the 32 lanes of a warp (one plan per lane): the forward scan
// is one flat predicated loop over sub-layers with the same trip count in every lane, the vote is
// a uniform loop over real layers on a per-sub-layer stage map, and the rare general cases are
// loops whose trip count is normally 1.
// ---------------------------------------------------------------------------
template <int MAXS, int MAXL>
MB_HD int fwd_start(const Scratch<MAXS, MAXL> &w, int s) {
    if (s == 0) return 0;
    const uint16_t e = w.fe[s - 1];
    return (e & kPos) + ((e & kBroke) ? 1 : 0);
}

template <int MAXS, int MAXL>
MB_HD bool fwd_nonempty(const Scratch<MAXS, MAXL> &w, int s) {
    return (int)(w.fe[s] & kPos) > fwd_start(w, s);
}

MB_HD void sub_store(uint64_t *subw, int j, int stage) {
    reinterpret_cast<uint8_t *>(subw)[(j / kH) * 8 + (j % kH)] = (uint8_t)stage;
}

MB_HD int popc64(uint64_t v) {
#if defined(__CUDA_ARCH__)
    return __popcll(v);
#else
    return __builtin_popcountll(v);
#endif
}
MB_HD int ctz64(uint64_t v) {            // v != 0
#if defined(__CUDA_ARCH__)
    return __ffsll((long long)v) - 1;
#else
    return __builtin_ctzll(v);
#endif
}
MB_HD int popc32(uint32_t v) {
#if defined(__CUDA_ARCH__)
    return __popc(v);
#else
    return __builtin_popcount(v);
#endif
}
MB_HD int ctz32(uint32_t v) {            // v != 0
#if defined(__CUDA_ARCH__)
    return __ffs((int)v) - 1;
#else
    return __builtin_ctz(v);
#endif
}
MB_HD int clz32(uint32_t v) {            // v != 0
#if defined(__CUDA_ARCH__)
    return __clz((int)v);
#else
    return __builtin_clz(v);
#endif
}
MB_HD int clz64(uint64_t v) {            // v != 0
#if defined(__CUDA_ARCH__)
    return __clzll((long long)v);
#else
    return __builtin_clzll(v);
#endif
}

// 0x80 in every byte of x that equals c
MB_HD uint64_t swar_eq(uint64_t x, int c) {
    const uint64_t y = x ^ ((uint64_t)c * kOnes);
    const uint64_t lo7 = 0x7F7F7F7F7F7F7F7FULL;
    return ~((((y & lo7) + lo7) | y) | lo7);
}

// number of bytes of x (bytes 0..6) equal to c
MB_HD int swar_count(uint64_t x, int c) { return popc64(swar_eq(x, c) & 0x0080808080808080ULL); }

// Owner of a real layer from the packed stages of its 7 sub-layers (bytes 0..6 of v, byte 7 = 0xFF).
// Reference (model/load_balancer.py:293-296): the stage holding more than half of them, else nobody (kDropped,
// quirk Q5).  A stage holding >= 4 of 7 holds the middle one or one of the first three, so four candidates do.
// `plurality` (opt-in METIS_FIX_Q5, not the reference): the stage holding most, lowest stage among equals.
MB_HD int layer_owner(uint64_t v, bool plurality) {
    if (plurality) {
        int best = 0, own = (int)kDropped;
#pragma unroll 1
        for (int q = 0; q < kH; ++q) {
            const int cq = (int)((v >> (8 * q)) & 0xFF);
            const int n = swar_count(v, cq);
            if (n > best || (n == best && cq < own)) { best = n; own = cq; }
        }
        return own;
    }
    const int c3 = (int)((v >> 24) & 0xFF);
    if (swar_count(v, c3) * 2 > kH) return c3;                // count > hallucination / 2 (:295)
    const int c0 = (int)(v & 0xFF), c1 = (int)((v >> 8) & 0xFF), c2 = (int)((v >> 16) & 0xFF);
    if (swar_count(v, c0) * 2 > kH) return c0;
    if (c1 != c0 && swar_count(v, c1) * 2 > kH) return c1;
    if (c2 != c1 && c2 != c0 && swar_count(v, c2) * 2 > kH) return c2;
    return (int)kDropped;
}

template <int MAXS, int MAXL, class X>
MB_HD int balance_run(const Tables &T, int S, Scratch<MAXS, MAXL> &w, const X &x) {
    const int L = T.p.num_layers;
    if (T.p.norm_len < L) return METIS_FATAL_INDEX;       // expand_lc_demand[layer_id] IndexError (:219/:238)
    const double *dlay = T.dlay;
    const double *lc = T.norm_lc;
    const int N = kH * L;
    const int lim = (N - 1 - kH) > 0 ? (N - 1 - kH) : 0;   // :218
    const int last = S - 1;
    int broken = METIS_FATAL_NONE;                           // scratch invariant violated (never observed): reported at
                                                             // the end - an exit inside the loops below would keep
                                                             // the lanes of the bulk round from re-joining (Lockstep)

    x.sync();                                                // lane-strided writes below: earlier readers are done
#pragma unroll (X::kUniform ? 1 : 0)
    for (int s = x.lane(); s < S; s += x.width()) { w.capa[s] = w.perf[s]; w.got[s] = 0; w.cnt[s] = 0; }
    x.sync();

    x.mark(10);
    // ---- forward pass (:216-231): flat scan, layer by layer, 7 sub-layers each -----------------
    int k = 0, sTop = -1;
    bool topSkip = false;
    if (S > 1) {
        int s = 0, j = 0;
        double c = w.capa[0];
#pragma unroll (X::kUniform ? 1 : 0)
        for (int r = 0; r + 1 < L; ++r) {
            const double d = dlay[r];
            const int nsub = (r == L - 2) ? kH - 1 : kH;     // the last 8 sub-layers are reserved
            // one plan per thread: the layer's packed stage word is built in registers and stored once (the skipped
            // sub-layers' bytes are filled in by the leftover pass below)
            const int s_in = s;
            uint64_t v = 0;
#pragma unroll
            for (int q = 0; q < kH; ++q) {
                if (q < nsub) {
                    if (s < last) {
                        if (c > d) {
                            c -= d;
                            v |= (uint64_t)(uint32_t)s << (8 * q);
                        } else {                                 // sub-layer j does not fit: skipped, stage closes
                            w.capa[s] = c;
                            w.fe[s] = (uint16_t)(j | kBroke);
                            ++s;
                            c = w.capa[s];
                        }
                    }
                    ++j;
                }
            }
            if (s_in < last) w.subw[r] = v;
        }
        if (s < last) {                                          // ran into the reserved tail
            x.note(kPathTail);
            w.capa[s] = c;
            w.fe[s] = (uint16_t)lim;
#pragma unroll (X::kUniform ? 1 : 0)
            for (int t = s + 1; t < last; ++t) w.fe[t] = (uint16_t)lim;
            k = lim;
            sTop = s;
        } else {
            k = (w.fe[last - 1] & kPos) + 1;
            sTop = last - 1;
            topSkip = true;
        }
    }

    x.mark(11);
    x.converge();
    // ---- backward pass (:233-249): last stage takes a contiguous tail [m, N) -----------------
    int m;
    {
        double c = w.capa[last];
        const double dl = dlay[L - 1];
#pragma unroll (X::kUniform ? 1 : 0)
        for (int i = 0; i < kH; ++i) c -= dl;               // unconditional while len < hallucination (:237-241)
        m = N - kH;
        int sp = S - 2;
#pragma unroll (X::kUniform ? 1 : 0)
        while (m > 0) {
            const int j = m - 1;
            bool un = (j >= k);
            if (!un) {                                       // below k only skipped sub-layers are unassigned
#pragma unroll (X::kUniform ? 1 : 0)
                while (sp >= 0 && (!(w.fe[sp] & kBroke) || (int)(w.fe[sp] & kPos) > j)) --sp;
                un = (sp >= 0 && (int)(w.fe[sp] & kPos) == j);
            }
            if (!un) break;                                  // (layer_id + 1) != min(...) from here on (:243)
            const double d = dlay[j / kH];
            if (!(c > d)) break;                             // :246 fails; every later id fails :243
            c -= d;
            m = j;
            if (j < k) w.fe[sp] |= kTaken;
        }
        w.capa[last] = c;
    }

    x.mark(12);
    x.converge();
    // ---- leftovers (:251-287), ascending: first the skipped sub-layers, then the middle block --
    // get_proper_stage: lo = stage of the largest assigned id below j whose stage holds nothing
    // above j, hi = stage of the smallest assigned id above j whose stage holds nothing below j.
    {
        int start = 0;                                        // first sub-layer of stage s's forward interval
#pragma unroll (X::kUniform ? 1 : 0)
        for (int s = 0; s < last; ++s) {
            const uint16_t e = w.fe[s];
            const int pos = e & kPos;
            const int next_start = pos + ((e & kBroke) ? 1 : 0);
            if ((e & (kBroke | kTaken)) != kBroke) { start = next_start; continue; }
            const int j = pos;
            int lo = 0;
            if (pos > start) {
                lo = s;                                       // common case: stage s itself ends right below j
            } else {
                x.note(kPathIrregular);
#pragma unroll (X::kUniform ? 1 : 0)
                for (int u = s;; --u) {
                    if (u < s) {                              // skipped sub-layer of stage u (already placed)
                        const int t = w.lstk[u];
                        const bool above = (t == last) || (fwd_nonempty(w, t) && fwd_start(w, t) > j);
                        if (!above) { lo = t; break; }
                    }
                    if (fwd_nonempty(w, u)) { lo = u; break; }
                    if (u == 0) break;
                }
            }
            int hi = s + 1;
            if (hi < last && !((int)(w.fe[hi] & kPos) > next_start && !w.got[hi])) {
                ++hi;                                         // stage s+1 is empty or already holds a leftover
#pragma unroll (X::kUniform ? 1 : 0)
                while (hi < last && (!fwd_nonempty(w, hi) || w.got[hi])) ++hi;
            }
            if (lo > hi) { broken = METIS_FATAL_SCRATCH; hi = lo; }
            int pick = lo;
            double best = w.capa[lo];
#pragma unroll (X::kUniform ? 1 : 0)
            for (int t = lo + 1; t <= hi; ++t)
                if (w.capa[t] > best) { best = w.capa[t]; pick = t; }
            w.capa[pick] -= dlay[j / kH];
            w.lstk[s] = (uint8_t)pick;
            w.got[pick] = 1;
            sub_store(w.subw, j, pick);
            start = next_start;
        }
    }
    x.converge();
    const int nblk = m - k;                                   // any length up to 7 * L: the picks go to subw
    if (nblk > 0) x.note(kPathMiddle);
    {
        int below = -1;                                       // stage of the nearest block item not on `last`
#pragma unroll (X::kUniform ? 1 : 0)
        for (int t = 0; t < nblk; ++t) {
            const int j = k + t;
            int lo = 0;
            if (below >= 0) lo = below;
            else if (sTop >= 0) {
#pragma unroll (X::kUniform ? 1 : 0)
                for (int u = sTop;; --u) {
                    if (u < sTop || topSkip) {
                        const uint16_t eu = w.fe[u];
                        if ((eu & (kBroke | kTaken)) == kBroke) {
                            const int t2 = w.lstk[u];
                            if (t2 != last) { lo = t2; break; }   // forward intervals all lie below the block
                        }
                    }
                    if (fwd_nonempty(w, u)) { lo = u; break; }
                    if (u == 0) break;
                }
            }
            int pick = lo;
            double best = w.capa[lo];
#pragma unroll (X::kUniform ? 1 : 0)
            for (int t2 = lo + 1; t2 <= last; ++t2)
                if (w.capa[t2] > best) { best = w.capa[t2]; pick = t2; }
            w.capa[pick] -= dlay[j / kH];
            if (pick != last) below = pick;
            sub_store(w.subw, j, pick);
        }
    }

    x.mark(13);
    x.converge();
    // ---- majority vote back to real layers (:290-308) ------------------------------------------
    // A stage holding >= 4 of a layer's 7 sub-layers holds the middle one or one of the first
    // three, so at most four candidates are counted (SWAR byte compare on the packed layer word).
    x.sync();
    int run_own = (int)kDropped, run_first = 0, run_len = 0;
#pragma unroll (X::kUniform ? 1 : 0)
    for (int r = x.lane(); r < L; r += x.width()) {
        const int nlow = m - kH * r;                         // sub-layers of r below the backward tail
        int own;
        if (nlow <= 0) {
            own = last;
        } else {
            uint64_t v = w.subw[r];
            if (nlow < kH) {
                const uint64_t mask = (1ULL << (8 * nlow)) - 1ULL;
                v = (v & mask) | (((uint64_t)last * kOnes) & ~mask);
            }
            v |= 0xFF00000000000000ULL;
            own = layer_owner(v, (T.p.corrected & METIS_FIX_Q5) != 0);
        }
        reinterpret_cast<uint8_t *>(w.ownerw)[r] = (uint8_t)own;
        {
            // first / last / count of the layers of each stage (:300-306), one update per run of equal owners
            if (own == run_own) ++run_len;
            else {
                if (run_own != (int)kDropped) {
                    if (w.cnt[run_own] == 0) w.first[run_own] = (uint16_t)run_first;
                    w.lastl[run_own] = (uint16_t)(r - 1);
                    w.cnt[run_own] = (uint16_t)(w.cnt[run_own] + run_len);
                }
                run_own = own; run_first = r; run_len = 1;
            }
        }
    }
    if (run_own != (int)kDropped) {
        if (w.cnt[run_own] == 0) w.first[run_own] = (uint16_t)run_first;
        w.lastl[run_own] = (uint16_t)(L - 1);
        w.cnt[run_own] = (uint16_t)(w.cnt[run_own] + run_len);
    }
    x.sync();
    x.mark(14);
    x.converge();
    uint8_t *owner = reinterpret_cast<uint8_t *>(w.ownerw);
    x.sync();
#pragma unroll (X::kUniform ? 1 : 0)
    for (int s = x.lane(); s < S; s += x.width())            // :300-306
        w.capa[s] = w.cnt[s] ? w.perf[s] - range_sum<X>(T, kRangeNorm, 0, lc, w.first[s], (int)w.lastl[s] + 1) : w.perf[s];
    x.sync();

    x.mark(15);
    x.converge();
    // ---- boundary adjustment (:310-356): at most three committed single-layer moves ---------
#pragma unroll (X::kUniform ? 1 : 0)
    for (int n = 1; n <= 3; ++n) {
        int top = 0x7FFFFFFF;
        double maxc = -INFINITY;
#pragma unroll (X::kUniform ? 1 : 0)
        for (int t = x.lane(); t < S; t += x.width())        // stable: lowest index among equal maxima (:329-331)
            if (w.capa[t] > maxc) { maxc = w.capa[t]; top = t; }
        x.argmax_first(maxc, top);
        if (top == 0x7FFFFFFF) top = 0;
        int nb = -1;
        double val = INFINITY;
        if (top - 1 >= 0 && w.capa[top - 1] < val) { nb = top - 1; val = w.capa[top - 1]; }
        if (top + 1 < S && w.capa[top + 1] < val) { nb = top + 1; }
        if (nb < 0 || w.cnt[nb] <= 1) break;                 // no-op rounds leave the state unchanged
        const int layer = (top > nb) ? w.lastl[nb] : w.first[nb];
        const double dl = lc[layer];
        const double ntop = w.capa[top] - dl;
        const double nnb = w.capa[nb] + dl;
        double newmax = -INFINITY;
#pragma unroll (X::kUniform ? 1 : 0)
        for (int t = x.lane(); t < S; t += x.width()) {
            const double v = (t == top) ? ntop : (t == nb) ? nnb : w.capa[t];
            if (v > newmax) newmax = v;
        }
        newmax = x.max_all(newmax);
        if (newmax > maxc) break;                            // :352 (not committed)
        x.sync();
        owner[layer] = (uint8_t)top;
        w.capa[top] = ntop;
        w.capa[nb] = nnb;
        if (top > nb) { int r = layer - 1; while (owner[r] != nb) --r; w.lastl[nb] = (uint16_t)r; }
        else          { int r = layer + 1; while (owner[r] != nb) ++r; w.first[nb] = (uint16_t)r; }
        if (w.cnt[top] == 0) { w.first[top] = (uint16_t)layer; w.lastl[top] = (uint16_t)layer; }
        else {
            if (layer < (int)w.first[top]) w.first[top] = (uint16_t)layer;
            if (layer > (int)w.lastl[top]) w.lastl[top] = (uint16_t)layer;
        }
        ++w.cnt[top];
        --w.cnt[nb];
        x.sync();
    }

    x.mark(16);
    x.converge();
    w.part[0] = 0;                                           // :358-364
#pragma unroll (X::kUniform ? 1 : 0)
    for (int s = 0; s < S; ++s) w.part[s + 1] = (uint16_t)(w.part[s] + w.cnt[s]);
    return broken;
}

// ---------------------------------------------------------------------------
// DataLoadBalancer.partition_data (model/load_balancer.py:155-179) on a rank range.
// Replicas are grouped in runs of equal device type (ranks are laid out type by type).
// ---------------------------------------------------------------------------
struct HSplit {
    int nruns;
    int type[METIS_MAX_TYPES];
    int n[METIS_MAX_TYPES];      // replicas in the run
    int base[METIS_MAX_TYPES];   // int(bs * share)
    int plus[METIS_MAX_TYPES];   // leading replicas of the run that get +1
};

MB_HD_NOINLINE int partition_data(const Tables &T, int ns, int rank_lo, int count, int dp, int tpc, int bs,
                                  HSplit &out, uint32_t &aux, bool q10 = false) {
    const int gsz = count / dp;
    double perf[METIS_MAX_TYPES];
    PySum total;
    out.nruns = 0;
#pragma unroll 1
    for (int i = 0; i < dp; ++i) {
        const int t = q10 ? type_of_q10(T, ns, rank_lo + i * gsz) : type_of_rank(T, ns, rank_lo + i * gsz);
        if (out.nruns == 0 || out.type[out.nruns - 1] != t) {
            const int key = key_of(T, t, tpc, 1);
            if (key < 0) { aux = ((uint32_t)tpc << 16) | 1u; return METIS_FATAL_KEY_EXEC; }
            const double e = T.exec_full[key];
            if (e == 0.0) return METIS_FATAL_ZERODIV;
            out.type[out.nruns] = t;
            out.n[out.nruns] = 0;
            perf[out.nruns] = 1. / e;
            ++out.nruns;
        }
        ++out.n[out.nruns - 1];
        total.add(perf[out.nruns - 1]);
    }
    const double tot = total.result();
    double frac[METIS_MAX_TYPES];
    int assigned = 0;
#pragma unroll 1
    for (int r = 0; r < out.nruns; ++r) {
        const double v = (double)bs * (perf[r] / tot);
        const int b = (int)v;
        out.base[r] = b;
        out.plus[r] = 0;
        frac[r] = v - (double)b;
        assigned += b * out.n[r];
    }
    int rem = bs - assigned;
    bool used[METIS_MAX_TYPES];
#pragma unroll 1
    for (int r = 0; r < out.nruns; ++r) used[r] = false;
#pragma unroll 1
    for (int it = 0; it < out.nruns && rem > 0; ++it) {      // stable descending order of the remainders
        int pick = -1;
#pragma unroll 1
        for (int r = 0; r < out.nruns; ++r)
            if (!used[r] && (pick < 0 || frac[r] > frac[pick])) pick = r;
        used[pick] = true;
        const int g = rem < out.n[pick] ? rem : out.n[pick];
        out.plus[pick] = g;
        rem -= g;
    }
    if (rem > 0) return METIS_FATAL_SCRATCH;                  // reference would raise IndexError (:177)
    return METIS_FATAL_NONE;
}

// Sink interface expected by evaluate_plan (see metis_search.cu / tests/hostsim):
//   void partition_call(); void balancer_run(); void keyerror(); void phase(int) (profiling hook);
//   void fatal(uint32_t ordinal, int code, uint32_t aux);
//   void emit(const PlanDesc&, int step, int nrep, double cost, const uint8_t *tpc, const uint16_t *part);

// Optional tap of intermediate values for the verbose transcript (metis_trace.cuh); null in the search kernels.
struct TraceTap {
    double *demand;     // [S] stage_memory_demand of the last partition attempt (load_balancer.py:133)
    double *state;      // [S] memory_state of that attempt
    double cost[5];     // execution_cost, fb_sync_cost, max parameter update, max dp, pp_cost (cost_estimator.py:239-240)
};

MB_HD int halvings_of(const MetisProblem &p, int S, const uint8_t *gcode, const uint8_t *tpc, int bs_total) {
    int ltp = 0, lbs = 0;
    while ((2 << ltp) <= p.max_tp) ++ltp;                     // floor(log2(max_tp))
    while ((2 << lbs) <= p.max_bs) ++lbs;
    int u = 0;
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
    for (int s = 0; s < S; ++s) {
        const int g = gcode[s], t = tpc[s];
        int lm = 0;                                           // floor(log2(mbs)), mbs = bs_total >> log2(dp)
        while ((2 << lm) <= (bs_total >> (g - t))) ++lm;
        int room = g - t;
        if (ltp - t < room) room = ltp - t;
        if (lbs - lm < room) room = lbs - lm;
        if (room > 0) u += room;
    }
    return u;
}

template <int MAXS, int MAXL, class X = Serial, bool ONE = false>
struct PlanEvaluator {
    const Tables &T;
    Scratch<MAXS, MAXL> &w;
    X x;
    PlanDesc pd;
    int bs_total;         // gbs // batches
    int nbad;             // stages of the current strategy that violate _is_valid_strategies
    uint32_t aux;
    TraceTap *tap;        // verbose transcript only

    MB_HD PlanEvaluator(const Tables &t, Scratch<MAXS, MAXL> &s, const X &lanes = X())
        : T(t), w(s), x(lanes), bs_total(0), nbad(0), aux(0), tap(nullptr) {}

    MB_HD int group(int s) const { return 1 << w.gcode[s]; }
    MB_HD int dp_of(int s) const { return (1 << w.gcode[s]) >> w.tpc[s]; }

    // one stage of IntraStagePlanGenerator._is_valid_strategies (search_space/plan.py:238-249);
    // gbs // dp // batches == (gbs // batches) >> log2(dp) because dp is a power of two
    MB_HD bool stage_bad(int g, int t) const {
        const int mbs = bs_total >> (g - t);
        return mbs == 0 || mbs > T.p.max_bs || (1 << t) > T.p.max_tp;
    }

    // Start of a plan.  The reference starts from (dp = group, tp = 1) and, while no memory state
    // exists, always halves the stage with the largest dp (plan.py:252-266).  Every strategy on that
    // path is invalid (mbs == 0 somewhere) until all dp <= B = 2^floor(log2(gbs // batches)), and no
    // stage with dp <= B is touched before that, so the first strategy that can be valid is
    // tp_s = max(1, group_s / B) - jumping there skips only strategies that have no effect.
    // If that strategy is invalid it stays invalid for the rest of the chain (mbs and tp only grow).
    // returns 1 ready, 0 plan has no valid strategy, -1 scratch limits exceeded
    MB_HD int begin(const PlanDesc &plan) {
        pd = plan;
        if (pd.S > MAXS || T.p.num_layers > MAXL) return -1;
        bs_total = T.p.gbs / pd.batches;
        int lb = 0;
#pragma unroll (X::kUniform ? 1 : 0)
        while ((2 << lb) <= bs_total) ++lb;
        nbad = 0;
        int a = 0;
        for (int s = 0; s < pd.S; ++s) {                     // set_groups + first strategy in one pass
            const int g = pd.row[s];
            const int t = g > lb ? g - lb : 0;
            if (stage_bad(g, t)) { nbad = 1; return 0; }     // the plan can never become valid: drop it now
            w.gcode[s] = (uint8_t)g;
            w.rs[s] = (uint16_t)a;
            a += 1 << g;
            w.tpc[s] = (uint8_t)t;
        }
        w.rs[pd.S] = (uint16_t)a;
        return nbad == 0 ? 1 : 0;
    }

    // IntraStagePlanGenerator._next_strategy (search_space/plan.py:251-268); keeps nbad current
    MB_HD bool next_strategy(bool have_state) {
        int pick = -1;
        if (have_state) {
            double best = 0.0;
#pragma unroll (X::kUniform ? 1 : 0)
            for (int s = 0; s < pd.S; ++s)
                if (w.gcode[s] != w.tpc[s] && (pick < 0 || w.mstate[s] < best)) { pick = s; best = w.mstate[s]; }
        } else {                                             // default state 1/dp: largest dp first
            int best = -1;
#pragma unroll (X::kUniform ? 1 : 0)
            for (int s = 0; s < pd.S; ++s) {
                const int ldp = (int)w.gcode[s] - (int)w.tpc[s];
                if (ldp != 0 && ldp > best) { pick = s; best = ldp; }
            }
        }
        if (pick < 0) return false;
        const int g = w.gcode[pick], t = w.tpc[pick];
        nbad += (stage_bad(g, t + 1) ? 1 : 0) - (stage_bad(g, t) ? 1 : 0);
        x.sync();                                            // every lane has read tpc[pick] before any lane rewrites it
        w.tpc[pick] = (uint8_t)(t + 1);
        x.sync();
        return true;
    }

    MB_HD bool valid() const { return nbad == 0; }

    // Scheduling hint only (never part of a result): how many more strategies the chain of this plan can visit.
    // Every step of IntraStagePlanGenerator halves the dp of ONE stage (search_space/plan.py:257-266), a stage can
    // be halved until dp = 1, tp = max_tp or mbs = max_bs; measured on BASELINE configs[2], the number of
    // LayerComputeBalancer runs of a chain is 2 * halvings + 2 with correlation 0.98.
    MB_HD int halvings() const { return halvings_of(T.p, pd.S, w.gcode, w.tpc, bs_total); }

    // StagePerformance.get_device_group_memory_capacity, one stage (model/device_group.py:87-101)
    MB_HD double memory_capacity(int a, int b) const {
        const int nt = T.p.num_types;
        if (ONE || nt == 1) return T.type_memory[0] * (double)(b - a);
        const int32_t *end = T.run_end + pd.ns * nt;
        const uint8_t *typ = T.run_type + pd.ns * nt;
        PySum acc;
        int lo = 0;
#pragma unroll (X::kUniform ? 1 : 0)
        for (int k = 0; k < nt; ++k) {
            const int hi = end[k];
            const int x = (a > lo ? a : lo), y = (b < hi ? b : hi);
            if (y > x) acc.add(T.type_memory[typ[k]] * (double)(y - x));
            lo = hi;
        }
        return acc.result();
    }

    // hetero replica cost for StagePerformance (model/device_group.py:40-52): sum of full-model times
    MB_HD int replica_perf_cost(int type, int tpc, int h, double &out) {
        double acc = 0.;
#pragma unroll (X::kUniform ? 1 : 0)
        for (int bit = 30; bit >= 0; --bit) {
            const int piece = 1 << bit;
            if (!(h & piece)) continue;
            const int key = key_of(T, type, tpc, piece);
            if (key < 0) { aux = ((uint32_t)tpc << 16) | (uint32_t)piece; return METIS_FATAL_KEY_EXEC; }
            acc += T.exec_full[key];
        }
        out = acc;
        return 0;
    }

    // mixed-type stage of get_intra_stage_compute_performance (model/device_group.py:68-76)
    MB_HD_NOINLINE int hetero_performance(int a, int b, int dp, int tpc, double &p) {
        HSplit hs;
        int rc = partition_data(T, pd.ns, a, b - a, dp, tpc, bs_total, hs, aux);
        if (rc) return rc;
        double mx = -INFINITY;
#pragma unroll (X::kUniform ? 1 : 0)
        for (int r = 0; r < hs.nruns; ++r) {
            double c;
            if (hs.plus[r] > 0) {
                rc = replica_perf_cost(hs.type[r], tpc, hs.base[r] + 1, c);
                if (rc) return rc;
                if (c > mx) mx = c;
            }
            if (hs.plus[r] < hs.n[r]) {
                rc = replica_perf_cost(hs.type[r], tpc, hs.base[r], c);
                if (rc) return rc;
                if (c > mx) mx = c;
            }
        }
        p = (mx != 0.0) ? 1. / mx : 0.0;
        return 0;
    }

    // start rank of stage s (prefix sum of the group sizes, filled by set_groups)
    MB_HD int rank_start(int s) const { return w.rs[s]; }

    MB_HD void set_groups(const uint8_t *row) {
        int a = 0;
#pragma unroll (X::kUniform ? 1 : 0)
        for (int s = 0; s < pd.S; ++s) { w.gcode[s] = row[s]; w.rs[s] = (uint16_t)a; a += 1 << row[s]; }
        w.rs[pd.S] = (uint16_t)a;
    }

    // StagePerformance.get_intra_stage_compute_performance (model/device_group.py:54-85) -> w.perf
    MB_HD int compute_performance() {
        const bool one_type = ONE || T.p.num_types == 1;
        int fail = 0;
        x.sync();
#pragma unroll (X::kUniform ? 1 : 0)
        for (int s = x.lane(); s < pd.S; s += x.width()) {
            const int g = w.gcode[s], tpc = w.tpc[s];
            double p = 0.0;
            if (one_type) {
                const int bs = bs_total >> (g - tpc);
                const int key = key_of(T, 0, tpc, bs);
                if (key < 0) { aux = ((uint32_t)tpc << 16) | (uint32_t)bs; fail = METIS_FATAL_KEY_EXEC; }
                else if (T.exec_full[key] == 0.0) fail = METIS_FATAL_ZERODIV;
                else p = T.inv_exec[key];                     // 1. / profile_cost
            } else {
                const int a = rank_start(s), b = a + (1 << g);
                const int ta = type_of_rank(T, pd.ns, a), tb = type_of_rank(T, pd.ns, b - 1);
                if (ta == tb) {
                    const int bs = bs_total >> (g - tpc);
                    const int key = key_of(T, ta, tpc, bs);
                    if (key < 0) { aux = ((uint32_t)tpc << 16) | (uint32_t)bs; fail = METIS_FATAL_KEY_EXEC; }
                    else if (T.exec_full[key] == 0.0) fail = METIS_FATAL_ZERODIV;
                    else p = T.inv_exec[key];
                } else {
                    const int rc = hetero_performance(a, b, 1 << (g - tpc), tpc, p);
                    if (rc) fail = rc;
                }
            }
            w.perf[s] = p;
            w.extra[s] = fail ? (double)fail + (double)aux * 256.0 : 0.0;   // per-stage error mailbox (cooperative mode)
        }
        x.sync();
        x.converge();
        PySum total;
#pragma unroll (X::kUniform ? 1 : 0)
        for (int s = 0; s < pd.S; ++s) {                     // first failing stage in stage order, like the reference
            if (w.extra[s] != 0.0) {
                const uint64_t code = (uint64_t)w.extra[s];
                aux = (uint32_t)(code >> 8);
                return (int)(code & 0xFF);
            }
            total.add(w.perf[s]);
        }
        const double tot = total.result();
        if (tot == 0.0) return METIS_FATAL_ZERODIV;
        x.sync();
#pragma unroll (X::kUniform ? 1 : 0)
        for (int s = x.lane(); s < pd.S; s += x.width()) w.perf[s] = w.perf[s] / tot;
        x.sync();
        return 0;
    }

    // mixed-type stage of _get_stage_memory_demand (model/load_balancer.py:45-52, quirk Q6)
    MB_HD_NOINLINE int hetero_memory_demand(int s, int type0, double &demand) {
        const int la = w.part[s], lb = w.part[s + 1], tpc = w.tpc[s];
        HSplit hs;                                           // whole-cluster device list (quirk Q6)
        const int rc = partition_data(T, pd.ns, 0, T.p.q10_devices, dp_of(s), tpc, bs_total, hs, aux, true);
        if (rc) return rc;
#pragma unroll (X::kUniform ? 1 : 0)
        for (int r = 0; r < hs.nruns; ++r)
#pragma unroll (X::kUniform ? 1 : 0)
            for (int i = 0; i < hs.n[r]; ++i) {
                const int h = hs.base[r] + (i < hs.plus[r] ? 1 : 0);
#pragma unroll (X::kUniform ? 1 : 0)
                for (int bit = 30; bit >= 0; --bit) {
                    const int piece = 1 << bit;
                    if (!(h & piece)) continue;
                    const int key = key_of(T, type0, tpc, piece);
                    if (key < 0) { aux = ((uint32_t)tpc << 16) | (uint32_t)piece; return METIS_FATAL_KEY_MEMORY; }
                    demand += range_sum<X>(T, kRangeMem, key, T.mem + (size_t)key * T.p.lpad, la, lb) * kMemCoef;
                }
            }
        return 0;
    }

    // Opt-in METIS_FIX_Q6 (NOT the reference; mirrored by oracle.stage_memory_demand_own_type): the stage's own
    // devices decide the memory profile; a mixed-type stage needs the memory of its largest replica.
    MB_HD_NOINLINE int memory_demand_own_type(int s, double &demand) {
        const int la = w.part[s], lb = w.part[s + 1], tpc = w.tpc[s], g = w.gcode[s];
        const int a = rank_start(s), b = a + (1 << g);
        const int ta = type_of_rank(T, pd.ns, a), tb = type_of_rank(T, pd.ns, b - 1);
        if (ta == tb) {
            const int bs = bs_total >> (g - tpc);
            const int key = key_of(T, ta, tpc, bs);
            if (key < 0) { aux = ((uint32_t)tpc << 16) | (uint32_t)bs; return METIS_FATAL_KEY_MEMORY; }
            demand += range_sum<SerialUniform>(T, kRangeMem, key, T.mem + (size_t)key * T.p.lpad, la, lb) * kMemCoef;
            return 0;
        }
        HSplit hs;
        const int rc = partition_data(T, pd.ns, a, b - a, 1 << (g - tpc), tpc, bs_total, hs, aux);
        if (rc) return rc;
        double worst = 0.0;
#pragma unroll 1
        for (int r = 0; r < hs.nruns; ++r)
#pragma unroll 1
            for (int v = 0; v < 2; ++v) {
                const int cntv = v ? hs.plus[r] : hs.n[r] - hs.plus[r];
                const int h = hs.base[r] + v;
                if (cntv <= 0 || h == 0) continue;
                double need = 0.0;
#pragma unroll 1
                for (int bit = 30; bit >= 0; --bit) {
                    const int piece = 1 << bit;
                    if (!(h & piece)) continue;
                    const int key = key_of(T, hs.type[r], tpc, piece);
                    if (key < 0) { aux = ((uint32_t)tpc << 16) | (uint32_t)piece; return METIS_FATAL_KEY_MEMORY; }
                    need += range_sum<SerialUniform>(T, kRangeMem, key, T.mem + (size_t)key * T.p.lpad, la, lb) * kMemCoef;
                }
                if (need > worst) worst = need;
            }
        demand += worst;
        return 0;
    }

    // LayerLoadBalancer._adj_compute_performance (model/load_balancer.py:71-107)
    // in: w.perf (c_capa), w.extra (m_demand); out: w.perf; returns 1 = None, 0 ok, <0 fatal (negated code)
    MB_HD_NOINLINE int adjust_performance() {
        const int S = pd.S;
        const bool one_type = ONE || T.p.num_types == 1;
        double *ratio = reinterpret_cast<double *>(w.subw);      // free after the vote (MAXL >= MAXS)
        x.sync();
#pragma unroll (X::kUniform ? 1 : 0)
        for (int s = x.lane(); s < S; s += x.width()) {          // independent per stage (:80-89)
            const int a = one_type ? 0 : rank_start(s), b = a + group(s);
            const double c = w.perf[s], md = w.extra[s];
            const double mc = one_type ? T.type_memory[0] * (double)group(s) : memory_capacity(a, b);
            double av, adj;
            if (mc > md) {
                adj = c;
                av = (c * mc / md) - c;
            } else {
                av = 0.0;
                adj = c * (mc / md) * 0.9;
            }
            w.capa[s] = av;           // available_compute_capacity
            w.mstate[s] = adj;        // adj_sc_capa
        }
        x.sync();
        double need = 0.;
        PySum avail_sum;
#pragma unroll (X::kUniform ? 1 : 0)
        for (int s = 0; s < S; ++s) {                            // order-dependent accumulations (:89-91)
            const int a = one_type ? 0 : rank_start(s);
            const double mc = one_type ? T.type_memory[0] * (double)group(s) : memory_capacity(a, a + group(s));
            if (!(mc > w.extra[s])) need += (w.perf[s] - w.mstate[s]);
            avail_sum.add(w.capa[s]);
        }
        if (avail_sum.result() < need) return 1;
        x.sync();
#pragma unroll (X::kUniform ? 1 : 0)
        for (int s = x.lane(); s < S; s += x.width()) w.extra[s] = 0.;
        x.sync();
        int guard = 0;
#pragma unroll (X::kUniform ? 1 : 0)
        while (need > 0.01) {
            PySum tot;
#pragma unroll (X::kUniform ? 1 : 0)
            for (int s = 0; s < S; ++s) tot.add(w.capa[s] > 0.001 ? w.perf[s] : 0.0);
            const double tmp_total = tot.result();
            x.sync();
#pragma unroll (X::kUniform ? 1 : 0)
            for (int s = x.lane(); s < S; s += x.width())        // c_capa_ratio list (:98), before the updates
                ratio[s] = w.capa[s] > 0.001 ? w.perf[s] / tmp_total : 0.0;
            x.sync();
#pragma unroll (X::kUniform ? 1 : 0)
            for (int s = 0; s < S; ++s) {                        // :100-104, sequential: `need` changes as it goes
                const double av = w.capa[s];
                const double want = need * ratio[s];
                const double give = want > av ? av : want;
                w.extra[s] += give;
                w.capa[s] -= give;
                need -= give;
            }
            if (++guard > 4096) return -METIS_FATAL_HANG;
        }
        x.sync();
#pragma unroll (X::kUniform ? 1 : 0)
        for (int s = x.lane(); s < S; s += x.width()) w.perf[s] = w.extra[s] + w.mstate[s];
        x.sync();
        return 0;
    }

    // One attempt of LayerLoadBalancer.partition_layer (model/load_balancer.py:127-143) after
    // balance_run: memory demand (:29-55), OOM test (:57-63) and, when memory is exceeded, the
    // capacity re-weighting.  returns 1 = partition accepted (w.mstate = memory_state), 2 = retry
    // with the adjusted w.perf, 0 = (None, -1, None), <0 = fatal (negated code).  After the third
    // failed attempt the reference still evaluates _adj_compute_performance and discards it; that
    // call is skipped here.
    MB_HD int memory_phase(int attempt) {
        const int S = pd.S;
        const bool one_type = ONE || T.p.num_types == 1;
        const int type0 = T.run_type[pd.ns * T.p.num_types];
        const bool q10_short = T.p.q10_devices < T.p.total_devices;   // node 0 has fewer GPUs than the average (Q10)
        const bool own_type = (T.p.corrected & METIS_FIX_Q6) != 0;
        x.sync();                                            // balance_run's last readers of capa/extra/mstate are done
#pragma unroll (X::kUniform ? 1 : 0)
        for (int s = x.lane(); s < S; s += x.width()) {
            const int g = w.gcode[s], tpc = w.tpc[s];
            const int a = (one_type && !q10_short) ? 0 : rank_start(s), b = a + (1 << g);
            double md = 0.001, err = 0.0;
            if (own_type) {                                  // opt-in METIS_FIX_Q6 (not the reference)
                const int rc = memory_demand_own_type(s, md);
                if (rc) err = (double)rc + (double)aux * 256.0;
            } else if (q10_short && b > T.p.q10_devices) {
                err = (double)METIS_FATAL_INDEX;             // device_types[rank]: IndexError (load_balancer.py:36, Q10)
            } else if (one_type || type_of_q10(T, pd.ns, a) == type_of_q10(T, pd.ns, b - 1)) {
                const int bs = bs_total >> (g - tpc);
                const int key = key_of(T, type0, tpc, bs);
                if (key < 0) err = (double)METIS_FATAL_KEY_MEMORY + (double)(((uint32_t)tpc << 16) | (uint32_t)bs) * 256.0;
                else md += range_sum<X>(T, kRangeMem, key, T.mem + (size_t)key * T.p.lpad, w.part[s], w.part[s + 1]) * kMemCoef;
            } else {
                const int rc = hetero_memory_demand(s, type0, md);
                if (rc) err = (double)rc + (double)aux * 256.0;
            }
            w.extra[s] = md;
            const double mc = one_type ? T.type_memory[0] * (double)(1 << g) : memory_capacity(rank_start(s), rank_start(s) + (1 << g));
            w.capa[s] = mc - md;
            w.mstate[s] = err;
            if (tap) { tap->demand[s] = md; tap->state[s] = mc - md; }
        }
        x.sync();
        x.converge();
        bool oom = false;
#pragma unroll (X::kUniform ? 1 : 0)
        for (int s = 0; s < S; ++s) {
            if (w.mstate[s] != 0.0) {
                const uint64_t code = (uint64_t)w.mstate[s];
                aux = (uint32_t)(code >> 8);
                return -(int)(code & 0xFF);
            }
            if (w.capa[s] < 0) oom = true;
        }
        if (!oom) {
            x.sync();
#pragma unroll (X::kUniform ? 1 : 0)
            for (int s = x.lane(); s < S; s += x.width()) w.mstate[s] = w.capa[s];
            x.sync();
            return 1;
        }
        if (attempt >= 3) return 0;
        x.mark(21);
        const int rc = adjust_performance();
        if (rc < 0) return rc;
        return rc == 1 ? 0 : 2;
    }

    // LayerLoadBalancer.partition_layer (model/load_balancer.py:121-144)
    // returns attempt number 1..3, 0 = (None, -1, None), <0 = fatal (negated code)
    template <class Sink>
    MB_HD_NOINLINE int partition_layer(Sink &sink) {
#pragma unroll (X::kUniform ? 1 : 0)
        for (int attempt = 1; attempt <= 3; ++attempt) {
            sink.balancer_run();
            const int rc = balance_run<MAXS, MAXL>(T, pd.S, w, x);
            if (rc) return -rc;
            const int r = memory_phase(attempt);
            if (r == 1) return attempt;
            if (r <= 0) return r;
        }
        return 0;
    }

    // bandwidth of a set of ranks given as node range / strided group (model/cluster_bandwidth.py:169-195)
    MB_HD double bw_of_node_range(int n0, int n1) const {
        const int per = T.p.devices_per_node;
        if (n0 == n1) return T.bw_first[type_of_q10(T, pd.ns, n0 * per)];
        double slow = INFINITY;
        const int nt = T.p.num_types;
        const int32_t *end = T.q10_end + pd.ns * nt;
        const uint8_t *typ = T.run_type + pd.ns * nt;
        int lo = 0;
#pragma unroll (X::kUniform ? 1 : 0)
        for (int k = 0; k < nt; ++k) {                       // types whose node run intersects [n0, n1]
            const int hi = end[k];
            if (hi > lo && n0 * per < hi && (n1 + 1) * per > lo) {
                const double v = T.bw_min[typ[k]];
                if (v < slow) slow = v;
            }
            lo = hi;
        }
        return slow;
    }

    MB_HD double dp_bandwidth(int a, int dp, int tp) const {
        const int per = T.p.devices_per_node;
        double slow = INFINITY;
#pragma unroll (X::kUniform ? 1 : 0)
        for (int d = 0; d < dp; ++d) {                       // group d = ranks a + d + i*dp (:148-156)
            const int n0 = (a + d) / per;
            int nlast = n0;
            bool multi = false;
            double gmin = INFINITY;
            int tprev = -1;
#pragma unroll (X::kUniform ? 1 : 0)
            for (int i = 0; i < tp; ++i) {
                const int node = (a + d + i * dp) / per;
                if (node != nlast) { multi = true; nlast = node; }
                const int t = type_of_q10(T, pd.ns, node * per);
                if (t != tprev) { const double v = T.bw_min[t]; if (v < gmin) gmin = v; tprev = t; }
            }
            const double bw = multi ? gmin : T.bw_first[type_of_q10(T, pd.ns, n0 * per)];
            if (bw < slow) slow = bw;
        }
        return slow;
    }

    // mixed-type stage of _get_execution_cost (model/cost_estimator.py:189-197 with :152-173)
    MB_HD_NOINLINE int hetero_exec_cost(int a, int b, int dp, int tpc, int la, int lb, double &len) {
        HSplit hs;
        uint32_t dummy;
        if (partition_data(T, pd.ns, a, b - a, dp, tpc, bs_total, hs, dummy)) return 1;
        len = -INFINITY;
#pragma unroll (X::kUniform ? 1 : 0)
        for (int r = 0; r < hs.nruns; ++r)
#pragma unroll (X::kUniform ? 1 : 0)
            for (int v = 0; v < 2; ++v) {
                const int cntv = v ? hs.plus[r] : hs.n[r] - hs.plus[r];
                const int h = hs.base[r] + v;
                if (cntv <= 0 || h == 0) continue;
                double acc = 0.;
#pragma unroll (X::kUniform ? 1 : 0)
                for (int bit = 30; bit >= 0; --bit) {
                    const int piece = 1 << bit;
                    if (!(h & piece)) continue;
                    if (piece > T.p.max_bs) return 1;            // :166-167
                    const int key = key_of(T, hs.type[r], tpc, piece);
                    if (key < 0) return 1;
                    acc += range_sum<X>(T, kRangeLc, key, T.lc + (size_t)key * T.p.lpad, la, lb);
                }
                if (acc > len) len = acc;
            }
        return 0;
    }

    // _get_fb_sync_cost over the device types of ranks [a, b) (model/cost_estimator.py:57-72, quirk Q9)
    MB_HD int fb_sync_cost(int a, int b, int tpc, int mbs, double &out) const {
        const int nt = T.p.num_types;
        const int32_t *end = T.run_end + pd.ns * nt;
        const uint8_t *typ = T.run_type + pd.ns * nt;
        double mx = -INFINITY;
        int lo = 0;
#pragma unroll (X::kUniform ? 1 : 0)
        for (int k = 0; k < nt; ++k) {
            const int hi = end[k];
            if ((a > lo ? a : lo) < (b < hi ? b : hi)) {
                const int key = key_of(T, typ[k], tpc, mbs);
                if (key < 0) return 1;
                const double v = T.fb_sync[key];
                if (v == 0.0) return 1;                       // falsy -> KeyError
                if (v > mx) mx = v;
            }
            lo = hi;
        }
        out = mx;
        return 0;
    }

    // HeteroCostEstimator.get_cost (model/cost_estimator.py:199-244); returns 0 ok, 1 KeyError.
    // x / tp is evaluated as x * 2^-log2(tp) (same real quotient, same rounding); the remaining
    // quotients come from the derived tables when the cluster has a single bandwidth value.
    MB_HD int get_cost(double &cost_out) {
        const int per = T.p.devices_per_node;
        const int Lm = T.p.num_layers;
        const bool one_type = ONE || T.p.num_types == 1;
        const bool ubw = T.p.uniform_bw != 0;
        const int nstage = pd.label < pd.S ? pd.label : pd.S;  // zip(range(plan.num_stage), strategies)
        // rank_node_map holds num_nodes * devices(node 0) ranks (cluster_bandwidth.py:34-47, Q10): a costed stage
        // (or its pipeline successor) beyond that raises KeyError -> the candidate is skipped
        if (T.p.q10_devices < T.p.total_devices && rank_start(nstage) > T.p.q10_devices) return 1;
        // execution time of every stage first (independent range sums; w.capa[s] = time, w.extra[s] = error flag)
        x.sync();
#pragma unroll (X::kUniform ? 1 : 0)
        for (int s = x.lane(); s < nstage; s += x.width()) {
            const int g = w.gcode[s], tpc = w.tpc[s];
            const int a = one_type ? 0 : rank_start(s), b = a + (1 << g);
            const int la = w.part[s], lb = w.part[s + 1];
            const int ldp = g - tpc;
            const int ta = one_type ? 0 : type_of_rank(T, pd.ns, a);
            const int tb = one_type ? 0 : type_of_rank(T, pd.ns, b - 1);
            double len = 0.0, err = 0.0;
            if (ta == tb) {                                   // _get_execution_cost :175-188
                const int key = key_of(T, ta, tpc, bs_total >> ldp);
                if (key < 0) err = 1.0;
                else len = range_sum<X>(T, kRangeLc, key, T.lc + (size_t)key * T.p.lpad, la, lb);
            } else if (hetero_exec_cost(a, b, 1 << ldp, tpc, la, lb, len)) {
                err = 1.0;
            }
            w.capa[s] = len;
            w.extra[s] = err;
        }
        x.sync();
        bool bad = false;
#pragma unroll (X::kUniform ? 1 : 0)
        for (int s = x.lane(); s < nstage; s += x.width()) bad = bad || (w.extra[s] != 0.0);
        if (x.any(bad)) return 1;                             // KeyError raised while costing a stage
        double *ppterm = reinterpret_cast<double *>(w.subw);  // free after the vote (MAXL >= MAXS)
        double max_len = -INFINITY, max_upd = -INFINITY, max_dp = -INFINITY;
#pragma unroll (X::kUniform ? 1 : 0)
        for (int s = x.lane(); s < nstage; s += x.width()) {  // independent per-stage terms
            const int g = w.gcode[s], tpc = w.tpc[s];
            const int la = w.part[s], lb = w.part[s + 1];
            const int ldp = g - tpc;
            const int mbs = bs_total >> ldp;
            const double inv_tp = pow2_neg(tpc);              // 1 / tp, exact power of two
            if (w.capa[s] > max_len) max_len = w.capa[s];
            double pp = 0.0;
            if (s < nstage - 1) {
                if (ubw) {                                    // :224-227 via the derived tables
                    pp = (lb == Lm - 1) ? T.pp_vocab[mbs * T.p.num_tp + tpc] : T.pp_hidden[mbs];
                } else {
                    double act;
                    if (lb == Lm - 1)
                        act = (double)((int64_t)mbs * T.p.sequence_length * T.p.vocab_size) * inv_tp;
                    else
                        act = (double)((int64_t)mbs * T.p.sequence_length * T.p.hidden_size);
                    const int a = rank_start(s), b2 = rank_start(s + 2);
                    pp = act / (bw_of_node_range(a / per, (b2 - 1) / per) * 1048576.0);
                }
            }
            ppterm[s] = pp;
            // get_parameter_size_by_stage (model/activation_parameter.py:40-51)
            int ntr = lb - la;
            double params = 0.0;
            if (la == 0) { params += T.p.input_params * inv_tp; --ntr; }
            if (lb == Lm) { params += T.p.output_params * inv_tp; --ntr; }
            params += T.p.transformer_params * inv_tp * (double)ntr;
            double dpc;                                       // :37-43
            if (ubw) dpc = T.dpk[ldp] * params;
            else {
                const int dp = 1 << ldp;
                dpc = (double)(2 * (dp - 1)) / ((double)dp * (dp_bandwidth(rank_start(s), dp, 1 << tpc) * 1048576.0)) * params;
            }
            if (dpc > max_dp) max_dp = dpc;
            const double upd = T.p.optimizer_time * inv_tp * T.ratio[lb - la];   // :145-147
            if (upd > max_upd) max_upd = upd;
        }
        max_len = x.max_all(max_len);
        max_upd = x.max_all(max_upd);
        max_dp = x.max_all(max_dp);
        x.sync();
        PySum lens_sum;                                       // order-dependent sums, stage order
        double pp_cost = 0., fb_sync = 0.;
#pragma unroll (X::kUniform ? 1 : 0)
        for (int s = 0; s < nstage; ++s) {
            lens_sum.add(w.capa[s]);
            if (s < nstage - 1) pp_cost += ppterm[s];
        }
        {
            const int s = nstage - 1;                         // _get_fb_sync_cost of the last costed stage
            const int a = one_type ? 0 : rank_start(s), b = a + group(s);
            double v;
            if (fb_sync_cost(a, b, w.tpc[s], bs_total >> (w.gcode[s] - w.tpc[s]), v)) return 1;
            fb_sync = v * (double)pd.batches;
        }
        const double exec = ((double)(pd.batches - 1) * max_len) + lens_sum.result();   // :235-236
        const double bg = T.p.batch_generator * (double)pd.batches;
        cost_out = exec + fb_sync + max_upd + max_dp + pp_cost + bg;                   // :241-242
        if (tap) { tap->cost[0] = exec; tap->cost[1] = fb_sync; tap->cost[2] = max_upd; tap->cost[3] = max_dp; tap->cost[4] = pp_cost; }
        return 0;
    }

    // cost_het_cluster.py:31-48 for one inter-stage plan, with IntraStagePlanGenerator.has_next
    // (search_space/plan.py:192-226) inlined.  `only_step` >= 0 stops after emitting that step.
    // Sequential form (replay kernel and tests); the search kernel uses search_loop below.
    template <class Sink>
    MB_HD_NOINLINE void run(const PlanDesc &plan, Sink &sink, int only_step = -1) {
        const int ok = begin(plan);
        if (ok < 0) { sink.fatal(plan.ordinal, METIS_FATAL_SCRATCH, 0); return; }
        if (ok == 0) return;
        bool started = false, have_state = false;
        int nrep = 0, step = 0;
#pragma unroll (X::kUniform ? 1 : 0)
        for (;;) {
            if (nrep == 1) return;                            // plan.py:194-195
            int attempt = 0;
#pragma unroll (X::kUniform ? 1 : 0)
            for (;;) {
                if (!started) started = true;                 // first strategy that can be valid (see begin)
                else if (!next_strategy(have_state)) return;  // :203-204
                if (!valid()) continue;
                sink.partition_call();
                int rc = compute_performance();
                if (rc) { sink.fatal(pd.ordinal, rc, aux); return; }
                attempt = partition_layer(sink);
                if (attempt < 0) { sink.fatal(pd.ordinal, -attempt, aux); return; }
                have_state = attempt > 0;                     // memory_state is None after a failure (:225)
                if (attempt > 0) break;
            }
            nrep = attempt;
            double cost;
            if (get_cost(cost) == 0) sink.emit(pd, step, nrep, cost, w.tpc, w.part);
            else sink.keyerror();
            if (only_step >= 0 && step == only_step) return;
            ++step;
        }
    }
};

// ---------------------------------------------------------------------------
// First task of a plan, one plan per thread (the bulk round of the search, metis_search.cu).
//
// The work per inter-stage plan is heavy-tailed: most plans need exactly one LayerComputeBalancer
// run (their first strategy is partitioned at the first attempt, which also ends the chain,
// plan.py:194-195); a few per cent need 10-36 *sequential* runs.  The first attempt of the first
// strategy of every admitted plan is therefore evaluated with 32 plans per warp in lockstep; a
// plan whose first attempt runs out of memory is handed to the chain kernel (one warp per plan,
// metis_coop.cuh), which walks the rest of the chain: from attempt 2 with the re-weighted stage
// performance left in w.perf (`resume` = CoopEvaluator::kRetry), or from the next strategy when the
// reference finds no re-weighting (kAdvance).
// returns true when the plan continues in the chain kernel; `chain_hint` then estimates how long its chain is
// (PlanEvaluator::halvings; used only to start long chains first).
// ---------------------------------------------------------------------------
template <int MAXS, int MAXL, bool ONE, class X = Serial, class Sink>
MB_HD bool first_task(const Tables &T, Scratch<MAXS, MAXL> &w, Sink &sink, bool has, const PlanDesc &plan, int &chain_hint,
                      int &resume) {
    // X = Lockstep (device, called by all 32 lanes of a warp, with or without a plan): the lanes are re-joined
    // between the phases and inside the balancer.  X = Serial: one thread on its own.
    PlanEvaluator<MAXS, MAXL, X, ONE> ev(T, w);
    bool cont = false;
    sink.phase(1);
    if (has) {                                               // ---- P ----
        const int ok = ev.begin(plan);
        if (ok < 0) sink.fatal(plan.ordinal, METIS_FATAL_SCRATCH, 0);
        has = ok == 1;
    }
    ev.x.rejoin(has);
    if (has) {
        sink.partition_call();
        const int rc = ev.compute_performance();
        if (rc) { sink.fatal(plan.ordinal, rc, ev.aux); has = false; }
    }
    sink.phase(2);
    ev.x.rejoin(has);
    if (has) {                                               // ---- R ----
        sink.balancer_run();
        const int rc = balance_run<MAXS, MAXL>(T, plan.S, w, ev.x);
        if (rc) { sink.fatal(plan.ordinal, rc, ev.aux); has = false; }
    }
    sink.phase(3);
    ev.x.rejoin(has);
    bool costing = false;
    if (has) {                                               // ---- M ----
        const int r = ev.memory_phase(1);
        if (r < 0) sink.fatal(plan.ordinal, -r, ev.aux);
        else if (r != 1) {                                   // out of memory: the rest in the chain kernel
            cont = true;
            chain_hint = ev.halvings();
            resume = r == 2 ? 2 : 3;                         // CoopEvaluator::kRetry (w.perf re-weighted) : kAdvance
        } else costing = true;                               // partition accepted at the first attempt
    }
    sink.phase(4);
    ev.x.rejoin(costing);
    if (costing) {                                           // ---- C ---- (num_repartition == 1 ends the chain)
        double cost;
        if (ev.get_cost(cost) == 0) sink.emit(plan, 0, 1, cost, w.tpc, w.part);
        else sink.keyerror();
    }
    sink.phase(0);
    ev.x.rejoin(true);
    return cont;
}

// ---------------------------------------------------------------------------
// HomoCostEstimator.get_cost (model/cost_estimator.py:98-138) for one UniformPlan.
// returns 0 ok, 1 KeyError; *oom = _detect_oom_occurrence
// ---------------------------------------------------------------------------
MB_HD int homo_cost(const Tables &T, int type, int dp, int pp, int tp, int mbs, int gbs, double &cost_out,
                    int &oom) {
    const int L = T.p.num_layers;
    const int per = T.p.devices_per_node;
    int tpc = 0;
#pragma unroll 1
    while ((1 << tpc) < tp) ++tpc;
    const int key = ((1 << tpc) == tp) ? key_of(T, type, tpc, mbs) : -1;   // unprofiled tp -> KeyError (:93-94)
    if (key < 0) return 1;
    const int num_mbs = gbs / mbs / dp;
    (void)type;
    const double intra = T.p.node0_bandwidth;                                // cluster_bandwidth.py:75-76
    const double inter = T.p.node0_bandwidth;                                // quirk Q2: same field
    const int base = (L - 2) / pp, rem = (L - 2) % pp;                       // model/utils.py:5-31
    PySum lens_sum;
    double max_len = -INFINITY, max_params = -INFINITY, max_mem = -INFINITY;
    double pp_cost = 0., fb_sync = 0.;
    int a = 0;
#pragma unroll 1
    for (int s = 0; s < pp; ++s) {
        int count = base + ((s >= 1 && s <= rem) ? 1 : 0) + (s == 0 ? 1 : 0) + (s == pp - 1 ? 1 : 0);
        const int b = a + count;
        const double len = py_sum_range(T.lc + (size_t)key * T.p.lpad, a, b);
        lens_sum.add(len);
        if (len > max_len) max_len = len;
        // sum(model_parameters[a:b]) over get_parameter_size(tp) (model/activation_parameter.py:34-38)
        PySum ps;
#pragma unroll 1
        for (int r = a; r < b && r < L; ++r) {
            const double v = (r == 0) ? T.p.input_params / (double)tp
                           : (r == L - 1) ? T.p.output_params / (double)tp
                           : T.p.transformer_params / (double)tp;
            ps.add(v);
        }
        const double sp = ps.result();
        if (sp > max_params) max_params = sp;
        const double sm = py_sum_range(T.mem + (size_t)key * T.p.lpad, a, b);
        if (sm > max_mem) max_mem = sm;
        if (s == pp - 1) {
            const double v = T.fb_sync[key];
            if (v == 0.0) return 1;
            fb_sync = v * (double)num_mbs;
        } else {
            double act;
            if (b == L - 1) act = (double)((int64_t)mbs * T.p.sequence_length * T.p.vocab_size) / (double)tp;
            else act = (double)((int64_t)mbs * T.p.sequence_length * T.p.hidden_size);
            double bw = intra;                                // cluster_bandwidth.py:111-123
#pragma unroll 1
            for (int d = 0; d < dp; ++d)
#pragma unroll 1
                for (int t = 0; t < tp; ++t) {
                    const int r0 = s * dp * tp + d * tp + t, r1 = r0 + dp * tp;
                    if (r0 / per != r1 / per) bw = inter;
                }
            pp_cost += act / (bw * 1048576.0);
        }
        a = b;
    }
    oom = (T.p.node0_memory < max_mem) ? 1 : 0;              // cost_estimator.py:31-32
    const double exec = ((double)(num_mbs - 1) * max_len) + lens_sum.result();
    const double upd = T.p.optimizer_time / (double)pp / (double)tp;
    double bw = intra;                                        // :125-132
#pragma unroll 1
    for (int p = 0; p < pp; ++p)
        if ((p * dp * tp) / per != ((p + 1) * dp * tp - 1) / per) bw = inter;
    const double dpc = (double)(2 * (dp - 1)) / ((double)dp * (bw * 1048576.0)) * max_params;
    const double bg = T.p.batch_generator * (double)num_mbs;
    cost_out = exec + fb_sync + upd + dpc + pp_cost + bg;
    return 0;
}

}  // namespace metis
