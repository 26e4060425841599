// metis_blob.cuh - the packed problem tables and the ordinal -> plan decoding, shared by the kernels of
// metis_search.cu and metis_recost.cu.
//
// pack_tables_kernel (metis_search.cu) flattens the profile tables of a MetisProblem into one 16 B-aligned blob laid out
// by make_layout; a kernel binds its Tables to that blob with make_tables.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "metis_eval.cuh"

namespace metis {

struct BlobLayout {
    uint32_t total;               // bytes staged into shared memory
    uint32_t key, lc, mem, exec_full, fb, norm, derived, tmem, bwf, bwm, runt, rune, q10e;
    uint32_t rsum, rsum_bytes;    // range-sum tables (Tables::rsum): behind the staged part, read from L2
};

static inline uint32_t align16(uint32_t v) { return (v + 15u) & ~15u; }

static inline BlobLayout make_layout(const MetisProblem &p) {
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

// `base`: the staged tables (a plain pointer to global memory, or the shared-memory address of the staged copy);
// `gblob`: the blob in global memory when its range-sum tables were filled for this launch (search kernels), else
// nullptr
template <class Space>
__device__ __forceinline__ TablesOf<Space> bind_tables(const MetisProblem &p, const BlobLayout &l,
                                                       typename Space::template ptr<uint8_t> base, const uint8_t *gblob) {
    TablesOf<Space> T;
    T.p = p;
    T.rsum = gblob ? reinterpret_cast<const double *>(gblob + l.rsum) : nullptr;
    T.key_index = tab_cast<int16_t>(base + l.key);
    T.lc = tab_cast<double>(base + l.lc);
    T.mem = tab_cast<double>(base + l.mem);
    T.exec_full = tab_cast<double>(base + l.exec_full);
    T.fb_sync = tab_cast<double>(base + l.fb);
    T.norm_lc = tab_cast<double>(base + l.norm);
    bind_derived(T, tab_cast<double>(base + l.derived));
    T.type_memory = tab_cast<double>(base + l.tmem);
    T.bw_first = tab_cast<double>(base + l.bwf);
    T.bw_min = tab_cast<double>(base + l.bwm);
    T.run_type = base + l.runt;
    T.run_end = tab_cast<int32_t>(base + l.rune);
    T.q10_end = tab_cast<int32_t>(base + l.q10e);
    return T;
}

__device__ __forceinline__ Tables make_tables(const MetisProblem &p, const BlobLayout &l, const uint8_t *base,
                                              const uint8_t *gblob = nullptr) {
    return bind_tables<GenericSpace>(p, l, base, gblob);
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

// Packs the tables of `problem` into `workspace` on `stream` for a replay kernel (one thread per plan, tables read from
// global memory), after the checks of metis_het_detail: returns METIS_OK with the blob's layout and address, or the
// error code (METIS_E_ARG, METIS_E_CAPACITY, METIS_E_CUDA).  Defined in metis_search.cu.
int stage_replay_tables(const MetisProblem *problem, void *workspace, int64_t workspace_bytes, cudaStream_t stream,
                        BlobLayout &lay, const uint8_t *&blob);

// The workspace bytes stage_replay_tables needs for `problem`, or METIS_E_ARG.  Defined in metis_search.cu.
int64_t replay_tables_bytes(const MetisProblem *problem);

// One scenario's packed tables, what make_tables needs (the profile what-ifs, metis_profile.cu and metis_noise.cu)
struct ScenarioTables {
    MetisProblem p;
    BlobLayout lay;
    const uint8_t *blob;
};

// Packs the tables of problems[0 .. K) (stage_replay_tables), problem j's at `blobs` + the sum of
// align256(replay_tables_bytes(problems[i])) for i < j, then writes their K descriptors to `desc` with one
// host-to-device copy.  Returns METIS_OK or stage_replay_tables' error code; launch and copy errors are left for
// cudaGetLastError.  Defined in metis_profile.cu.
int stage_scenarios(const MetisProblem *problems, int K, ScenarioTables *desc, uint8_t *blobs, cudaStream_t stream);

// What het_profile_kernel stores for candidate i of n under scenario j: `unknown` for a record that is no plan of the
// space, else `store` with profile_candidate's cost, headroom and status (metis_recost.cuh).
struct ProfileOut {                   // metis_het_profile_recost: all three, at j * n + i
    double *cost, *headroom;
    uint8_t *status;
    __device__ void unknown(int j, long long i, long long n) const {
        const size_t at = (size_t)j * n + i;
        cost[at] = headroom[at] = (double)NAN;
        status[at] = (uint8_t)(METIS_FATAL_SCRATCH | METIS_FATAL_SCRATCH << 4);
    }
    __device__ void store(int j, long long i, long long n, double c, double h, uint8_t st) const {
        const size_t at = (size_t)j * n + i;
        cost[at] = c;
        headroom[at] = h;
        status[at] = st;
    }
};

struct NoiseOut {                     // metis_het_profile_noise_eval: cost and the usable byte, at j * ld + i
    double *cost;
    uint8_t *usable;
    long long ld;
    __device__ void unknown(int j, long long i, long long) const {
        const size_t at = (size_t)j * ld + i;
        cost[at] = (double)NAN;
        usable[at] = 0;
    }
    __device__ void store(int j, long long i, long long, double c, double h, uint8_t st) const {
        const size_t at = (size_t)j * ld + i;
        cost[at] = c;
        usable[at] = st == 0 && h >= 0.0 ? 1 : 0;
    }
};

// Launches het_profile_kernel (metis_profile.cu) on `stream` when n > 0: one thread per record of records[0 .. n)
// (detail row at detail + i * stride), the block walking the K scenarios of `scen` in step.  Launch errors are left
// for cudaGetLastError.
template <class Out>
void launch_profile_kernel(const MetisPlanSpace &sp, const ScenarioTables *scen, int K, const MetisRecord *records,
                           int64_t n, const uint8_t *detail, int stride, const Out &out, cudaStream_t stream);

}  // namespace metis
