// Profile-noise what-if of a finished search (include/metis_b200.h, metis_het_profile_noise_*).
//
//   key_meta_kernel          each profile key's device type, log2(tp) and bs, from key_index: the Philox counter of a
//                            value names its key by these
//   noise_rows_kernel        one thread per (sample, key, layer): the sample's layer_compute and layer_memory entries
//   noise_keys_kernel        one thread per (sample, key): exec_full (the sum of the sample's layer_compute row) and
//                            fb_sync.  Every other table of a sample is the base problem's, norm_lc included (only the
//                            balancer reads it, and no balancer runs here).  All samples share the base key set, num_bs
//                            and lpad, so one BlobLayout; stage_scenarios (metis_profile.cu) packs each sample's
//                            tables and writes their descriptors.
//   het_profile_kernel       metis_profile.cu's kernel of the profile what-if, launched with NoiseOut: cost and the
//                            usable byte of every (sample, candidate)
//   noise_min / noise_first  per sample, the lowest cost_order_key of a usable candidate, then the lowest position that
//                            holds it (group_min_kernel / group_first_kernel's two passes, with a warp's minimum taken
//                            before its one atomicMin)
//   noise_accumulate_kernel  one thread per candidate, the chunk's samples in order: noise_accumulate (metis_noise.cuh)
//
// Search what-if (metis_het_search_noise_*): the same draw, each sample's norm_lc included, for a fresh search per sample.
//   noise_norm_kernel        one thread per sample: noisy_norm (metis_noise.cuh) of the profile's first-listed tp1_bs1
//                            row, the base's norm_lc when its sigma is 0 or when the noisy total is 0 (then flagged)
#include <cuda_runtime.h>

#include <cmath>
#include <cstdint>
#include <vector>

#include "../../include/metis_b200.h"
#include "metis_blob.cuh"
#include "metis_internal.h"
#include "metis_noise.cuh"
#include "metis_query.cuh"

namespace metis {

constexpr int kReduceThreads = 256;
constexpr int kMaxSamples = 65535;

// Where a chunk's pieces sit in the workspace (from its 256-aligned start).  A sample's arrays are its layer_compute,
// layer_memory, exec_full and fb_sync, then, with `norm_len` > 0 (the search what-if), its norm_lc.
struct NoiseLayout {
    int64_t desc, meta, arrays, array_stride, replay, replay_stride, total;
};

static NoiseLayout noise_layout(const MetisProblem &b, int count, int64_t replay_bytes, int norm_len = 0) {
    NoiseLayout l;
    const int64_t K = b.num_keys, row = (int64_t)b.num_keys * b.lpad;
    l.desc = 0;
    l.meta = align256((int64_t)count * (int64_t)sizeof(ScenarioTables));
    l.arrays = l.meta + align256(K * 4);
    l.array_stride = align256((2 * row + 2 * K + norm_len) * (int64_t)sizeof(double));
    l.replay = l.arrays + (int64_t)count * l.array_stride;
    l.replay_stride = align256(replay_bytes);
    l.total = l.replay + (int64_t)count * l.replay_stride + 256;
    return l;
}

__global__ void key_meta_kernel(const __grid_constant__ MetisProblem b, uint32_t *meta) {
    const int per_type = b.num_tp * b.num_bs;
    const int e = blockIdx.x * kReduceThreads + threadIdx.x;
    if (e >= b.num_types * per_type) return;
    const int k = b.key_index[e];
    if (k < 0) return;
    const int ti = e / per_type, r = e % per_type;
    meta[k] = pack_key_meta(ti, r / b.num_bs, r % b.num_bs + 1);
}

__global__ void __launch_bounds__(kReduceThreads)
noise_rows_kernel(const __grid_constant__ MetisProblem b, const __grid_constant__ MetisNoiseSpec spec,
                  const uint32_t *__restrict__ meta, uint8_t *arrays, long long array_stride) {
    const long long row = (long long)b.num_keys * b.lpad;
    const long long e = (long long)blockIdx.x * kReduceThreads + threadIdx.x;
    if (e >= row) return;
    const int s = blockIdx.y;
    const uint32_t j = (uint32_t)(spec.first + s);
    double *lc = reinterpret_cast<double *>(arrays + s * array_stride), *lm = lc + row;
    const uint32_t m = meta[e / b.lpad], l = (uint32_t)(e % b.lpad);
    lc[e] = noisy_value(b.layer_compute[e], spec.sigma[0], spec.type_code, spec.seed, j, m, kNoiseCompute, l);
    lm[e] = noisy_value(b.layer_memory[e], spec.sigma[1], spec.type_code, spec.seed, j, m, kNoiseMemory, l);
}

__global__ void __launch_bounds__(kReduceThreads)
noise_keys_kernel(const __grid_constant__ MetisProblem b, const __grid_constant__ MetisNoiseSpec spec,
                  const uint32_t *__restrict__ meta, uint8_t *arrays, long long array_stride) {
    const int k = blockIdx.x * kReduceThreads + threadIdx.x;
    if (k >= b.num_keys) return;
    const int s = blockIdx.y;
    const long long row = (long long)b.num_keys * b.lpad;
    double *lc = reinterpret_cast<double *>(arrays + s * array_stride), *ef = lc + 2 * row, *fb = ef + b.num_keys;
    const uint32_t m = meta[k];
    ef[k] = spec.sigma[0][m & 0xff] == 0.0 ? b.exec_full[k] : noisy_exec_full(lc + (long long)k * b.lpad, b.lpad);
    fb[k] = noisy_value(b.fb_sync[k], spec.sigma[2], spec.type_code, spec.seed, (uint32_t)(spec.first + s), m,
                        kNoiseFbSync, 0);
}

__global__ void __launch_bounds__(kReduceThreads)
noise_norm_kernel(const __grid_constant__ MetisProblem b, const __grid_constant__ MetisNoiseSpec spec,
                  const __grid_constant__ MetisNormSource src, uint8_t *arrays, long long array_stride,
                  long long norm_at, uint8_t *zero) {
    const int s = blockIdx.x * kReduceThreads + threadIdx.x;
    if (s >= spec.count) return;
    double *out = reinterpret_cast<double *>(arrays + s * array_stride + norm_at);
    const bool drawn = src.sigma != 0.0 &&
                       noisy_norm(src.row, src.len, src.sigma, spec.seed, (uint32_t)(spec.first + s), src.type_code, out);
    if (!drawn)
        for (int i = 0; i < b.norm_len; ++i) out[i] = b.norm_lc[i];
    zero[s] = src.sigma != 0.0 && !drawn;
}

__device__ __forceinline__ unsigned long long warp_min(unsigned long long v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long u = __shfl_xor_sync(0xffffffffu, v, o);
        v = u < v ? u : v;
    }
    return v;
}

__global__ void noise_best_init_kernel(int count, unsigned long long *key, unsigned long long *first) {
    const int s = blockIdx.x * kReduceThreads + threadIdx.x;
    if (s >= count) return;
    key[s] = ~0ULL;
    first[s] = ~0ULL;
}

// grid (x: blocks striding over the candidates, y: sample)
__global__ void __launch_bounds__(kReduceThreads)
noise_min_kernel(const double *__restrict__ cost, const uint8_t *__restrict__ usable, long long n,
                 unsigned long long *key) {
    const size_t row = (size_t)blockIdx.y * n;
    unsigned long long m = ~0ULL;
    for (long long i = (long long)blockIdx.x * kReduceThreads + threadIdx.x; i < n;
         i += (long long)gridDim.x * kReduceThreads)
        if (usable[row + i]) {
            const unsigned long long k = cost_order_key(cost[row + i]);
            m = k < m ? k : m;
        }
    m = warp_min(m);
    if ((threadIdx.x & 31) == 0 && m != ~0ULL) atomicMin(&key[blockIdx.y], m);
}

__global__ void __launch_bounds__(kReduceThreads)
noise_first_kernel(const double *__restrict__ cost, const uint8_t *__restrict__ usable, long long n,
                   const unsigned long long *__restrict__ key, unsigned long long *first) {
    const size_t row = (size_t)blockIdx.y * n;
    const unsigned long long want = key[blockIdx.y];
    unsigned long long m = ~0ULL;
    for (long long i = (long long)blockIdx.x * kReduceThreads + threadIdx.x; i < n;
         i += (long long)gridDim.x * kReduceThreads)
        if (usable[row + i] && cost_order_key(cost[row + i]) == want) {
            m = (unsigned long long)i;
            break;                                            // later i of this thread are larger
        }
    m = warp_min(m);
    if ((threadIdx.x & 31) == 0 && m != ~0ULL) atomicMin(&first[blockIdx.y], m);
}

// the position's own cost (not the key's image, which folds -0.0 into +0.0); -1 / NaN for a sample with no usable
// candidate
__global__ void noise_best_finish_kernel(int count, const double *__restrict__ cost, long long n,
                                         unsigned long long *key, unsigned long long *first) {
    const int s = blockIdx.x * kReduceThreads + threadIdx.x;
    if (s >= count) return;
    const unsigned long long f = first[s];
    reinterpret_cast<double *>(key)[s] = f == ~0ULL ? (double)NAN : cost[(size_t)s * n + f];
}

__global__ void __launch_bounds__(kReduceThreads)
noise_accumulate_kernel(int count, double t, const double *__restrict__ cost, const uint8_t *__restrict__ usable,
                        long long n, const long long *__restrict__ best_pos, const double *__restrict__ best_cost,
                        int32_t *wins, int32_t *near, int32_t *usable_count, double *regret, double *sum) {
    const long long i = (long long)blockIdx.x * kReduceThreads + threadIdx.x;
    if (i >= n) return;
    int32_t w = wins[i], nr = near[i], u = usable_count[i];
    double r = regret[i], sm = sum[i];
    for (int s = 0; s < count; ++s) {
        const size_t at = (size_t)s * n + i;
        noise_accumulate(usable[at] != 0, cost[at], best_pos[s] == i, best_cost[s], t, w, nr, u, r, sm);
    }
    wins[i] = w;
    near[i] = nr;
    usable_count[i] = u;
    regret[i] = r;
    sum[i] = sm;
}

static unsigned blocks_of(long long n, int threads) { return (unsigned)((n + threads - 1) / threads); }

static const char *check_spec(const MetisNoiseSpec *spec, int num_types) {
    if (spec->count < 1 || spec->count > kMaxSamples || spec->first < 0 || spec->first > kMaxSamples - spec->count)
        return "samples out of range (1 <= count, first + count <= 65535)";
    for (int f = 0; f < 3; ++f)
        for (int t = 0; t < METIS_MAX_TYPES; ++t) {
            const double s = spec->sigma[f][t];
            if (!(s >= 0.0 && s < 1.0)) return "sigma must be finite and in [0, 1)";
        }
    for (int t = 0; t < num_types; ++t)
        if (spec->type_code[t] < 1 || spec->type_code[t] > 6) return "type_code out of range (1 .. 6)";
    if (!std::isfinite(spec->near_factor) || !(spec->near_factor >= 1.0)) return "near_factor must be finite and >= 1";
    return nullptr;
}

// Sample s of a chunk drawn into `ws` (layout `lay`): `base` with its drawn tables, norm_lc too when `own_norm`
static MetisProblem sample_problem(const MetisProblem &base, const NoiseLayout &lay, const uint8_t *ws, int s,
                                   bool own_norm) {
    MetisProblem p = base;
    const int64_t row = (int64_t)base.num_keys * base.lpad;
    const double *lc = reinterpret_cast<const double *>(ws + lay.arrays + (int64_t)s * lay.array_stride);
    p.layer_compute = lc;
    p.layer_memory = lc + row;
    p.exec_full = lc + 2 * row;
    p.fb_sync = lc + 2 * row + base.num_keys;
    if (own_norm) p.norm_lc = lc + 2 * row + 2 * base.num_keys;
    return p;
}

// The chunk's layer_compute, layer_memory, exec_full and fb_sync from the base's, then every sample's tables packed
// and their descriptors written (stage_scenarios).  A search what-if has launched noise_norm_kernel before.
static int draw_chunk(const MetisProblem &base, const MetisNoiseSpec &spec, const NoiseLayout &lay, uint8_t *ws,
                      bool own_norm, cudaStream_t stream) {
    uint32_t *meta = reinterpret_cast<uint32_t *>(ws + lay.meta);
    uint8_t *arrays = ws + lay.arrays;
    const int count = spec.count;
    key_meta_kernel<<<blocks_of((long long)base.num_types * base.num_tp * base.num_bs, kReduceThreads),
                      kReduceThreads, 0, stream>>>(base, meta);
    const long long row = (long long)base.num_keys * base.lpad;
    noise_rows_kernel<<<dim3(blocks_of(row, kReduceThreads), count), kReduceThreads, 0, stream>>>(
        base, spec, meta, arrays, lay.array_stride);
    noise_keys_kernel<<<dim3(blocks_of(base.num_keys, kReduceThreads), count), kReduceThreads, 0, stream>>>(
        base, spec, meta, arrays, lay.array_stride);
    std::vector<MetisProblem> samples((size_t)count);
    for (int s = 0; s < count; ++s) samples[(size_t)s] = sample_problem(base, lay, ws, s, own_norm);
    return stage_scenarios(samples.data(), count, reinterpret_cast<ScenarioTables *>(ws + lay.desc), ws + lay.replay,
                           stream);
}

// The layout of a search what-if chunk, or why it cannot be drawn
static const char *search_noise_layout(const MetisProblem *base, const MetisNoiseSpec *spec, NoiseLayout &lay,
                                       int &rc) {
    rc = METIS_E_ARG;
    if (base->num_types < 1 || base->num_types > METIS_MAX_TYPES) return "num_types out of range";
    if (const char *why = check_spec(spec, base->num_types)) return why;
    const int64_t replay = replay_tables_bytes(base);
    if (replay < 0) {
        rc = (int)replay;
        return "bad base problem";
    }
    lay = noise_layout(*base, spec->count, replay, base->norm_len);
    rc = METIS_OK;
    return nullptr;
}

}  // namespace metis

using namespace metis;

extern "C" {

int64_t metis_het_profile_noise_workspace_bytes(const MetisProblem *base, int32_t count) {
    if (!base || count < 1 || count > kMaxSamples) return METIS_E_ARG;
    const int64_t b = replay_tables_bytes(base);
    if (b < 0) return b;
    return noise_layout(*base, count, b).total;
}

int metis_het_profile_noise_draw(const MetisProblem *base, const MetisNoiseSpec *spec, void *workspace,
                                 int64_t workspace_bytes, void *stream_) {
    if (!base || !spec || !workspace) return fail_arg("metis_het_profile_noise_draw: NULL argument");
    if (base->num_types < 1 || base->num_types > METIS_MAX_TYPES)
        return fail_arg("metis_het_profile_noise_draw: num_types out of range");
    if (const char *why = check_spec(spec, base->num_types)) return fail_arg(why);
    const int64_t replay = replay_tables_bytes(base);
    if (replay < 0) return (int)replay;
    const NoiseLayout lay = noise_layout(*base, spec->count, replay);
    if (workspace_bytes < lay.total) return METIS_E_CAPACITY;
    const int rc = draw_chunk(*base, *spec, lay, align_workspace(workspace), false, static_cast<cudaStream_t>(stream_));
    if (rc) return rc;
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? METIS_OK : fail_cuda(e, "metis_het_profile_noise_draw");
}

int64_t metis_het_search_noise_workspace_bytes(const MetisProblem *base, int32_t count) {
    if (!base || count < 1 || count > kMaxSamples) return METIS_E_ARG;
    const int64_t b = replay_tables_bytes(base);
    if (b < 0) return b;
    return noise_layout(*base, count, b, base->norm_len).total;
}

int metis_het_search_noise_draw(const MetisProblem *base, const MetisNoiseSpec *spec, const MetisNormSource *norm,
                                void *workspace, int64_t workspace_bytes, uint8_t *norm_zero, void *stream_) {
    if (!base || !spec || !norm || !norm->row || !workspace || !norm_zero)
        return fail_arg("metis_het_search_noise_draw: NULL argument");
    NoiseLayout lay;
    int rc;
    if (const char *why = search_noise_layout(base, spec, lay, rc)) return rc == METIS_E_ARG ? fail_arg(why) : rc;
    if (norm->len != base->norm_len) return fail_arg("metis_het_search_noise_draw: norm->len != base->norm_len");
    if (norm->type_code < 1 || norm->type_code > 6)
        return fail_arg("metis_het_search_noise_draw: norm->type_code out of range (1 .. 6)");
    if (!(norm->sigma >= 0.0 && norm->sigma < 1.0))
        return fail_arg("metis_het_search_noise_draw: norm->sigma must be finite and in [0, 1)");
    if (workspace_bytes < lay.total) return METIS_E_CAPACITY;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    uint8_t *ws = align_workspace(workspace);
    const long long norm_at = (2LL * base->num_keys * base->lpad + 2LL * base->num_keys) * (long long)sizeof(double);
    noise_norm_kernel<<<blocks_of(spec->count, kReduceThreads), kReduceThreads, 0, stream>>>(
        *base, *spec, *norm, ws + lay.arrays, lay.array_stride, norm_at, norm_zero);
    rc = draw_chunk(*base, *spec, lay, ws, true, stream);
    if (rc) return rc;
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? METIS_OK : fail_cuda(e, "metis_het_search_noise_draw");
}

int metis_het_search_noise_problem(const MetisProblem *base, const MetisNoiseSpec *spec, int32_t s,
                                   const void *workspace, MetisProblem *sample) {
    if (!base || !spec || !workspace || !sample) return fail_arg("metis_het_search_noise_problem: NULL argument");
    NoiseLayout lay;
    int rc;
    if (const char *why = search_noise_layout(base, spec, lay, rc)) return rc == METIS_E_ARG ? fail_arg(why) : rc;
    if (s < 0 || s >= spec->count) return fail_arg("metis_het_search_noise_problem: sample out of range (0 .. count-1)");
    *sample = sample_problem(*base, lay, align_workspace(const_cast<void *>(workspace)), s, true);
    return METIS_OK;
}

int metis_het_profile_noise_eval(const MetisPlanSpace *space, const MetisNoiseSpec *spec, const void *workspace,
                                 const MetisRecord *records, int64_t n, const uint8_t *detail, int32_t detail_stride,
                                 double *cost, uint8_t *usable, int64_t ld, void *stream_) {
    if (!space || !spec || !workspace || (n > 0 && (!records || !detail || !cost || !usable)))
        return fail_arg("metis_het_profile_noise_eval: NULL argument");
    if (n < 0) return fail_arg("metis_het_profile_noise_eval: negative number of records");
    if (ld < n) return fail_arg("metis_het_profile_noise_eval: ld < n");
    if (spec->count < 1 || spec->count > kMaxSamples)
        return fail_arg("metis_het_profile_noise_eval: count out of range (1 .. 65535)");
    if (detail_stride < 3 * space->max_stage + 1)
        return fail_arg("metis_het_profile_noise_eval: detail_stride too small (3 * max_stage + 1)");
    const ScenarioTables *desc = reinterpret_cast<const ScenarioTables *>(align_workspace(const_cast<void *>(workspace)));
    launch_profile_kernel(*space, desc, spec->count, records, n, detail, detail_stride, NoiseOut{cost, usable, ld},
                          static_cast<cudaStream_t>(stream_));
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? METIS_OK : fail_cuda(e, "het_profile_kernel");
}

int metis_het_profile_noise_reduce(const MetisNoiseSpec *spec, const double *cost, const uint8_t *usable, int64_t n,
                                   int64_t *best_pos, double *best_cost, int32_t *wins, int32_t *near,
                                   int32_t *usable_count, double *regret, double *sum, void *stream_) {
    if (!spec || !best_pos || !best_cost ||
        (n > 0 && (!cost || !usable || !wins || !near || !usable_count || !regret || !sum)))
        return fail_arg("metis_het_profile_noise_reduce: NULL argument");
    if (n < 0) return fail_arg("metis_het_profile_noise_reduce: negative number of records");
    if (spec->count < 1 || spec->count > kMaxSamples)
        return fail_arg("metis_het_profile_noise_reduce: count out of range (1 .. 65535)");
    if (!std::isfinite(spec->near_factor) || !(spec->near_factor >= 1.0))
        return fail_arg("metis_het_profile_noise_reduce: near_factor must be finite and >= 1");
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    const int count = spec->count;
    auto *key = reinterpret_cast<unsigned long long *>(best_cost);
    auto *first = reinterpret_cast<unsigned long long *>(best_pos);
    noise_best_init_kernel<<<blocks_of(count, kReduceThreads), kReduceThreads, 0, stream>>>(count, key, first);
    if (n > 0) {
        const unsigned bx = blocks_of(n, kReduceThreads) < 64 ? blocks_of(n, kReduceThreads) : 64;
        noise_min_kernel<<<dim3(bx, count), kReduceThreads, 0, stream>>>(cost, usable, n, key);
        noise_first_kernel<<<dim3(bx, count), kReduceThreads, 0, stream>>>(cost, usable, n, key, first);
    }
    noise_best_finish_kernel<<<blocks_of(count, kReduceThreads), kReduceThreads, 0, stream>>>(count, cost, n, key,
                                                                                             first);
    if (n > 0)
        noise_accumulate_kernel<<<blocks_of(n, kReduceThreads), kReduceThreads, 0, stream>>>(
            count, spec->near_factor, cost, usable, n, reinterpret_cast<const long long *>(best_pos), best_cost, wins,
            near, usable_count, regret, sum);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? METIS_OK : fail_cuda(e, "profile noise reduction kernels");
}

}  // extern "C"
