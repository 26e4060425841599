// Profile what-ifs of a finished search (include/metis_b200.h, metis_het_profile_recost; metis_noise.cu's
// metis_het_profile_noise_eval launches the same kernel).
//
//   het_profile_kernel<Out>  one thread per costed candidate: the strategies and partition of its detail row and the
//                            device groups of its plan, held fixed, under every scenario profile in turn.  The block
//                            walks the scenarios in step: thread 0 binds the block's Tables to scenario j's packed
//                            blob, then each thread runs profile_candidate (metis_recost.cuh): get_cost
//                            (RecostEvaluator::load + scenario_cost, the evaluator of the bandwidth what-if) and the
//                            memory state of every stage (PlanEvaluator::stage_memory) under those tables.  `Out`
//                            (metis_blob.cuh) is what a caller keeps: ProfileOut cost, headroom and status, NoiseOut
//                            cost and the usable byte.
//
// A scenario keeps its own uniform_bw and derived tables: its bandwidths are the searched cluster's, so under the
// searched profile the kernel computes what the search computed, bit for bit.  Scenarios may differ in key set,
// num_bs and lpad, so each one has its own blob and layout; stage_scenarios packs them and writes their descriptors.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdint>
#include <vector>

#include "../../include/metis_b200.h"
#include "metis_blob.cuh"
#include "metis_internal.h"
#include "metis_recost.cuh"

namespace metis {

constexpr int kProfileThreads = 128;
constexpr int kMaxScenarios = 65535;
constexpr int kPS = METIS_MAX_STAGES, kPL = METIS_MAX_LAYERS;

template <class Out>
__global__ void __launch_bounds__(kProfileThreads)
het_profile_kernel(const __grid_constant__ MetisPlanSpace sp, const ScenarioTables *__restrict__ scen, int K,
                   const MetisRecord *__restrict__ records, long long n, const uint8_t *__restrict__ detail, int stride,
                   const __grid_constant__ Out out) {
    __shared__ Tables s_T;
    const long long i = (long long)blockIdx.x * kProfileThreads + threadIdx.x;
    Scratch<kPS, kPL> w;
    RecostEvaluator<kPS, kPL> ev(s_T, w);
    PlanDesc pd;
    const bool known = i < n && decode_plan(sp, records[i].ordinal, pd) && pd.S <= kPS;
    for (int j = 0; j < K; ++j) {
        __syncthreads();                                      // the previous scenario's tables are no longer read
        if (threadIdx.x == 0) s_T = make_tables(scen[j].p, scen[j].lay, scen[j].blob);
        __syncthreads();
        if (i >= n) continue;
        if (!known) {                                         // not a plan of this space: never a searched candidate
            out.unknown(j, i, n);
            continue;
        }
        double c, h;
        const uint8_t st = profile_candidate(ev, pd, detail + (size_t)i * stride, c, h);
        out.store(j, i, n, c, h, st);
    }
}

template <class Out>
void launch_profile_kernel(const MetisPlanSpace &sp, const ScenarioTables *scen, int K, const MetisRecord *records,
                           int64_t n, const uint8_t *detail, int stride, const Out &out, cudaStream_t stream) {
    if (n <= 0) return;
    const unsigned nb = (unsigned)((n + kProfileThreads - 1) / kProfileThreads);
    het_profile_kernel<Out><<<nb, kProfileThreads, 0, stream>>>(sp, scen, K, records, n, detail, stride, out);
}

template void launch_profile_kernel<ProfileOut>(const MetisPlanSpace &, const ScenarioTables *, int,
                                                const MetisRecord *, int64_t, const uint8_t *, int,
                                                const ProfileOut &, cudaStream_t);
template void launch_profile_kernel<NoiseOut>(const MetisPlanSpace &, const ScenarioTables *, int, const MetisRecord *,
                                              int64_t, const uint8_t *, int, const NoiseOut &, cudaStream_t);

int stage_scenarios(const MetisProblem *problems, int K, ScenarioTables *desc, uint8_t *blobs, cudaStream_t stream) {
    std::vector<ScenarioTables> host((size_t)K);
    for (int j = 0; j < K; ++j) {
        const int64_t bytes = replay_tables_bytes(&problems[j]);
        if (bytes < 0) return (int)bytes;
        ScenarioTables &d = host[(size_t)j];
        d.p = problems[j];
        const int rc = stage_replay_tables(&problems[j], blobs, align256(bytes), stream, d.lay, d.blob);
        if (rc) return rc;
        blobs += align256(bytes);
    }
    // pageable source: staged before the call returns, so `host` may go
    cudaMemcpyAsync(desc, host.data(), host.size() * sizeof(ScenarioTables), cudaMemcpyHostToDevice, stream);
    return METIS_OK;
}

}  // namespace metis

using namespace metis;

extern "C" {

int64_t metis_het_profile_recost_workspace_bytes(const MetisProblem *scenarios, int32_t num_scenarios) {
    if (!scenarios || num_scenarios < 1 || num_scenarios > kMaxScenarios) return METIS_E_ARG;
    int64_t total = align256((int64_t)num_scenarios * (int64_t)sizeof(ScenarioTables)) + 256;
    for (int j = 0; j < num_scenarios; ++j) {
        const int64_t b = replay_tables_bytes(&scenarios[j]);
        if (b < 0) return b;
        total += align256(b);
    }
    return total;
}

int metis_het_profile_recost(const MetisPlanSpace *space, const MetisProblem *scenarios, int32_t num_scenarios,
                             const MetisRecord *records, int64_t n, const uint8_t *detail, int32_t detail_stride,
                             double *costs, double *headroom, uint8_t *status, void *workspace,
                             int64_t workspace_bytes, void *stream_) {
    if (!space || !scenarios || !workspace || (n > 0 && (!records || !detail || !costs || !headroom || !status)))
        return fail_arg("metis_het_profile_recost: NULL argument");
    if (n < 0) return fail_arg("metis_het_profile_recost: negative number of records");
    if (num_scenarios < 1 || num_scenarios > kMaxScenarios)
        return fail_arg("metis_het_profile_recost: num_scenarios out of range (1 .. 65535)");
    if (detail_stride < 3 * space->max_stage + 1)
        return fail_arg("metis_het_profile_recost: detail_stride too small (3 * max_stage + 1)");
    const MetisProblem &p0 = scenarios[0];
    for (int j = 1; j < num_scenarios; ++j) {                 // the searched cluster and flags, in every scenario
        const MetisProblem &q = scenarios[j];
        if (q.num_types != p0.num_types || q.num_layers != p0.num_layers || q.gbs != p0.gbs ||
            q.num_nodes != p0.num_nodes || q.devices_per_node != p0.devices_per_node ||
            q.total_devices != p0.total_devices || q.num_node_sequences != p0.num_node_sequences ||
            q.q10_devices != p0.q10_devices || q.uniform_bw != p0.uniform_bw || q.corrected != p0.corrected)
            return fail_arg("metis_het_profile_recost: a scenario differs from scenarios[0] outside the profile");
    }
    const int64_t need = metis_het_profile_recost_workspace_bytes(scenarios, num_scenarios);
    if (need < 0) return (int)need;
    if (workspace_bytes < need) return METIS_E_CAPACITY;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    uint8_t *base = align_workspace(workspace);
    ScenarioTables *desc = reinterpret_cast<ScenarioTables *>(base);
    const int rc = stage_scenarios(scenarios, num_scenarios, desc,
                                   base + align256((int64_t)num_scenarios * (int64_t)sizeof(ScenarioTables)), stream);
    if (rc) return rc;
    launch_profile_kernel(*space, desc, num_scenarios, records, n, detail, detail_stride,
                          ProfileOut{costs, headroom, status}, stream);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? METIS_OK : fail_cuda(e, "het_profile_kernel");
}

}  // extern "C"
