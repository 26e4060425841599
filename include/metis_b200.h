/*
 * metis_b200.h - C ABI of libmetis_b200.so (hand-written sm_90a CUDA).
 *
 * The reference (SamsungLabs/Metis @ ed41176) is pure Python and has no FFI
 * layer; its seam for the plan-search hot path is the pair of Python functions
 *     cost_het_cluster(args, gpu_cluster, profile_data, model_config,
 *                      cost_estimator, layer_load_balancer)   cost_het_cluster.py:21-50
 *     cost_homo_cluster(args, gpu_cluster, cost_estimator)    cost_homo_cluster.py:21-37
 * Each entry point below replaces the body of one of those loops (or one of the
 * functions they call); INTEGRATION.md shows the ctypes stub a maintainer would
 * add to the reference.  Conventions:
 *   - plain pointers and sizes only; every buffer is caller-allocated and
 *     caller-freed; pointers marked [device] must be CUDA device memory on the
 *     current device, [host] ordinary (ideally pinned) host memory;
 *   - every call only ENQUEUES work on `stream` (a cudaStream_t passed as
 *     void*, NULL = default stream) and returns; results are valid after the
 *     caller synchronises that stream;
 *   - return value 0 on success, a negative METIS_E_* code otherwise; the
 *     library never throws and keeps no global state;
 *   - no CPU fallback exists: without a CUDA device every compute entry point
 *     returns METIS_E_CUDA.
 */
#ifndef METIS_B200_H
#define METIS_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define METIS_ABI_VERSION 2

/* return codes */
#define METIS_OK            0
#define METIS_E_CUDA       -1   /* CUDA runtime error (see metis_last_error) */
#define METIS_E_ARG        -2   /* bad argument / unsupported size            */
#define METIS_E_CAPACITY   -3   /* caller buffer too small                    */

/* per-plan fatal codes (the reference would abort the whole search, quirk Q8) */
#define METIS_FATAL_NONE        0
#define METIS_FATAL_KEY_EXEC    1   /* KeyError 'tp{t}_bs{b}' in StagePerformance (model/device_group.py:38,49,79) */
#define METIS_FATAL_KEY_MEMORY  2   /* KeyError in _get_stage_memory_demand (model/load_balancer.py:43,51)          */
#define METIS_FATAL_INDEX       3   /* IndexError: fewer profiled layers than --num_layers (load_balancer.py:219)   */
#define METIS_FATAL_HANG        4   /* reference loop at load_balancer.py:96-104 would not terminate                */
#define METIS_FATAL_SCRATCH     5   /* internal scratch exceeded (more stages / leftovers than compiled limits)     */
#define METIS_FATAL_ZERODIV     6   /* ZeroDivisionError in the reference (zero profiled time / zero total)         */

/* MetisProblem.corrected bits (SURVEY.md 8(f)-4; never set by default) */
#define METIS_FIX_Q5  1   /* a layer goes to the stage holding MOST of its 7 sub-layers (lowest stage on ties):
                             no layer is dropped (the reference keeps only count > 3.5, load_balancer.py:293-296) */
#define METIS_FIX_Q6  2   /* memory demand from the profile of the stage's OWN device type; mixed-type stage:
                             largest replica instead of the sum over a whole-cluster split (load_balancer.py:41-52) */

/* limits compiled into the kernels */
#define METIS_MAX_TYPES   8
#define METIS_MAX_STAGES  128
#define METIS_MAX_LAYERS  256   /* scratch size; --num_layers itself is limited to 255 (one-byte partition entries) */

/*
 * Flattened search problem: the dict-of-dicts `profile_data` (data_loader.py:39-61),
 * `GPUCluster` (gpu_cluster.py:8-58), `ModelConfig` / `GPTActivationAndParam`
 * (utils.py:72-79, model/activation_parameter.py:5-51) and the flags read on the
 * hot path (cost_het_cluster.py:25-36) as dense arrays.
 *
 * A profile key 'tp{t}_bs{b}' of device type d is  key_index[(d*num_tp + log2(t))*num_bs + (b-1)]
 * (-1 = not profiled).  Layer tables are zero-padded to `lpad` entries.
 */
typedef struct MetisProblem {
    int32_t num_types;            /* distinct device types in the cluster                          */
    int32_t num_tp;               /* tp levels 1,2,4,.. covered by key_index                        */
    int32_t num_bs;               /* batch sizes 1..num_bs covered by key_index                     */
    int32_t num_keys;             /* profiled (type,tp,bs) keys                                     */
    int32_t lpad;                 /* padded length of the per-layer tables                          */
    int32_t num_layers;           /* --num_layers                                                   */
    int32_t norm_len;             /* len(norm_layer_duration)  (load_balancer.py:22-27)             */
    int32_t gbs;                  /* --gbs                                                          */
    int32_t max_tp;               /* --max_profiled_tp_degree                                       */
    int32_t max_bs;               /* --max_profiled_batch_size                                      */
    int32_t num_nodes;            /* gpu_cluster.get_num_nodes()                                    */
    int32_t devices_per_node;     /* gpu_cluster.get_num_devices_per_node() (node 0, quirk Q10)     */
    int32_t total_devices;
    int32_t num_node_sequences;
    int32_t uniform_bw;           /* 1 when every type has the same first/min bandwidth             */
    int32_t q10_devices;          /* num_nodes x devices of node 0: length of the rank lists the reference builds
                                     with node 0's GPU count (load_balancer.py:109-119, cluster_bandwidth.py:34-47;
                                     quirk Q10); == total_devices when every node has the same count   */
    int32_t corrected;            /* opt-in deviations from the reference (0 = strict parity): METIS_FIX_* bits  */
    int32_t reserved1;
    int64_t sequence_length, hidden_size, vocab_size;
    double optimizer_time;        /* profile_data['model']['optimizer_time'] (= 2 x optimizer_time_ms) */
    double batch_generator;       /* profile_data['model']['batch_generator']                       */
    double input_params, transformer_params, output_params;   /* activation_parameter.py:22-24      */
    double node0_bandwidth;       /* gpu_cluster.get_intra_bandwidth(0) (homo path, cluster_bandwidth.py:75-76) */
    double node0_memory;          /* gpu_cluster.get_device_memory(0)   (cost_estimator.py:31-32)    */
    const int16_t *key_index;     /* [device] [num_types][num_tp][num_bs]                           */
    const double *layer_compute;  /* [device] [num_keys][lpad]  'layer-computes'                    */
    const double *layer_memory;   /* [device] [num_keys][lpad]  'memory'                            */
    const double *exec_full;      /* [device] [num_keys]  sum(layer-computes)   (Python sum, host)  */
    const double *fb_sync;        /* [device] [num_keys]  0.0 = falsy -> KeyError (quirk Q9)        */
    const double *norm_lc;        /* [device] [norm_len]                                            */
    const double *type_memory;    /* [device] [num_types] get_device_memory_for_device_type()       */
    const double *type_bw_first;  /* [device] [num_types] _get_intra_bandwidth(type)                */
    const double *type_bw_min;    /* [device] [num_types] _get_inter_bandwidth([type]) (quirk Q2)   */
    const uint8_t *ns_run_type;   /* [device] [num_node_sequences][num_types] type id of k-th run   */
    const int32_t *ns_run_end;    /* [device] [num_node_sequences][num_types] cumulative rank count */
    const int32_t *ns_q10_end;    /* [device] [num_node_sequences][num_types] cumulative (nodes of the type x devices of
                                     node 0): the type runs of the Q10 rank list                        */
} MetisProblem;

/* One block of inter-stage plans sharing (ns_idx, num_stage): plan.py:153-175 incl. quirk Q1. */
typedef struct MetisPlanBlock {
    int64_t first_ordinal;        /* ordinal of (row 0, batches = gbs)                              */
    int64_t rows_offset;          /* byte offset of row 0 in MetisPlanSpace.rows                    */
    int32_t num_rows;             /* device-group rows in the block                                 */
    int16_t ns_idx;
    int16_t label_stage;          /* InterStagePlan.num_stage as emitted (1 for Q1 blocks)          */
    int16_t num_stage;            /* len(device_groups)                                             */
    int16_t reserved[3];
} MetisPlanBlock;

/*
 * The enumerated candidate space.  ordinal = first_ordinal + row*num_div + div_idx
 * reproduces the order of InterStagePlanGenerator.__next__ (plan.py:153-175).
 * Rows hold log2(group size), one byte per stage (device_group.py:93-107 order).
 */
typedef struct MetisPlanSpace {
    int64_t num_plans;
    int64_t rows_bytes;           /* size of the `rows` blob (must stay below 4 GiB)                   */
    int32_t num_blocks;
    int32_t num_div;
    int32_t max_stage;            /* largest num_stage of any block (sizes the per-plan task state)  */
    int32_t reserved;
    const MetisPlanBlock *blocks; /* [device] [num_blocks]                                          */
    const int32_t *batches;       /* [device] [num_div] divisors of gbs, descending (plan.py:120-124) */
    const uint8_t *rows;          /* [device]                                                       */
} MetisPlanSpace;

/* 16-byte record per costed candidate (one per estimate_costs.append, cost_het_cluster.py:44-46). */
typedef struct MetisRecord {
    double cost;
    uint32_t ordinal;             /* inter-stage plan ordinal                                       */
    uint16_t step;                /* index of the yield inside the plan's intra-stage chain         */
    uint8_t num_repartition;      /* IntraStagePlan.num_repartition (1..3)                          */
    uint8_t num_stage;
} MetisRecord;

/* Summary written to host memory by metis_het_search (valid after stream sync). */
typedef struct MetisSearchSummary {
    uint64_t num_records;         /* C: candidates costed (may exceed record capacity: then truncated) */
    uint64_t num_partition_calls; /* B: LayerLoadBalancer.partition_layer invocations               */
    uint64_t num_balancer_runs;   /* LayerComputeBalancer.run invocations                           */
    uint64_t num_keyerror;        /* candidates skipped by `except KeyError` (cost_het_cluster.py:47) */
    uint64_t fatal_ordinal;       /* lowest ordinal that hit a fatal condition, UINT64_MAX if none  */
    uint32_t fatal_code;          /* METIS_FATAL_* of that ordinal                                  */
    uint32_t fatal_aux;           /* tp<<16 | bs of the missing key when applicable                 */
    MetisRecord best;             /* argmin (cost, ordinal, step); cost = +inf when no record       */
    uint64_t reserved[6];         /* [0] plans admitted (have a valid first strategy), [1] plans handed from the
                                     bulk round to the chain kernel, [2] the instantiation of the search
                                     kernels that ran: MAXS | MAXL << 16 | ONE << 32 (scratch sized for
                                     MAXS stages / MAXL layers; ONE = single-type cluster), [3] the
                                     out-of-memory partition attempts of a search with misses
                                     (metis_het_search_outputs; exact past the capacity, 0 without); rest 0 */
} MetisSearchSummary;

/*
 * 16-byte record per out-of-memory partition attempt (metis_het_search_outputs): one pass of the partition_layer loop
 * whose memory test fails (model/load_balancer.py:57-63,127-143), the third attempt and the attempts whose re-weighting
 * is None included.  deficit, ordinal and key sit where MetisRecord keeps cost, ordinal and step, so
 * metis_sort_records orders misses too: METIS_SORT_POSITION by (ordinal, call, attempt), the order the reference
 * prints them; METIS_SORT_RANKED closest first (smallest deficit), ties in that order.
 */
typedef struct MetisMiss {
    double deficit;               /* -min_s memory_state[s] (MB), > 0                                  */
    uint32_t ordinal;             /* inter-stage plan ordinal                                       */
    uint16_t key;                 /* call << 2 | attempt: call = 0-based partition_layer call of the plan, attempt 1..3;
                                     a plan makes at most num_stage * floor(log2(max_tp)) + 1 <= 3 841 calls (every
                                     strategy of its chain doubles one stage's tp), so the call fits in 14 bits */
    uint8_t stage;                /* lowest stage attaining that minimum                            */
    uint8_t num_stage;
} MetisMiss;

/* Shard of the ordinal space evaluated by one call (multi-GPU: rank r of n, interleaved tiles). */
typedef struct MetisShard {
    int32_t rank;                 /* 0 <= rank < world                                              */
    int32_t world;
    int32_t tile;                 /* plans per interleave tile (multiple of 32)                     */
    int32_t reserved;             /* tuning: minimum number of admitted plans for which the bulk round (first
                                     partition attempt, one plan per thread) runs before the chain kernel;
                                     0 = default (12 x resident chain warps), INT32_MAX = chain kernel only */
} MetisShard;

const char *metis_last_error(void);
int metis_abi_version(void);

/*
 * Optional: CUDA events (cudaEvent_t as void*) that the NEXT metis_het_search call on this host
 * thread records immediately before and after its search kernel, so a caller can time that kernel
 * alone on the launching stream.  Pass NULLs to clear.
 */
void metis_set_profile_events(void *before_kernel, void *after_kernel);

/* Bytes of device scratch metis_het_search needs for a shard of `num_plans` plans: the packed tables
 * plus two lists of 16 B per plan (worst case: every plan has a valid strategy); `max_stage` is ignored.
 * metis_het_detail / metis_het_trace / metis_het_breakdown / metis_homo_cost / metis_homo_breakdown need
 * metis_het_workspace_bytes(problem, 0, 1).
 * About 36 B per plan in all: a space whose workspace, rows and records do not fit the device (or that has 2^32
 * plans or 4 GiB of rows) is searched in ordinal windows, each a MetisPlanSpace of its own
 * (metis_b200.flatten.plan_windows sizes them with this function). */
int64_t metis_het_workspace_bytes(const MetisProblem *problem, int64_t num_plans, int32_t max_stage);

/*
 * Replaces the loop of cost_het_cluster.py:24-48 for the shard's plans.
 *   records      [device] capacity MetisRecord slots (unordered; sort by (ordinal, step) to get
 *                estimate_costs order); may be NULL with capacity 0 when only the best is wanted
 *   detail       [device] optional, capacity * detail_stride bytes: per record
 *                dp code[num_stage], tp code[num_stage] (log2) then layer_partition[num_stage+1]
 *                (uint8 each); detail_stride >= 3*space->max_stage+1, or NULL
 *   workspace    [device] metis_het_workspace_bytes(problem, plans in shard, space->max_stage) bytes
 *   summary      [host]   filled asynchronously (use pinned memory)
 */
int metis_het_search(const MetisProblem *problem, const MetisPlanSpace *space, const MetisShard *shard,
                     MetisRecord *records, int64_t capacity, uint8_t *detail, int32_t detail_stride,
                     void *workspace, int64_t workspace_bytes, MetisSearchSummary *summary, void *stream);

/*
 * metis_het_search that also writes each record's memory headroom: headroom[i] = min over all num_stage stages of
 * memory_state (capacity - demand, model/load_balancer.py:57-63) of the partition attempt that record i accepted,
 * the value MetisBreakdown.min_headroom reports for it.
 *   headroom [device] capacity doubles aligned with records, or NULL (then exactly metis_het_search)
 */
int metis_het_search_headroom(const MetisProblem *problem, const MetisPlanSpace *space, const MetisShard *shard,
                              MetisRecord *records, int64_t capacity, uint8_t *detail, int32_t detail_stride,
                              double *headroom, void *workspace, int64_t workspace_bytes, MetisSearchSummary *summary,
                              void *stream);

/*
 * metis_het_search_headroom that also writes every out-of-memory partition attempt of the search as a MetisMiss, in no
 * particular order (sort them with metis_sort_records).  The number of attempts lands in summary->reserved[3], also
 * when it exceeds miss_capacity (then only the first miss_capacity are written: search again with more room).
 *   misses [device] miss_capacity records, or NULL (then exactly metis_het_search_headroom)
 */
int metis_het_search_outputs(const MetisProblem *problem, const MetisPlanSpace *space, const MetisShard *shard,
                             MetisRecord *records, int64_t capacity, uint8_t *detail, int32_t detail_stride,
                             double *headroom, MetisMiss *misses, int64_t miss_capacity, void *workspace,
                             int64_t workspace_bytes, MetisSearchSummary *summary, void *stream);

/*
 * Re-evaluates the listed (ordinal, step) candidates and writes their strategies and
 * partition (same layout as `detail` above).  Used to materialise the winner / a ranked slice.
 *   picks [device] n MetisRecord (only ordinal and step are read)
 */
int metis_het_detail(const MetisProblem *problem, const MetisPlanSpace *space, const MetisRecord *picks,
                     int64_t n, uint8_t *detail, int32_t detail_stride, void *workspace,
                     int64_t workspace_bytes, void *stream);

/*
 * Verbose transcript (debug): replays the listed inter-stage plans, one thread each, and records the values the
 * reference prints while it evaluates them (search_space/plan.py:207-218, model/load_balancer.py:92,132-133,143,
 * model/cost_estimator.py:193,201-203,239-240, cost_het_cluster.py:43,48) as a stream of 64-bit words per plan; the
 * layout is documented in metis_b200/csrc/metis_trace.cuh and decoded by metis_b200/verbose.py.
 *   ordinals [device] n uint32 plan ordinals;  trace [device] n * words_per_plan uint64 (words_per_plan >= 64)
 */
int metis_het_trace(const MetisProblem *problem, const MetisPlanSpace *space, const uint32_t *ordinals, int64_t n,
                    uint64_t *trace, int32_t words_per_plan, void *workspace, int64_t workspace_bytes, void *stream);

/*
 * Cost breakdown of costed candidates: what HeteroCostEstimator.get_cost adds up (model/cost_estimator.py:235-242) and
 * the memory headroom of the accepted partition attempt (IntraStagePlan.memory_state, model/load_balancer.py:57-63).
 */
typedef struct MetisBreakdown {          /* 64 B per candidate */
    double terms[6];              /* execution, fb_sync, max parameter update, max dp, pp, batch generate; summed left to
                                     right they give the record's cost                                            */
    double min_headroom;          /* min over the stages of memory_state (capacity - demand)                        */
    int16_t min_stage;            /* its stage, lowest on ties                                                      */
    int16_t costed_stages;        /* min(InterStagePlan.num_stage, len(device_groups)): the stages get_cost walks (Q1) */
    int16_t num_stage;            /* len(device_groups); 0 = the pick is not a costed candidate of the space        */
    int16_t reserved;
} MetisBreakdown;

/* per-stage fields of metis_het_breakdown's stage_out, in this order */
#define METIS_BD_PERFORMANCE  0   /* stage compute performance fed to the accepted balancer run                      */
#define METIS_BD_EXEC_TIME    1   /* stage execution time (lens[s], cost_estimator.py:208-210)                       */
#define METIS_BD_CAPACITY     2   /* stage memory capacity                                                          */
#define METIS_BD_DEMAND       3   /* stage memory demand of the accepted attempt                                    */
#define METIS_BD_STATE        4   /* memory_state = capacity - demand                                               */
#define METIS_BD_DP           5   /* dp cost                                                                        */
#define METIS_BD_UPDATE       6   /* parameter update cost                                                          */
#define METIS_BD_PP           7   /* pp hop cost to the next stage (0 for the last costed stage)                    */
#define METIS_BD_FIELDS       8

/*
 * Replays the plans of the listed candidates (one thread per distinct ordinal; each plan's chain runs once however
 * many of its steps are asked for) and writes their breakdowns.
 *   picks     [device] n MetisRecord sorted by (ordinal, step); only ordinal and step are read
 *   out       [device] n MetisBreakdown
 *   stage_out [device] optional: n x METIS_BD_FIELDS x stage_stride doubles, field-major per pick; NaN past
 *             num_stage, and in the cost fields (exec time, dp, update, pp) past costed_stages.
 *             stage_stride >= num_stage of every pick (a pick with more stages gets no stage rows), or NULL
 *   workspace [device] metis_het_workspace_bytes(problem, 0, 1) bytes
 */
int metis_het_breakdown(const MetisProblem *problem, const MetisPlanSpace *space, const MetisRecord *picks, int64_t n,
                        MetisBreakdown *out, double *stage_out, int32_t stage_stride, void *workspace,
                        int64_t workspace_bytes, void *stream);

/*
 * Network what-if: HeteroCostEstimator.get_cost (model/cost_estimator.py:199-244) of costed candidates under other
 * bandwidth tables.  Bandwidth enters only the cost model, so the strategies and partition a search found stay valid;
 * each candidate is re-costed from its detail row with no balancer run.  Every scenario goes through the general
 * (non-uniform) bandwidth path; under the search's own tables the costs equal the search's bit for bit.
 *   records    [device] n MetisRecord of one search (any order); only ordinal is read
 *   detail     [device] n rows of detail_stride bytes: dp codes[S], tp codes[S], partition[S+1], as the search writes
 *              them; detail_stride >= 3 * space->max_stage + 1
 *   bandwidths [device] num_scenarios x 2 x num_types doubles: bw_first[T] then bw_min[T] of each scenario
 *              (MetisProblem.type_bw_first / type_bw_min)
 *   costs      [device] num_scenarios x n doubles: costs[j * n + i] is record i's cost under scenario j; NaN when its
 *              replay raises a KeyError (cannot happen for a record the search costed)
 *   workspace  [device] metis_het_workspace_bytes(problem, 0, 1) bytes
 */
int metis_het_recost(const MetisProblem *problem, const MetisPlanSpace *space, const MetisRecord *records, int64_t n,
                     const uint8_t *detail, int32_t detail_stride, const double *bandwidths, int32_t num_scenarios,
                     double *costs, void *workspace, int64_t workspace_bytes, void *stream);

/*
 * Regret of re-costed candidates: best[j] = min_i costs[j * n + i] and regret[i] = max_j (costs[j * n + i] - best[j]),
 * in fp64 (absolute, not a ratio: costs of rough profiles may be negative).  Exact, whatever the reduction order.
 * NaN costs are skipped by the min.  With n == 0, best[j] = +inf.
 *   costs     [device] num_scenarios x n doubles (metis_het_recost's layout), 1 <= num_scenarios <= 65535
 *   best      [device] num_scenarios doubles;  regret [device] n doubles
 *   workspace [device] metis_recost_regret_workspace_bytes(num_scenarios, n) bytes
 */
int64_t metis_recost_regret_workspace_bytes(int32_t num_scenarios, int64_t n);
int metis_recost_regret(const double *costs, int32_t num_scenarios, int64_t n, double *best, double *regret,
                        void *workspace, int64_t workspace_bytes, void *stream);

/*
 * Profile what-if: costed candidates of one search under other profiles, with their device groups, strategies and
 * layer partition held fixed (no strategy chain, no balancer run: not what a search under the scenario returns).
 * For scenario j, record i:
 *   costs[j * n + i]    HeteroCostEstimator.get_cost (model/cost_estimator.py:199-244) under scenario j's tables;
 *                       NaN when it raises
 *   headroom[j * n + i] min over all S stages of memory capacity - LayerLoadBalancer._get_stage_memory_demand
 *                       (model/load_balancer.py:29-55, quirks Q6 and Q10) under scenario j; NaN when the demand raises
 *   status[j * n + i]   cost_code | memory_code << 4, each METIS_FATAL_NONE or a METIS_FATAL_* code: cost_code is
 *                       METIS_FATAL_KEY_EXEC whenever get_cost raises; memory_code is the first failing stage's
 *                       METIS_FATAL_KEY_MEMORY / KEY_EXEC (a missing key), METIS_FATAL_INDEX (Q10) or
 *                       METIS_FATAL_ZERODIV (the data split of a mixed-type stage)
 *   A candidate is usable under scenario j when status == 0 and headroom >= 0.
 * Each scenario is a MetisProblem flattened from a profile under the searched cluster, model flags and corrections:
 * its profile tables (keys, num_bs, lpad, ...) may differ, its scalar fields outside the profile must equal
 * scenarios[0]'s (num_types, num_layers, gbs, num_nodes, devices_per_node, total_devices, num_node_sequences,
 * q10_devices, uniform_bw, corrected; otherwise METIS_E_ARG).  Its cluster tables (memory, bandwidth, node sequence
 * runs) are not compared: the caller builds every scenario from the searched cluster.  Under the searched profile,
 * costs and headroom equal the search's, bit for bit.
 *   space      the searched plan space;  records [device] n MetisRecord of it (any order), only ordinal is read
 *   detail     [device] n rows of detail_stride bytes, as for metis_het_recost; detail_stride >= 3 * max_stage + 1
 *   costs, headroom [device] num_scenarios x n doubles;  status [device] num_scenarios x n bytes
 *   1 <= num_scenarios <= 65535;  workspace [device] metis_het_profile_recost_workspace_bytes(scenarios, num_scenarios)
 *   bytes (METIS_E_CAPACITY when smaller), laid out as the scenarios' descriptors, then each one's packed tables
 */
int64_t metis_het_profile_recost_workspace_bytes(const MetisProblem *scenarios, int32_t num_scenarios);
int metis_het_profile_recost(const MetisPlanSpace *space, const MetisProblem *scenarios, int32_t num_scenarios,
                             const MetisRecord *records, int64_t n, const uint8_t *detail, int32_t detail_stride,
                             double *costs, double *headroom, uint8_t *status,
                             void *workspace, int64_t workspace_bytes, void *stream);

/*
 * Profile-noise what-if: the profile what-if above under seeded samples of the searched profile, drawn on the device,
 * reduced to per-candidate counts without the K x n arrays leaving the device.  Sample j is search.noisy_profile
 * (profile, sigma, seed, j): every layer-computes and memory entry and every fb_sync of each key multiplied by its own
 * factor 1 + s * (2u - 1), u from Philox4x32-10 of (j, index, bs, field << 16 | type << 8 | log2 tp) under the seed
 * (metis_b200/csrc/metis_noise.cuh).  A chunk of `count` samples, j = first .. first + count - 1, goes through three
 * calls on one stream:
 *   draw      metis_het_profile_noise_draw: the chunk's layer_compute, layer_memory, exec_full and fb_sync from the
 *             base problem's (the searched problem, bound on the device), every other table the base's, each sample's
 *             tables packed, into the workspace
 *   evaluate  metis_het_profile_noise_eval, per record range: cost[s * ld + i] (NaN when get_cost raises) and
 *             usable[s * ld + i] (status == 0 and headroom >= 0, as metis_het_profile_recost) of record i under sample
 *             first + s
 *   reduce    metis_het_profile_noise_reduce, once all n records are evaluated: per sample, best_pos[s] / best_cost[s]
 *             the usable record of lowest cost, ties to the lowest position (-1 / NaN when none is usable); per record,
 *             the chunk's samples added in order to wins (best_pos == i), near (usable and cost <= best_cost * t),
 *             usable (count), regret (max of cost - best_cost; +inf once unusable) and sum (costs of usable samples,
 *             left to right).  The caller zeroes wins, near, usable and sum and sets regret to -inf before the first
 *             chunk; the results do not depend on the chunk size.
 */
typedef struct MetisNoiseSpec {
    double sigma[3][METIS_MAX_TYPES];  /* [field - 1][device type of the problem]: layer-computes, memory, fb_sync;
                                          each finite, in [0, 1); 0 leaves the field as it is                      */
    uint64_t seed;
    int32_t first;                     /* the chunk's first sample j                                                */
    int32_t count;                     /* samples in the chunk: 1 <= count, first + count <= 65535                  */
    uint8_t type_code[METIS_MAX_TYPES];/* 1-based utils.DeviceType position of each device type of the problem     */
    double near_factor;                /* 1.0 + within: finite, >= 1                                                */
} MetisNoiseSpec;

/* workspace bytes of one chunk of `count` samples of `base`, or METIS_E_ARG */
int64_t metis_het_profile_noise_workspace_bytes(const MetisProblem *base, int32_t count);
int metis_het_profile_noise_draw(const MetisProblem *base, const MetisNoiseSpec *spec, void *workspace,
                                 int64_t workspace_bytes, void *stream);
/* records / detail as for metis_het_profile_recost; cost, usable [device] spec->count rows of ld >= n entries */
int metis_het_profile_noise_eval(const MetisPlanSpace *space, const MetisNoiseSpec *spec, const void *workspace,
                                 const MetisRecord *records, int64_t n, const uint8_t *detail, int32_t detail_stride,
                                 double *cost, uint8_t *usable, int64_t ld, void *stream);
/* cost, usable [device] spec->count x n (ld = n); best_pos, best_cost [device] spec->count; wins, near, usable_count,
 * regret, sum [device] n */
int metis_het_profile_noise_reduce(const MetisNoiseSpec *spec, const double *cost, const uint8_t *usable, int64_t n,
                                   int64_t *best_pos, double *best_cost, int32_t *wins, int32_t *near,
                                   int32_t *usable_count, double *regret, double *sum, void *stream);

/*
 * Search what-if: a fresh search under each seeded sample of the profile (search.noisy_profile), the balancer's layer
 * weights included.  The draw is metis_het_profile_noise_draw's, and it also writes each sample's norm_lc
 * (load_balancer.py:22-27, quirk Q3): the tp1_bs1 layer-computes of the profile's FIRST-LISTED entry, which need not be
 * a device type of the cluster, each multiplied by its factor (field 1, tp 1, bs 1, that entry's device type), then
 * each divided by their CPython sum.  Under sigma 0 for that entry's layer-computes it is the base's norm_lc.  The
 * workspace's descriptors at its start serve metis_het_profile_noise_eval as after metis_het_profile_noise_draw, and
 * metis_het_search_noise_problem gives sample s's MetisProblem (device pointers into the workspace) for
 * metis_het_search / metis_het_detail.  The workspace must not change while those run.
 */
typedef struct MetisNormSource {
    const double *row;            /* [device] len doubles: the first-listed entry's tp1_bs1 'layer-computes'         */
    int32_t len;                  /* == base->norm_len                                                            */
    int32_t type_code;            /* 1-based utils.DeviceType position of that entry's device type (1 .. 6)       */
    double sigma;                 /* its layer-computes sigma, finite, in [0, 1)                                  */
} MetisNormSource;

/* workspace bytes of one chunk of `count` samples of `base`, or METIS_E_ARG */
int64_t metis_het_search_noise_workspace_bytes(const MetisProblem *base, int32_t count);
/* norm_zero [device] spec->count bytes: 1 where the sample's noisy norm total is 0 (the reference raises
 * ZeroDivisionError; that sample's norm_lc is then the base's), else 0.  spec->near_factor is checked, not read. */
int metis_het_search_noise_draw(const MetisProblem *base, const MetisNoiseSpec *spec, const MetisNormSource *norm,
                                void *workspace, int64_t workspace_bytes, uint8_t *norm_zero, void *stream);
/* host only: sample s (0 <= s < spec->count) of the chunk drawn into workspace with the same base and spec */
int metis_het_search_noise_problem(const MetisProblem *base, const MetisNoiseSpec *spec, int32_t s,
                                   const void *workspace, MetisProblem *sample);

/*
 * metis_homo_cost with the cost terms and the per-stage memory sums (HomoCostEstimator.get_cost returns them as
 * stage_memory, model/cost_estimator.py:121-138).
 *   terms        [device] n x 6 doubles: execution, fb_sync, parameter update, dp, pp, batch generate
 *   stage_memory [device] n x stage_stride doubles, NaN past pp
 *   status       [device] n int32: 0 ok, 1 KeyError (plan skipped), 2 oom flag set, 3 pp > stage_stride
 */
int metis_homo_breakdown(const MetisProblem *problem, int32_t type_id, const int32_t *plans, int64_t n, double *terms,
                         double *stage_memory, int32_t stage_stride, int32_t *status, void *workspace,
                         int64_t workspace_bytes, void *stream);

/*
 * Replaces HomoCostEstimator.get_cost (model/cost_estimator.py:98-138) for n UniformPlans
 * (search_space/plan.py:12-18), as called from cost_homo_cluster.py:29.
 *   plans  [device] n x 5 int32 (dp, pp, tp, mbs, gbs)
 *   cost   [device] n doubles;  status [device] n int32: 0 ok, 1 KeyError (plan skipped), 2 oom flag set
 */
int metis_homo_cost(const MetisProblem *problem, int32_t type_id, const int32_t *plans, int64_t n,
                    double *cost, int32_t *status, void *workspace, int64_t workspace_bytes, void *stream);

/*
 * LayerComputeBalancer.run (model/load_balancer.py:197-207) for n independent instances.
 *   capa [device] n x stride doubles (stage capacities), num_stage [device] n int32,
 *   lc [device] norm_len doubles, partition [device] n x (stride+1) uint16 out (0xFFFF first = error),
 *   workspace [device] >= norm_len*8 + 256 bytes
 */
int metis_layer_balance(const double *capa, const int32_t *num_stage, int64_t n, int32_t stride,
                        const double *lc, int32_t norm_len, int32_t num_layers, uint16_t *partition,
                        void *workspace, int64_t workspace_bytes, void *stream);

/*
 * Orders the records written by metis_het_search on the device (stable LSD radix sort, one cooperative kernel).
 *   METIS_SORT_POSITION        by (ordinal, step): the order of `estimate_costs` as the reference appends it
 *                              (cost_het_cluster.py:44)
 *   METIS_SORT_RANKED          by (cost, ordinal, step): `sorted(estimate_costs, key=lambda kv: kv[-1])`
 *                              (cost_het_cluster.py:76; Python's sort is stable, so equal costs stay in
 *                              estimate_costs order)
 *   METIS_SORT_BY_COST_STABLE  by cost only, equal costs keep their current order (the second half of
 *                              METIS_SORT_RANKED, for records that are already in position order)
 *   records   [device] n records, sorted in place
 *   perm_out  [device] optional n uint32: perm_out[i] = index before the call of the record now at i
 *   workspace [device] metis_sort_workspace_bytes(n) bytes
 */
#define METIS_SORT_POSITION        0
#define METIS_SORT_RANKED          1
#define METIS_SORT_BY_COST_STABLE  2
int64_t metis_sort_workspace_bytes(int64_t n);
int metis_sort_records(MetisRecord *records, int64_t n, int32_t mode, uint32_t *perm_out, void *workspace,
                       int64_t workspace_bytes, void *stream);

/*
 * Headroom-constrained views of the ranked list (metis_select.cu).  Inputs, all on the device:
 *   records  n records in estimate_costs order (only the cost is read)
 *   headroom n doubles aligned with records (metis_het_search_headroom), no NaN
 *   rank     n uint32: the perm_out of metis_sort_records(METIS_SORT_BY_COST_STABLE) on those records, i.e. the
 *            ranked list sorted(estimate_costs, key=cost) as positions in estimate_costs order
 *   workspace [device] metis_headroom_workspace_bytes(n) bytes
 *   count    [host] written asynchronously (use pinned memory)
 *
 * metis_headroom_select: the first k entries of the ranked list whose headroom is >= min_headroom (finite), in ranked
 *   order, as positions into out [device, k uint32]; *count = how many of the n qualify.
 * metis_headroom_front: the cost / headroom Pareto front.  A candidate is on it iff no other one has cost <= and
 *   headroom >= with one of the two strict; of several with equal (cost, headroom) only the first in estimate_costs
 *   order is kept.  out [device, n uint32] gets the front's positions by ascending cost (headroom then strictly
 *   increases); *count = the front's length.
 */
int64_t metis_headroom_workspace_bytes(int64_t n);
int metis_headroom_select(const double *headroom, const uint32_t *rank, int64_t n, double min_headroom, int64_t k,
                          uint32_t *out, uint64_t *count, void *workspace, int64_t workspace_bytes, void *stream);
int metis_headroom_front(const MetisRecord *records, const double *headroom, const uint32_t *rank, int64_t n,
                         uint32_t *out, uint64_t *count, void *workspace, int64_t workspace_bytes, void *stream);

/*
 * Plan queries of a finished search (metis_query.cu).  A MetisPlanFilter is a set of conditions on one candidate of
 * the reference's estimate_costs list (cost_het_cluster.py:44-46); it selects among the candidates the search found,
 * it does not constrain the search (the strategy chain ran unconstrained).  A candidate is admitted when
 *   min_stages <= len(device_groups) <= max_stages, num_repartition <= max_repartition,
 *   bit ns_idx of ns_mask and bit (index of its batches in MetisPlanSpace.batches) of div_mask are set,
 * and, with METIS_QUERY_NEEDS_TP in flags (the tp codes of its detail row are read), every stage s has
 *   log2(tp) <= max_tp_code; with uniform_tp, the tp of stage 0; with METIS_QUERY_BY_TYPE, log2(tp) <=
 *   type_tp_code[d] for every device type d among the ranks [sum(groups[:s]), sum(groups[:s+1])) of the node
 *   sequence's placement (ns_run_type / ns_run_end, model/device_group.py:22-32, 60-64).
 * The group of an admitted candidate is the mixed radix of the digits of its num_keys key fields (first most
 * significant); digit k is the field's value as below, in 0 .. key_range[k]-1 (outside: no group).
 */
#define METIS_QUERY_KEY_NS       0   /* node sequence index                                           */
#define METIS_QUERY_KEY_STAGES   1   /* len(device_groups) - 1                                        */
#define METIS_QUERY_KEY_BATCHES  2   /* rank of batches among the divisors of gbs, smallest first       */
#define METIS_QUERY_KEY_MAX_TP   3   /* log2 of the largest tp of any stage (reads the detail row)     */
#define METIS_QUERY_KEY_NREP     4   /* num_repartition - 1                                           */
#define METIS_QUERY_MAX_KEYS     5
#define METIS_QUERY_NEEDS_TP     1   /* flags: the conditions read the tp codes                         */
#define METIS_QUERY_BY_TYPE      2   /* flags: type_tp_code holds a limit                               */
#define METIS_QUERY_NO_GROUP     0xFFFFFFFFu

typedef struct MetisPlanFilter {
    int32_t min_stages, max_stages;
    int32_t max_repartition;
    int32_t max_tp_code;            /* 255 = no limit                                                  */
    int32_t uniform_tp;
    int32_t flags;                  /* METIS_QUERY_NEEDS_TP | METIS_QUERY_BY_TYPE                      */
    uint8_t type_tp_code[METIS_MAX_TYPES];   /* per device type id; 255 = no limit                    */
    uint32_t ns_mask[8];            /* 256 node sequences                                              */
    uint32_t div_mask[8];           /* 256 divisors of gbs                                             */
    int32_t num_keys;
    int32_t key_field[METIS_QUERY_MAX_KEYS];
    int32_t key_range[METIS_QUERY_MAX_KEYS];
    int32_t reserved;
} MetisPlanFilter;

/*
 * Filter and group key of n candidates, one thread each: mask[i] = 1 when candidate i is admitted and, if headroom
 * is given, headroom[i] >= min_headroom; group[i] its group, METIS_QUERY_NO_GROUP when mask[i] == 0.
 *   records  [device] n MetisRecord of `space` (ordinal and num_repartition are read)
 *   detail   [device] n rows of detail_stride bytes aligned with records (the search's layout), or NULL when flags has
 *            no METIS_QUERY_NEEDS_TP and no key is METIS_QUERY_KEY_MAX_TP
 *   headroom [device] n doubles aligned with records, or NULL;  mask [device] n bytes;  group [device] n uint32 or NULL
 * Reads only the problem's ns_run_type / ns_run_end and the space: no workspace, no table packing.
 */
int metis_query_mark(const MetisProblem *problem, const MetisPlanSpace *space, const MetisPlanFilter *filter,
                     const MetisRecord *records, int64_t n, const uint8_t *detail, int32_t detail_stride,
                     const double *headroom, double min_headroom, uint8_t *mask, uint32_t *group, void *stream);

/*
 * Best candidate of every group: over the n candidates with group[i] != METIS_QUERY_NO_GROUP (group[i] <
 * num_groups <= 2^24), count[g] members, cost[g] the lowest cost and first[g] the lowest position i of a member with
 * that cost (-0.0 and +0.0 are one cost), present[g] = count[g] > 0.  Exact whatever the order of the atomics.
 *   records [device] n MetisRecord (the cost is read);  group [device] n uint32
 *   count [device] num_groups uint64;  cost [device] num_groups doubles (+inf without members);
 *   first [device] num_groups int64 (-1 without members);  present [device] num_groups bytes
 */
int metis_query_groups(const MetisRecord *records, const uint32_t *group, int64_t n, int64_t num_groups,
                       uint64_t *count, double *cost, int64_t *first, uint8_t *present, void *stream);

/*
 * Stable compaction of a byte mask (metis_select.cu, the two-level pass of metis_headroom_select): the first k
 * entries i of 0..n-1 whose mask[order[i]] != 0 (order = NULL: the identity), in that order, written as order[i] (i)
 * to out [device, k uint32]; *count [host] = how many qualify.  With order = the rank permutation of
 * metis_sort_records(METIS_SORT_BY_COST_STABLE) this is a ranked selection under a filter.
 *   workspace [device] metis_headroom_workspace_bytes(n) bytes
 */
int metis_mask_select(const uint8_t *mask, const uint32_t *order, int64_t n, int64_t k, uint32_t *out, uint64_t *count,
                      void *workspace, int64_t workspace_bytes, void *stream);

/*
 * Host-side enumeration of gen_dgroups_for_stages_with_variance (search_space/device_group.py:93-107)
 * in reference order.  Writes log2 codes, num_stages bytes per row, into out (host memory) and
 * returns the number of rows, or METIS_E_CAPACITY if capacity_rows is too small (call with
 * out == NULL to count).
 */
int64_t metis_enum_device_groups(int32_t num_stages, int32_t num_gpus, double variance,
                                 int32_t max_permute_len, uint8_t *out, int64_t capacity_rows);

/*
 * The same for every stage count first_stage..last_stage in one call, one host thread per stage count
 * (what InterStagePlanGenerator regenerates block by block, search_space/plan.py:130-142).  Tables are
 * written back to back into `out` (stage count s: rows_per_stage[s-first_stage] rows of s bytes).
 * Returns the total bytes (call with out == NULL to size the buffer; a second call with the buffer
 * recomputes the tables) or METIS_E_CAPACITY.
 */
int64_t metis_enum_device_group_tables(int32_t first_stage, int32_t last_stage, int32_t num_gpus,
                                       double variance, int32_t max_permute_len, int64_t *rows_per_stage,
                                       uint8_t *out, int64_t capacity_bytes);

/*
 * Device-side generation of the device-group rows (SURVEY.md 8(f)-1).  The host lists the compositions of every
 * stage count and merges their groups (search_space/device_group.py:7-81) - thousands of compositions - and the GPU
 * writes their multiset permutations in the reference's order (search_space/utils.py:72-88): millions of rows that
 * never exist on the host or on PCIe.  One record = one slice of at most METIS_COMP_SLICE_ROWS consecutive
 * permutations of one composition (the walk is sequential, so a warp skips to its slice and writes only that).
 */
typedef struct MetisCompRec {
    int64_t row_offset;           /* byte offset of the slice's first row in the row blob                      */
    uint32_t pool_offset;         /* the composition's entry in the pool: num_groups lengths, then `stages` log2
                                     codes of the groups in sorted order (utils.py:57)                         */
    uint16_t stages;
    uint16_t num_groups;          /* merged groups (<= METIS_MAX_PERMUTE_GROUPS on the device)                 */
    uint32_t first_row;           /* permutations of the composition before this slice                        */
    uint32_t num_rows;            /* permutations in this slice                                                */
} MetisCompRec;
#define METIS_COMP_SLICE_ROWS 64
#define METIS_MAX_PERMUTE_GROUPS 32
/* host: fills recs / pool (call with recs == NULL to size: returns the number of records, *pool_bytes the
 * pool size, *max_groups the largest num_groups); rows_per_stage like metis_enum_device_group_tables */
int64_t metis_enum_compositions(int32_t first_stage, int32_t last_stage, int32_t num_gpus, double variance,
                                int32_t max_permute_len, int64_t *rows_per_stage, MetisCompRec *recs,
                                int64_t recs_capacity, uint8_t *pool, int64_t pool_capacity, int64_t *pool_bytes,
                                int32_t *max_groups);
/* device: recs / pool [device], rows [device] receives every row (same layout as metis_enum_device_group_tables) */
int metis_generate_rows(const MetisCompRec *recs, int64_t num_comps, const uint8_t *pool, uint8_t *rows, void *stream);

/*
 * Device-side listing of the compositions (SURVEY.md 8(f)-1): the same compositions, merged groups, row counts and
 * records as metis_enum_compositions, listed on the GPU one thread per composition (a composition is found from its
 * rank through a table of completion counts, so nothing walks the list), and handed out window by window: the host
 * never holds the whole list, only one window's records and pool.
 *   1. metis_list_workspace_bytes  (host only) sizes the workspace; optionally the compositions of each stage count
 *   2. metis_list_stages           lists every composition of first_stage..last_stage into the workspace and writes
 *                                  the rows of each stage count (what rows_per_stage of metis_enum_compositions holds)
 *   3. metis_list_window           for a set of row ranges, one per (stage count, rows) the window covers, writes the
 *                                  window's records and pool (call with recs == NULL to size)
 * A window's rows are its ranges back to back, in the order given: a record's row_offset is relative to that layout,
 * its pool_offset to the window's own pool.  The records of a range are metis_enum_compositions' slices cut to the
 * range (first_row = offset of the slice's first row inside the composition).  The workspace of step 2 must be kept,
 * unchanged, for step 3.
 */
typedef struct MetisListing {
    int32_t first_stage;          /* stage counts first_stage .. last_stage (last_stage <= METIS_MAX_STAGES)      */
    int32_t last_stage;
    int32_t num_gpus;
    int32_t max_permute_len;
    double variance;              /* --min_group_scale_variance                                                  */
    int32_t max_ranges;           /* most row ranges of one metis_list_window call                               */
    int32_t reserved;
} MetisListing;

typedef struct MetisRowRange {
    int32_t stages;               /* stage count of the range                                                    */
    int32_t reserved;
    int64_t first_row;            /* rows [first_row, end_row) of the stage count's table                        */
    int64_t end_row;
} MetisRowRange;

/* host: bytes of device workspace for `listing` (METIS_E_ARG when it cannot be listed); comps_per_stage [host],
 * optional: last_stage - first_stage + 1 int64, the compositions of each stage count */
int64_t metis_list_workspace_bytes(const MetisListing *listing, int64_t *comps_per_stage);
/* rows_per_stage [host] last_stage - first_stage + 1 int64; max_groups [host] the most merged groups of any
 * composition (a composition above METIS_MAX_PERMUTE_GROUPS is counted but never written as a record) */
int metis_list_stages(const MetisListing *listing, void *workspace, int64_t workspace_bytes, int64_t *rows_per_stage,
                      int32_t *max_groups, void *stream);
/* ranges [host] num_ranges <= listing->max_ranges; recs / pool [device] or NULL; sizes [host] 3 int64: records, pool
 * bytes, status (0 = written; bit 0: a range outside its stage count's table, bit 1: a composition of more than
 * METIS_MAX_PERMUTE_GROUPS merged groups in a range (its records are not written), bit 2: recs / pool too small
 * (nothing written)) */
int metis_list_window(const MetisListing *listing, void *workspace, int64_t workspace_bytes, const MetisRowRange *ranges,
                      int32_t num_ranges, MetisCompRec *recs, int64_t recs_capacity, uint8_t *pool,
                      int64_t pool_capacity, int64_t *sizes, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* METIS_B200_H */
