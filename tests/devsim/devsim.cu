// devsim.cu - TEST-ONLY device build of the layer balancer forms and of the WarpCoop lane primitives.
//
// The GPU counterpart of tests/hostsim: the search runs LayerComputeBalancer.run in three forms (balance_run with
// Serial in the replay kernels, balance_run with Lockstep in the bulk round, CoopEvaluator::balance_coop with WarpCoop
// in the chain kernel), and only inside whole searches do the last two meet inputs.  This library runs each form on
// caller-chosen capacity rows, with the scratch where the search keeps it, and reports which of the balancer's paths
// (BalancerPath, metis_eval.cuh) every row took.  Built and loaded only by tests/devsim_util.py with the library's
// own nvcc flags; the metis_b200 package never loads it.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include "../../metis_b200/csrc/metis_eval.cuh"
#include "../../metis_b200/csrc/metis_coop.cuh"
#include "../../metis_b200/csrc/metis_warp.cuh"

using namespace metis;

namespace {

// the product policies, plus a record of the paths taken (bit p of *notes = BalancerPath p)
struct NoteSerial : Serial {
    unsigned *notes;
    __device__ void note(int p) const { *notes |= 1u << p; }
};
struct NoteLockstep : Lockstep {
    unsigned *notes;
    __device__ void note(int p) const { *notes |= 1u << p; }
};
struct NoteWarp : WarpCoop {
    unsigned *notes;                        // the warp's word in shared memory; note() is called by all lanes alike
    __device__ void note(int p) const { if (leader()) *notes |= 1u << p; }
};

// the derived tables of a minimal problem (no keys, batch sizes or tp), entry by entry as pack_tables_kernel does
__global__ void derive_kernel(MetisProblem p, const double *norm_lc, double *derived) {
    const double bw[1] = {1.0};
    const DerivedLayout d = derived_layout(p);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < d.total; i += gridDim.x * blockDim.x)
        derived[i] = derive_entry(p, d, norm_lc, nullptr, bw, i);
}

__device__ Tables balancer_tables(const MetisProblem &p, const double *norm_lc, const double *derived) {
    Tables T;
    memset(&T, 0, sizeof(T));
    T.p = p;
    T.norm_lc = norm_lc;
    bind_derived(T, derived);
    return T;
}

struct Rows {
    const double *capa;
    const int32_t *ns;
    long long n;
    int stride;
    uint16_t *part;      // [n][stride + 1]
    int32_t *rc;         // METIS_FATAL_* per row
    uint32_t *notes;     // BalancerPath bits per row
    int32_t *block;      // length of the middle block (coop only; -1 elsewhere)
};

__device__ void store(const Rows &r, long long i, int S, int rc, unsigned notes, int block, const uint16_t *part) {
    r.rc[i] = rc;
    r.notes[i] = notes;
    r.block[i] = block;
    if (rc == 0)
        for (int s = 0; s <= S; ++s) r.part[i * (r.stride + 1) + s] = part[s];
}

// Serial: one thread per row, per-thread scratch (as layer_balance_kernel and the replay kernels)
template <int MAXS, int MAXL>
__global__ void serial_kernel(MetisProblem p, const double *lc, const double *derived, Rows r) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= r.n) return;
    const Tables T = balancer_tables(p, lc, derived);
    Scratch<MAXS, MAXL> w;
    const int S = r.ns[i];
    for (int s = 0; s < S; ++s) w.perf[s] = r.capa[i * r.stride + s];
    unsigned notes = 0;
    NoteSerial x;
    x.notes = &notes;
    const int rc = balance_run<MAXS, MAXL>(T, S, w, x);
    store(r, i, S, rc, notes, -1, w.part);
}

// Lockstep: 32 rows per warp, per-thread scratch, lanes re-joined around the run as in first_task (het_first_kernel)
template <int MAXS, int MAXL>
__global__ void lockstep_kernel(MetisProblem p, const double *lc, const double *derived, Rows r) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const Tables T = balancer_tables(p, lc, derived);
    Scratch<MAXS, MAXL> w;
    const bool has = i < r.n;
    const int S = has ? r.ns[i] : 0;
    for (int s = 0; s < S; ++s) w.perf[s] = r.capa[i * r.stride + s];
    unsigned notes = 0;
    NoteLockstep x;
    x.notes = &notes;
    x.rejoin(has);
    int rc = 0;
    if (has) rc = balance_run<MAXS, MAXL>(T, S, w, x);
    x.rejoin(true);
    if (has) store(r, i, S, rc, notes, -1, w.part);
}

template <int MAXS, int MAXL>
struct alignas(16) WarpScratch {
    Scratch<MAXS, MAXL> w;
    CoopMail mail;
    unsigned notes;
};

// Coop: one row per warp, CoopEvaluator::balance_coop on WarpCoop, scratch in shared memory (as het_chain_kernel)
template <int MAXS, int MAXL>
__global__ void coop_kernel(MetisProblem p, const double *lc, const double *derived, Rows r) {
    extern __shared__ __align__(16) uint8_t smem[];
    const long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (i >= r.n) return;                                    // whole warps leave together
    const Tables T = balancer_tables(p, lc, derived);
    WarpScratch<MAXS, MAXL> *ws = reinterpret_cast<WarpScratch<MAXS, MAXL> *>(smem) + (threadIdx.x >> 5);
    NoteWarp lanes;
    lanes.notes = &ws->notes;
    CoopEvaluator<MAXS, MAXL, NoteWarp> ev(T, ws->w, ws->mail, lanes);
    const int S = r.ns[i];
    ev.pd.S = S;
    for (int s = lanes.lane(); s < S; s += 32) ws->w.perf[s] = r.capa[i * r.stride + s];
    if (lanes.leader()) ws->notes = 0;
    __syncwarp();
    const int rc = ev.balance_coop();
    __syncwarp();
    if (lanes.leader()) {
        const int block = rc ? -1 : (ws->mail.m > ws->mail.k ? ws->mail.m - ws->mail.k : 0);
        store(r, i, S, rc, ws->notes, block, ws->w.part);
    }
}

template <int MAXS, int MAXL>
cudaError_t launch_balance(int policy, const MetisProblem &p, const double *lc, const double *derived, const Rows &r) {
    const int blocks = (int)((r.n + 127) / 128);
    if (policy == 0) serial_kernel<MAXS, MAXL><<<blocks, 128>>>(p, lc, derived, r);
    else if (policy == 1) lockstep_kernel<MAXS, MAXL><<<blocks, 128>>>(p, lc, derived, r);
    else {
        const int warps = 4;
        const size_t smem = warps * sizeof(WarpScratch<MAXS, MAXL>);
        cudaError_t e = cudaFuncSetAttribute(coop_kernel<MAXS, MAXL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        coop_kernel<MAXS, MAXL><<<(int)((r.n + warps - 1) / warps), warps * 32, smem>>>(p, lc, derived, r);
    }
    return cudaGetLastError();
}

// ---- WarpCoop primitives, one query per warp ----
enum LaneOp { kArgmax = 0, kArgmin, kImax, kImin, kMaxAll, kInclScan, kFirstGe, kFirstGeWindow, kBcastLast };

struct LaneQueries {
    int op;
    long long nq;
    const double *dv;      // [nq][32] per-lane doubles
    const int32_t *iv;     // [nq][32] per-lane ints
    const double *P;       // concatenated ascending arrays
    const int64_t *poff;   // [nq] offset of the query's array in P
    const int32_t *pn;     // [nq] n: the array holds P[0 .. n]
    const double *t;       // [nq]
    const int32_t *i0, *lo;
    double *od;            // [nq][32]
    int32_t *oi;           // [nq][32]
};

__global__ void lanes_kernel(LaneQueries q) {
    const long long k = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (k >= q.nq) return;
    const int lane = threadIdx.x & 31;
    const WarpCoop x;
    double v = q.dv[k * 32 + lane];
    int iv = q.iv[k * 32 + lane];
    int ri = 0;
    switch (q.op) {
    case kArgmax: x.argmax_first(v, iv); ri = iv; break;
    case kArgmin: x.argmin_first(v, iv); ri = iv; break;
    case kImax: { int m = (int)q.dv[k * 32 + lane]; x.imax_first(m, iv); v = m; ri = iv; } break;
    case kImin: { int m = (int)q.dv[k * 32 + lane]; x.imin_first(m, iv); v = m; ri = iv; } break;
    case kMaxAll: v = x.max_all(v); break;
    case kInclScan: ri = x.incl_scan(iv); break;
    case kFirstGe: ri = x.first_ge(q.P + q.poff[k], q.pn[k], q.t[k]); break;
    case kFirstGeWindow: ri = x.first_ge_window(q.P + q.poff[k], q.pn[k], q.i0[k], q.lo[k], q.t[k]); break;
    case kBcastLast: ri = x.bcast_last(iv); break;
    }
    q.od[k * 32 + lane] = v;
    q.oi[k * 32 + lane] = ri;
}

template <class V>
cudaError_t upload(V **dst, const V *src, size_t n) {
    cudaError_t e = cudaMalloc((void **)dst, (n ? n : 1) * sizeof(V));
    if (e == cudaSuccess && n) e = cudaMemcpy(*dst, src, n * sizeof(V), cudaMemcpyHostToDevice);
    return e;
}

}  // namespace

extern "C" {

// Runs one balancer form over n rows (capa[i][0 .. ns[i]), shared lc[0 .. norm_len) and num_layers) in the scratch of
// instantiation <maxs, maxl>.  policy: 0 Serial, 1 Lockstep, 2 Coop.  Returns 0, -1 for an unknown policy / tier /
// a row beyond the tier, or the CUDA error code.
int devsim_balance(int policy, int maxs, int maxl, const double *capa, const int32_t *ns, int64_t n, int32_t stride,
                   const double *lc, int32_t norm_len, int32_t num_layers, uint16_t *part, int32_t *rc,
                   uint32_t *notes, int32_t *block) {
    if (policy < 0 || policy > 2 || num_layers > maxl || n < 1) return -1;
    for (int64_t i = 0; i < n; ++i)
        if (ns[i] < 1 || ns[i] > maxs || ns[i] > stride) return -1;
    MetisProblem p;
    memset(&p, 0, sizeof(p));
    p.num_layers = num_layers;
    p.norm_len = norm_len;
    const int total = derived_layout(p).total;
    double *d_capa = nullptr, *d_lc = nullptr, *d_der = nullptr;
    int32_t *d_ns = nullptr, *d_rc = nullptr, *d_block = nullptr;
    uint16_t *d_part = nullptr;
    uint32_t *d_notes = nullptr;
    cudaError_t e = upload(&d_capa, capa, (size_t)n * stride);
    if (e == cudaSuccess) e = upload(&d_ns, ns, (size_t)n);
    if (e == cudaSuccess) e = upload(&d_lc, lc, (size_t)norm_len);
    if (e == cudaSuccess) e = cudaMalloc((void **)&d_der, (size_t)(total ? total : 1) * sizeof(double));
    if (e == cudaSuccess) e = cudaMalloc((void **)&d_part, (size_t)n * (stride + 1) * sizeof(uint16_t));
    if (e == cudaSuccess) e = cudaMalloc((void **)&d_rc, (size_t)n * sizeof(int32_t));
    if (e == cudaSuccess) e = cudaMalloc((void **)&d_notes, (size_t)n * sizeof(uint32_t));
    if (e == cudaSuccess) e = cudaMalloc((void **)&d_block, (size_t)n * sizeof(int32_t));
    if (e == cudaSuccess) e = cudaMemset(d_part, 0, (size_t)n * (stride + 1) * sizeof(uint16_t));
    if (e == cudaSuccess) {
        derive_kernel<<<8, 256>>>(p, d_lc, d_der);
        e = cudaGetLastError();
    }
    int bad_tier = 0;
    if (e == cudaSuccess) {
        const Rows r{d_capa, d_ns, (long long)n, stride, d_part, d_rc, d_notes, d_block};
        if (maxs == 64 && maxl == 128) e = launch_balance<64, 128>(policy, p, d_lc, d_der, r);
        else if (maxs == 96 && maxl == 128) e = launch_balance<96, 128>(policy, p, d_lc, d_der, r);
        else if (maxs == 128 && maxl == 256) e = launch_balance<128, 256>(policy, p, d_lc, d_der, r);
        else bad_tier = 1;
    }
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e == cudaSuccess && !bad_tier) {
        e = cudaMemcpy(part, d_part, (size_t)n * (stride + 1) * sizeof(uint16_t), cudaMemcpyDeviceToHost);
        if (e == cudaSuccess) e = cudaMemcpy(rc, d_rc, (size_t)n * sizeof(int32_t), cudaMemcpyDeviceToHost);
        if (e == cudaSuccess) e = cudaMemcpy(notes, d_notes, (size_t)n * sizeof(uint32_t), cudaMemcpyDeviceToHost);
        if (e == cudaSuccess) e = cudaMemcpy(block, d_block, (size_t)n * sizeof(int32_t), cudaMemcpyDeviceToHost);
    }
    cudaFree(d_capa); cudaFree(d_ns); cudaFree(d_lc); cudaFree(d_der);
    cudaFree(d_part); cudaFree(d_rc); cudaFree(d_notes); cudaFree(d_block);
    if (bad_tier) return -1;
    return e == cudaSuccess ? 0 : (int)e;
}

// Runs WarpCoop primitive `op` (LaneOp) on nq queries, one warp each.  Per query: 32 lane doubles dv and ints iv
// (imax_first / imin_first take their int values from dv), and for the searches the ascending array
// P[poff .. poff + pn] with t, i0, lo.  Every lane's result goes to od / oi.  Returns 0 or the CUDA error code.
int devsim_lanes(int op, int64_t nq, const double *dv, const int32_t *iv, const double *P, int64_t plen,
                 const int64_t *poff, const int32_t *pn, const double *t, const int32_t *i0, const int32_t *lo,
                 double *od, int32_t *oi) {
    LaneQueries q;
    memset(&q, 0, sizeof(q));
    q.op = op;
    q.nq = nq;
    double *d_dv = nullptr, *d_P = nullptr, *d_t = nullptr, *d_od = nullptr;
    int32_t *d_iv = nullptr, *d_pn = nullptr, *d_i0 = nullptr, *d_lo = nullptr, *d_oi = nullptr;
    int64_t *d_poff = nullptr;
    cudaError_t e = upload(&d_dv, dv, (size_t)nq * 32);
    if (e == cudaSuccess) e = upload(&d_iv, iv, (size_t)nq * 32);
    if (e == cudaSuccess) e = upload(&d_P, P, (size_t)plen);
    if (e == cudaSuccess) e = upload(&d_poff, poff, (size_t)nq);
    if (e == cudaSuccess) e = upload(&d_pn, pn, (size_t)nq);
    if (e == cudaSuccess) e = upload(&d_t, t, (size_t)nq);
    if (e == cudaSuccess) e = upload(&d_i0, i0, (size_t)nq);
    if (e == cudaSuccess) e = upload(&d_lo, lo, (size_t)nq);
    if (e == cudaSuccess) e = cudaMalloc((void **)&d_od, (size_t)nq * 32 * sizeof(double));
    if (e == cudaSuccess) e = cudaMalloc((void **)&d_oi, (size_t)nq * 32 * sizeof(int32_t));
    if (e == cudaSuccess) {
        q.dv = d_dv; q.iv = d_iv; q.P = d_P; q.poff = d_poff; q.pn = d_pn; q.t = d_t; q.i0 = d_i0; q.lo = d_lo;
        q.od = d_od; q.oi = d_oi;
        lanes_kernel<<<(int)((nq + 3) / 4), 128>>>(q);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e == cudaSuccess) e = cudaMemcpy(od, d_od, (size_t)nq * 32 * sizeof(double), cudaMemcpyDeviceToHost);
    if (e == cudaSuccess) e = cudaMemcpy(oi, d_oi, (size_t)nq * 32 * sizeof(int32_t), cudaMemcpyDeviceToHost);
    cudaFree(d_dv); cudaFree(d_iv); cudaFree(d_P); cudaFree(d_poff); cudaFree(d_pn); cudaFree(d_t);
    cudaFree(d_i0); cudaFree(d_lo); cudaFree(d_od); cudaFree(d_oi);
    return e == cudaSuccess ? 0 : (int)e;
}

}  // extern "C"
