// metis_warp.cuh - WarpCoop, the lane policy of the chain kernel (metis_search.cu, het_chain_kernel): one warp
// evaluates one plan with CoopEvaluator (metis_coop.cuh).  In a header of its own so that a test-only device build
// (tests/devsim) runs the very primitives the search runs.
#pragma once

#include <cuda_runtime.h>

#include "metis_coop.cuh"

namespace metis {

// Lane policy of the chain kernel (metis_coop.cuh): 32 lanes, leader = lane 0, __syncwarp between sections.
#ifdef METIS_PROFILE_PHASES
__device__ long long g_mark_acc[64];   // cycles per phase of the chain evaluator (leader lane)
#endif
struct WarpCoop {
#ifdef METIS_PROFILE_PHASES
    mutable long long t_last = 0;
    mutable int cur = 0;
    __device__ void mark(int id) const {
        if ((threadIdx.x & 31) != 0) return;
        const long long now = clock64();
        if (t_last) atomicAdd((unsigned long long *)&g_mark_acc[cur & 31], (unsigned long long)(now - t_last));
        cur = id; t_last = now;
    }
#else
    __device__ void mark(int) const {}
#endif
    __device__ void note(int) const {}         // balancer path taken (BalancerPath; recorded by tests/devsim only)
    // Start of every balancer run: meet the other warps of the block.  The 16 warps of a block walk different plans
    // through the same 55 KB of live code; left alone they spread over all its phases and miss the instruction cache
    // (icc hit rate 70 %, `no_instruction` the largest stall).  Starting each run together keeps them within a phase
    // or two of each other: measured 4.25 -> 3.93 ms on BASELINE configs[2] although every run now waits for the
    // slowest neighbour (16 warps evaluating the SAME plan, perfectly aligned, gain 17 %).  A warp that is out of
    // work keeps answering the barrier (het_chain_kernel) until nobody in the block works any more.
    // PTX named barrier 1 over the whole block with an OR reduction: arrivals from different program points (this gate
    // and the drain loop of het_chain_kernel) meet at the same barrier, which PTX defines (`bar.red`, all lanes of a
    // warp arrive together) and CUDA C++'s __syncthreads_or does not promise.
    // (one copy of the instruction, out of line: both callers arrive at the same program point)
    static __device__ __noinline__ int block_or(int pred) {
        int any;
        asm volatile("{\n\t.reg .pred p, q;\n\tsetp.ne.s32 q, %1, 0;\n\tbar.red.or.pred p, 1, %2, q;\n\tselp.s32 %0, 1, 0, p;\n\t}"
                     : "=r"(any) : "r"(pred), "r"((int)blockDim.x) : "memory");
        return any;
    }
    __device__ void gate() const { block_or(1); }
    __device__ int lane() const { return threadIdx.x & 31; }
    __device__ int width() const { return 32; }
    __device__ bool leader() const { return (threadIdx.x & 31) == 0; }
    __device__ void sync() const { __syncwarp(); }
    __device__ bool any(bool p) const { return __any_sync(0xFFFFFFFFu, p); }
    __device__ unsigned ballot(bool p) const { return __ballot_sync(0xFFFFFFFFu, p); }
    __device__ unsigned match_any(int v) const { return __match_any_sync(0xFFFFFFFFu, v); }
    // the crossing inside the 32-entry window P[i0 .. i0 + 31]?  (one load and one ballot; see OneLane::first_ge_window)
    __device__ int first_ge_window(const double *P, int n, int i0, int lo, double t) const {
        const int idx = i0 + (threadIdx.x & 31);
        const unsigned m = __ballot_sync(0xFFFFFFFFu, idx <= n && P[idx] >= t);
        if (m == 0u || ((m & 1u) && i0 > lo)) return -1;
        return i0 + __ffs(m) - 1;
    }
    // first i in [0, n] with P[i] >= t (P ascending, shared memory), n + 1 if none: 32-ary search by the whole warp
    __device__ __noinline__ int first_ge(const double *P, int n, double t) const {
        const unsigned full = 0xFFFFFFFFu;
        const int lane = threadIdx.x & 31;
        const int G = (n + 32) >> 5;                          // entries per lane group: ceil((n + 1) / 32)
        int ci = lane * G + G - 1;                            // last entry of this lane's group
        if (ci > n) ci = n;
        const unsigned m1 = __ballot_sync(full, P[ci] >= t);
        if (m1 == 0u) return n + 1;
        const int g0 = (__ffs(m1) - 1) * G;                   // the first group whose last entry reaches t holds the answer
#pragma unroll 1
        for (int off = 0; off < G; off += 32) {
            const int idx = g0 + off + lane;
            const unsigned m2 = __ballot_sync(full, off + lane < G && idx <= n && P[idx] >= t);
            if (m2) return g0 + off + __ffs(m2) - 1;
        }
        return n + 1;
    }
    __device__ int bcast_last(int v) const { return __shfl_sync(0xFFFFFFFFu, v, 31); }
    // Reductions with REDUX (one instruction per 32-bit max / min over the warp) on an order-preserving integer
    // image of the double (-0.0 and +0.0 share one key, like ==); no NaN reaches these.
    static __device__ __forceinline__ unsigned long long dkey(double v) {
        unsigned long long u = (unsigned long long)__double_as_longlong(v);
        if ((u << 1) == 0ULL) u = 0ULL;                      // -0.0 -> +0.0
        return u ^ ((u >> 63) ? ~0ULL : 0x8000000000000000ULL);
    }
    static __device__ __forceinline__ double dkey_inv(unsigned long long k) {
        const unsigned long long u = k ^ ((k >> 63) ? 0x8000000000000000ULL : ~0ULL);
        return __longlong_as_double((long long)u);
    }
    static __device__ __forceinline__ unsigned long long kmax(unsigned long long key, bool &mine) {
        const unsigned full = 0xFFFFFFFFu;
        const unsigned hi = (unsigned)(key >> 32), lo = (unsigned)key;
        const unsigned mh = __reduce_max_sync(full, hi);
        const bool c1 = hi == mh;
        const unsigned ml = __reduce_max_sync(full, c1 ? lo : 0u);
        mine = c1 && lo == ml;
        return ((unsigned long long)mh << 32) | ml;
    }
    __device__ void argmax_first(double &v, int &i) const {  // largest v, lowest index among equals
        bool mine;
        const unsigned long long k = kmax(dkey(v), mine);
        i = (int)__reduce_min_sync(0xFFFFFFFFu, mine ? (unsigned)i : 0xFFFFFFFFu);
        v = dkey_inv(k);
    }
    __device__ void argmin_first(double &v, int &i) const {  // smallest v, lowest index among equals
        bool mine;
        const unsigned long long k = ~kmax(~dkey(v), mine);
        i = (int)__reduce_min_sync(0xFFFFFFFFu, mine ? (unsigned)i : 0xFFFFFFFFu);
        v = dkey_inv(k);
    }
    __device__ void imax_first(int &v, int &i) const {
        const int m = __reduce_max_sync(0xFFFFFFFFu, v);
        i = (int)__reduce_min_sync(0xFFFFFFFFu, v == m ? (unsigned)i : 0xFFFFFFFFu);
        v = m;
    }
    __device__ void imin_first(int &v, int &i) const {
        const int m = __reduce_min_sync(0xFFFFFFFFu, v);
        i = (int)__reduce_min_sync(0xFFFFFFFFu, v == m ? (unsigned)i : 0xFFFFFFFFu);
        v = m;
    }
    __device__ double max_all(double v) const {
        bool mine;
        return dkey_inv(kmax(dkey(v), mine));
    }
    __device__ __noinline__ int incl_scan(int v) const {
        const int lane = threadIdx.x & 31;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int u = __shfl_up_sync(0xFFFFFFFFu, v, d);
            if (lane >= d) v += u;
        }
        return v;
    }
    __device__ int last_lane(int v) const { return __shfl_sync(0xFFFFFFFFu, v, 31); }
};

}  // namespace metis
