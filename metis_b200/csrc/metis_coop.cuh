// metis_coop.cuh - one warp evaluates one inter-stage plan's whole strategy chain (SURVEY.md 8a rows a5-a16).
//
// The chain of a plan (search_space/plan.py:192-268) is sequential: strategy k+1 is chosen from the memory state
// that the partition of strategy k produced, and a partition attempt replays LayerComputeBalancer.run
// (model/load_balancer.py:197-207) whose passes are compare-and-subtract chains in fp64.  What a warp can do in
// parallel is everything that is independent per stage or per layer: profile look-ups, range sums, the 7-way
// vote, arg-max / arg-min reductions, prefix sums.  The execution model is explicit and does not depend on how
// the hardware schedules the lanes of a warp:
//
//   PAR  sections  - a loop over stages / layers strided over the lanes (x.lane(), x.width()); iteration i only
//                    writes scratch entries with index i, and reads nothing that another iteration of the same
//                    section writes;
//   SEQ  sections  - executed by the leader lane alone (x.leader()); results leave the section through the
//                    scratch (w.*), never through registers;
//   x.sync()       - __syncwarp() between any two sections that communicate through the scratch;
//   reductions     - register values are combined with shuffles (x.argmax_first, x.argmin_first, x.max_all,
//                    x.any, x.incl_scan), whose result is identical in every lane.
//
// Control flow outside SEQ sections is uniform (every lane takes the same branches because the conditions are
// reduction results or values read from the scratch after a sync).
//
// The per-stage helpers of PlanEvaluator (metis_eval.cuh: mixed-type stages, bandwidth selection, memory
// capacity) are reused unchanged: inside a PAR section the lane that owns the stage calls them on its own copy
// of the evaluator.  Plain C++ (the policy supplies the warp primitives) so that tests/hostsim can compile the
// same source with g++; the host policy has one lane and can visit the PAR iterations in reverse order, which
// catches a dependence between iterations without a GPU.
#pragma once

#include "metis_eval.cuh"

namespace metis {

// Scalars a SEQ section hands to the following sections (per-warp scratch next to Scratch<>).
struct CoopMail {
    int m;        // first sub-layer of the backward tail (LayerComputeBalancer state)
    int err;      // METIS_FATAL_* raised inside a SEQ section
    int flag;     // generic boolean result
    int pad;
    double val;   // generic fp64 result (totals)
    double val2;
    int k;        // end of the forward pass: first sub-layer not offered to a forward stage
    int s_top;    // last stage the forward pass touched
    int top_skip; // 1 = that stage closed on a non-fitting sub-layer
    int pad2;
};

// Host / test policy: one lane.  `reverse` visits PAR iterations last-to-first.
struct OneLane {
    bool reverse = false;
    MB_HD int lane() const { return 0; }
    MB_HD int width() const { return 1; }
    MB_HD bool leader() const { return true; }
    MB_HD void sync() const {}
    MB_HD bool any(bool p) const { return p; }
    MB_HD unsigned ballot(bool p) const { return p ? 1u : 0u; }
    MB_HD unsigned match_any(int) const { return 1u; }
    // the same, looking only at P[i0 .. i0 + 31] (clipped to n): the index if the crossing lies inside the window
    // (P[i0] < t <= P[i] or i0 == lo), -1 if the window cannot tell
    MB_HD int first_ge_window(const double *P, int n, int i0, int lo, double t) const {
        for (int k = 0; k < 32 && i0 + k <= n; ++k)
            if (P[i0 + k] >= t) return (k > 0 || i0 <= lo) ? i0 + k : -1;
        return -1;
    }
    // first i in [0, n] with P[i] >= t (P ascending), n + 1 if none
    MB_HD int first_ge(const double *P, int n, double t) const {
        int lo = 0, hi = n + 1;
        while (lo < hi) { const int mid = (lo + hi) >> 1; if (P[mid] >= t) hi = mid; else lo = mid + 1; }
        return lo;
    }
    MB_HD int bcast_last(int v) const { return v; }
    MB_HD void argmax_first(double &, int &) const {}
    MB_HD void argmin_first(double &, int &) const {}
    MB_HD void imax_first(int &, int &) const {}
    MB_HD void imin_first(int &, int &) const {}
    MB_HD double max_all(double v) const { return v; }
    MB_HD int incl_scan(int v) const { return v; }
    MB_HD int last_lane(int v) const { return v; }
    MB_HD void mark(int) const {}
    MB_HD void note(int) const {}
    MB_HD void gate() const {}
};

// index of PAR iteration number `i` (0-based count of this lane's iterations) - lets the host policy reverse
template <class X>
MB_HD int par_index(const X &, int i, int n) { (void)n; return i; }
MB_HD int par_index(const OneLane &x, int i, int n) { return x.reverse ? n - 1 - i : i; }

#define METIS_PAR(x, var, n) \
    for (int var##_i = (x).lane(), var = par_index((x), var##_i, (n)); var##_i < (n); \
         var##_i += (x).width(), var = par_index((x), var##_i, (n)))

// ---------------------------------------------------------------------------------------------------------
// Sequential pieces of LayerComputeBalancer.run (model/load_balancer.py:216-287) for the leader lane: the
// compare-and-subtract chains in fp64.  Same state encoding as balance_run in metis_eval.cuh (fe[] interval ends
// with kBroke / kTaken, lstk[], the per-layer packed stage map subw[]).
// ---------------------------------------------------------------------------------------------------------
struct FillState {
    int k;          // first sub-layer not offered to a forward stage
    int s_top;      // last stage the forward pass touched (-1: none)
    bool top_skip;  // that stage closed on a non-fitting sub-layer
};

// forward pass (:216-231): stage s takes sub-layers while its capacity exceeds the next demand (strict compare,
// every subtraction rounded like the reference's) and closes on the first one that does not fit, which is skipped.
// Only the interval ends fe[] and the residual capacities are written; which stage owns a sub-layer follows from
// fe[] (CoopEvaluator::vote_coop), so the loop body is a compare and a subtract.
template <int MAXS, int MAXL>
MB_HD_NOINLINE FillState seq_forward(const Tables &T, int S, Scratch<MAXS, MAXL> &w) {
    const int L = T.p.num_layers;
    const double *dlay = T.dlay;
    const int N = kH * L;
    const int lim = (N - 1 - kH) > 0 ? (N - 1 - kH) : 0;   // :218
    const int last = S - 1;
    FillState st{0, -1, false};
    if (S > 1) {
        int s = 0, j = 0;
        double c = w.capa[0];
        bool done = false;
#pragma unroll 1
        for (int r = 0; r + 1 < L && !done; ++r) {
            const double d = dlay[r];
            const int nsub = (r == L - 2) ? kH - 1 : kH;     // the last 8 sub-layers are reserved
            if (nsub == kH && c > 9.0 * d) {
                // whole layer fits with room to spare: all seven compare-and-subtract steps take the "fits"
                // branch (c - 7d > d even after rounding), so only the subtractions remain
                c -= d; c -= d; c -= d; c -= d; c -= d; c -= d; c -= d;
                j += kH;
                continue;
            }
#pragma unroll
            for (int q = 0; q < kH; ++q) {
                if (q < nsub && !done) {
                    if (c > d) {
                        c -= d;
                    } else {                                     // sub-layer j + q does not fit: skipped, stage closes
                        w.capa[s] = c;
                        w.fe[s] = (uint16_t)((j + q) | kBroke);
                        ++s;
                        if (s >= last) done = true;
                        else c = w.capa[s];
                    }
                }
            }
            j += nsub;
        }
        if (s < last) {                                          // ran into the reserved tail
            w.capa[s] = c;
            w.fe[s] = (uint16_t)lim;
#pragma unroll 1
            for (int t = s + 1; t < last; ++t) w.fe[t] = (uint16_t)lim;
            st.k = lim;
            st.s_top = s;
        } else {
            st.k = (w.fe[last - 1] & kPos) + 1;
            st.s_top = last - 1;
            st.top_skip = true;
        }
    }
    return st;
}

// backward pass (:233-249): the last stage takes a contiguous tail [m, N); returns m
template <int MAXS, int MAXL>
MB_HD_NOINLINE int seq_backward(const Tables &T, int S, Scratch<MAXS, MAXL> &w, int k) {
    const int L = T.p.num_layers;
    const double *dlay = T.dlay;
    const int N = kH * L;
    const int last = S - 1;
    double c = w.capa[last];
    int r = L - 1;
    double d = dlay[r];
#pragma unroll 1
    for (int i = 0; i < kH; ++i) c -= d;                    // unconditional while len < hallucination (:237-241)
    int m = N - kH;
    // above k every sub-layer is unassigned: only the capacity test of :246 decides (layer by layer, top down)
    bool full = false;
#pragma unroll 1
    while (m > k && !full) {
        --r;
        d = dlay[r];
        const int floor_j = kH * r > k ? kH * r : k;        // lowest sub-layer of this layer that is still >= k
#pragma unroll 1
        while (m > floor_j) {
            if (!(c > d)) { full = true; break; }            // :246 fails; every later id fails :243
            c -= d;
            --m;
        }
    }
    if (!full) {                                            // reached k: below it only skipped sub-layers are unassigned
        int sp = S - 2;
#pragma unroll 1
        while (m > 0) {
            const int j = m - 1;
#pragma unroll 1
            while (sp >= 0 && (!(w.fe[sp] & kBroke) || (int)(w.fe[sp] & kPos) > j)) --sp;
            if (!(sp >= 0 && (int)(w.fe[sp] & kPos) == j)) break;   // (layer_id + 1) != min(...) from here on (:243)
            const double dj = dlay[j / kH];
            if (!(c > dj)) break;
            c -= dj;
            m = j;
            w.fe[sp] |= kTaken;
        }
    }
    w.capa[last] = c;
    return m;
}

// leftovers (:251-287), first part: the skipped sub-layers, ascending - general sequential form (any geometry:
// empty stages, stages that already hold a leftover).  get_proper_stage: lo = stage of the largest assigned id
// below j whose stage holds nothing above j, hi = stage of the smallest assigned id above j whose stage holds
// nothing below j.
template <int MAXS, int MAXL>
MB_HD_NOINLINE int seq_skipped(const Tables &T, int S, Scratch<MAXS, MAXL> &w) {
    const double *dlay = T.dlay;
    const int last = S - 1;
    int start = 0;                                        // first sub-layer of stage s's forward interval
#pragma unroll 1
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
#pragma unroll 1
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
#pragma unroll 1
            while (hi < last && (!fwd_nonempty(w, hi) || w.got[hi])) ++hi;
        }
        if (lo > hi) return METIS_FATAL_SCRATCH;
        int pick = lo;
        double best = w.capa[lo];
#pragma unroll 1
        for (int t = lo + 1; t <= hi; ++t)
            if (w.capa[t] > best) { best = w.capa[t]; pick = t; }
        w.capa[pick] -= dlay[j / kH];
        w.lstk[s] = (uint8_t)pick;
        w.got[pick] = 1;
        start = next_start;
    }
    return METIS_FATAL_NONE;
}

// lower end of get_proper_stage's range for the first sub-layer of the middle block [k, m) (:252-275): the stage
// holding the largest assigned id below k (forward intervals and placed skipped sub-layers all lie below it)
template <int MAXS, int MAXL>
MB_HD int middle_lo(int S, const Scratch<MAXS, MAXL> &w, const FillState &st) {
    const int last = S - 1;
    if (st.s_top < 0) return 0;
#pragma unroll 1
    for (int u = st.s_top;; --u) {
        if (u < st.s_top || st.top_skip) {
            const uint16_t eu = w.fe[u];
            if ((eu & (kBroke | kTaken)) == kBroke) {
                const int t2 = w.lstk[u];
                if (t2 != last) return t2;
            }
        }
        if (fwd_nonempty(w, u)) return u;
        if (u == 0) break;
    }
    return 0;
}

// CPython sum() of w-resident values v[0..n) in index order, for the leader lane (unrolled by 4: the loop overhead
// was a third of its instructions; measured -2 % on the whole search)
MB_HD_NOINLINE double seq_py_sum(const double *v, int n) {
    if (n <= 0) return 0.0;
    double f = 0.0 + v[0], c = 0.0;
#pragma unroll 4
    for (int i = 1; i < n; ++i) {
        const double x = v[i];
        const double t = f + x;
        if (fabs(f) >= fabs(x)) c += (f - t) + x;
        else c += (x - t) + f;
        f = t;
    }
    if (c != 0.0 && isfinite(c)) f += c;
    return f;
}

// ---------------------------------------------------------------------------------------------------------
// The chain evaluator.  One instance per lane (registers); `w` and `mail` are the warp's shared scratch.
// ---------------------------------------------------------------------------------------------------------
// ONE = the cluster has a single device type (compile-time: the mixed-type paths are not even instantiated,
// which halves the code the warps of an SM compete for in the instruction cache)
template <int MAXS, int MAXL, class X, bool ONE = false>
struct CoopEvaluator : PlanEvaluator<MAXS, MAXL, SerialUniform, ONE> {
    using Base = PlanEvaluator<MAXS, MAXL, SerialUniform, ONE>;
    using Base::T; using Base::w; using Base::pd; using Base::bs_total; using Base::nbad; using Base::aux;
    X x;
    CoopMail &mail;

    MB_HD CoopEvaluator(const Tables &t, Scratch<MAXS, MAXL> &s, CoopMail &mb, const X &lanes)
        : Base(t, s), x(lanes), mail(mb) {}

    // Start of a plan: groups, rank starts and the first strategy that can be valid (PlanEvaluator::begin,
    // search_space/plan.py:231-249).  The admission pass already dropped plans whose first strategy is invalid.
    MB_HD void begin_coop(const PlanDesc &plan) {
        pd = plan;
        bs_total = T.p.gbs / pd.batches;
        int lb = 0;
#pragma unroll 1
        while ((2 << lb) <= bs_total) ++lb;
        nbad = 0;
        x.sync();                                            // the previous chain of this warp is finished in every lane
        int carry = 0;
#pragma unroll 1
        for (int base = 0; base < pd.S; base += x.width()) { // rank starts: prefix sum of the group sizes
            const int s = base + x.lane();
            const int g = s < pd.S ? pd.row[s] : 0;
            const int sz = s < pd.S ? (1 << g) : 0;
            const int inc = x.incl_scan(sz);
            if (s < pd.S) {
                w.gcode[s] = (uint8_t)g;
                w.tpc[s] = (uint8_t)(g > lb ? g - lb : 0);
                w.rs[s] = (uint16_t)(carry + inc - sz);
            }
            carry += x.last_lane(inc);
        }
        if (x.leader()) w.rs[pd.S] = (uint16_t)carry;
        x.sync();
    }

    // IntraStagePlanGenerator._next_strategy (search_space/plan.py:251-268): the stage with the smallest memory
    // state (or, without a state, the largest dp) that still has dp != 1 halves its dp; first one among equals.
    MB_HD bool next_strategy_coop(bool have_state) {
        int pick = 0x7FFFFFFF;
        if (have_state) {
            double best = INFINITY;
            bool none = true;
            METIS_PAR(x, s, pd.S) {
                if (w.gcode[s] != w.tpc[s] && (none || w.mstate[s] < best || (w.mstate[s] == best && s < pick))) {
                    pick = s; best = w.mstate[s]; none = false;
                }
            }
            // NaN-free: memory states are differences of finite numbers
            x.argmin_first(best, pick);
        } else {
            int best = -1;
            METIS_PAR(x, s, pd.S) {
                const int ldp = (int)w.gcode[s] - (int)w.tpc[s];
                if (ldp != 0 && (ldp > best || (ldp == best && s < pick))) { pick = s; best = ldp; }
            }
            x.imax_first(best, pick);
        }
        if (pick == 0x7FFFFFFF) return false;
        const int g = w.gcode[pick], t = w.tpc[pick];
        nbad += (this->stage_bad(g, t + 1) ? 1 : 0) - (this->stage_bad(g, t) ? 1 : 0);
        x.sync();                                            // every lane has read tpc[pick]
        if (x.leader()) w.tpc[pick] = (uint8_t)(t + 1);
        x.sync();
        return true;
    }

    // first stage (in stage order) whose error mailbox is set: leader scan, rare path
    MB_HD_NOINLINE int first_error(const double *box, int n) {
        x.sync();
        if (x.leader()) {
            mail.err = 0;
#pragma unroll 1
            for (int s = 0; s < n; ++s)
                if (box[s] != 0.0) {
                    const uint64_t code = (uint64_t)box[s];
                    mail.err = (int)(code & 0xFF);
                    mail.pad = (int)(code >> 8);
                    break;
                }
        }
        x.sync();
        aux = (uint32_t)mail.pad;
        return mail.err;
    }

    // StagePerformance.get_intra_stage_compute_performance (model/device_group.py:54-85) -> w.perf
    MB_HD int compute_performance_coop() {
        const bool one_type = ONE || T.p.num_types == 1;
        bool failed = false;
        x.sync();
        METIS_PAR(x, s, pd.S) {
            const int g = w.gcode[s], tpc = w.tpc[s];
            double p = 0.0;
            int fail = 0;
            int ta = 0, tb = 0;
            if (!one_type) {
                const int a = this->rank_start(s), b = a + (1 << g);
                ta = type_of_rank(T, pd.ns, a); tb = type_of_rank(T, pd.ns, b - 1);
            }
            if (ta == tb) {
                const int bs = bs_total >> (g - tpc);
                const int key = key_of(T, ta, tpc, bs);
                if (key < 0) { aux = ((uint32_t)tpc << 16) | (uint32_t)bs; fail = METIS_FATAL_KEY_EXEC; }
                else if (T.exec_full[key] == 0.0) fail = METIS_FATAL_ZERODIV;
                else p = T.inv_exec[key];                     // 1. / profile_cost
            } else {
                const int a = this->rank_start(s);
                const int rc = this->hetero_performance(a, a + (1 << g), 1 << (g - tpc), tpc, p);
                if (rc) fail = rc;
            }
            w.perf[s] = p;
            w.extra[s] = fail ? (double)fail + (double)aux * 256.0 : 0.0;   // per-stage error mailbox
            failed = failed || fail != 0;
        }
        if (x.any(failed)) return first_error(w.extra, pd.S);
        x.sync();
        if (x.leader()) mail.val = seq_py_sum(w.perf, pd.S);     // sum(compute_performance) (:82)
        x.sync();
        const double tot = mail.val;
        if (tot == 0.0) return METIS_FATAL_ZERODIV;
        METIS_PAR(x, s, pd.S) w.perf[s] = w.perf[s] / tot;
        x.sync();
        return 0;
    }

    // Forward pass of LayerComputeBalancer (model/load_balancer.py:216-231), predicted and then verified exactly.
    //
    // Sequentially, stage s can only start once stage s-1 has closed, and closing takes one compare-and-subtract per
    // sub-layer.  Here the interval ends are first PREDICTED from the running sum psub of the demands: a stage with
    // capacity c that starts at a ends at the first b with psub[b + 1] >= c + psub[a] (one warp-wide search per
    // stage; what the real-number version of the pass would do).  Then every lane replays its stages' fills with
    // the reference's own operations - the strict compare and the rounded subtraction for every sub-layer - from the
    // predicted starts, which yields the exact residual capacities and VERIFIES the prediction: all compares up to
    // the predicted end must succeed and the one at the end must fail.  If every stage verifies, stage 0 started at
    // 0 and each next start follows from an exactly replayed fill, so the state equals the sequential pass
    // (induction over the stages).  If any stage fails (a compare decided by the last bits), the leader runs the
    // sequential pass.  returns true when the forward state (w.fe, w.capa, mail.k / s_top / top_skip) is final.
    MB_HD bool forward_coop() {
        const int S = pd.S, last = S - 1;
        const int L = T.p.num_layers;
        if (S < 4 || T.p.norm_len < L) { x.note(kPathSeqForward); return false; }   // nothing to overlap: sequential pass
        const int N = kH * L;
        const int lim = (N - 1 - kH) > 0 ? (N - 1 - kH) : 0;  // :218
        const double *dsub = T.dsub;
        const double *P = T.psub;
        // ---- prediction: uniform walk over the stages ----
        int a = 0, first_open = -1;
        int span = lim / last;                                // sub-layers the previous stage took: where to look first
#pragma unroll 1
        for (int s = 0; s < last; ++s) {
            int b = lim;
            bool closed = false;
            if (a < lim) {
                const double t = w.perf[s] + P[a];
                int i0 = a + span - 14;                       // a 32-entry window around the expected end
                if (i0 < a + 1) i0 = a + 1;
                int i = x.first_ge_window(P, N, i0, a + 1, t);
                if (i < 0) { x.note(kPathFirstGe); i = x.first_ge(P, N, t); }
                b = i - 1 > a ? i - 1 : a;
                if (b >= lim) b = lim; else closed = true;
                span = b - a;
            }
            if (x.leader()) { w.first[s] = (uint16_t)a; w.fe[s] = (uint16_t)(b | (closed ? kBroke : 0)); }
            if (!closed && first_open < 0) first_open = s;
            a = closed ? b + 1 : lim;
        }
        x.sync();
        // ---- exact replay of every stage from its predicted start ----
        bool bad = false;
        METIS_PAR(x, s, last) {
            const int st = w.first[s];
            const uint16_t e = w.fe[s];
            const int b = e & kPos;
            double c = w.perf[s];
#pragma unroll 4
            for (int j = st; j < b; ++j) {
                const double d = dsub[j];
                if (!(c > d)) { bad = true; break; }          // the reference would have closed the stage here
                c -= d;
            }
            if ((e & kBroke) && !bad && c > dsub[b]) bad = true;      // the reference would have gone on
            w.capa[s] = c;
        }
        if (x.any(bad)) {
            x.note(kPathVerifyFailed);
            x.sync();
            METIS_PAR(x, s, last) w.capa[s] = w.perf[s];      // restore the input of the sequential pass
            return false;
        }
        if (x.leader()) {
            if (first_open < 0) { mail.k = a; mail.s_top = last - 1; mail.top_skip = 1; }   // a = end of stage last-1, + 1
            else { mail.k = lim; mail.s_top = first_open; mail.top_skip = 0; }
        }
        return true;
    }

    // Forward pass, backward pass and leftovers of LayerComputeBalancer (model/load_balancer.py:216-287).
    //   forward     leader: compare-and-subtract chain over the sub-layers (seq_forward)
    //   backward    leader: the last stage's own compare-and-subtract chain
    //   skipped     one sub-layer per closed stage, ascending.  In the regular geometry (every stage up to the last
    //               touched one holds at least one sub-layer) get_proper_stage offers stage s's skipped sub-layer to
    //               {s, s+1} and the decision for s depends on the one for s-1 only through capa[s]: pick_s = s+1 iff
    //               capa[s+1] > capa[s] - [pick_{s-1} == s] * d_{s-1}.  Both outcomes are evaluated per stage; since
    //               subtracting can only favour s+1, a stage is "always s", "always s+1" or "copies its input", and
    //               the chain is resolved with two ballots (nearest constant stage below).  Any other geometry:
    //               leader, general sequential form.
    //   middle      the block [k, m) between forward and backward fills, ascending: arg-max over [lo, last] by the
    //               whole warp per sub-layer.
    // Writes w.capa, w.fe, w.lstk, the middle block's stages (bytes of w.subw), mail.k / m.  returns METIS_FATAL_* (0 = ok)
    MB_HD int fill_coop() {
        const int S = pd.S, last = S - 1;
        const double *dlay = T.dlay;
        x.sync();
        const bool fwd = forward_coop();
        x.sync();
        if (x.leader()) {
            if (!fwd) {
                const FillState st = seq_forward<MAXS, MAXL>(T, S, w);
                mail.k = st.k; mail.s_top = st.s_top; mail.top_skip = st.top_skip ? 1 : 0;
            }
            x.mark(11);
            mail.m = seq_backward<MAXS, MAXL>(T, S, w, mail.k);
            mail.err = 0;
        }
        x.sync();
        x.mark(12);
        const FillState st{mail.k, mail.s_top, mail.top_skip != 0};
        const int m = mail.m;
        if (st.s_top >= 0 && !st.top_skip) x.note(kPathTail);
        // ---- skipped sub-layers ----
        // stages 0 .. reach hold the forward intervals; regular = none of them is empty
        const int reach = st.s_top;                           // -1 when S == 1
        bool irregular = false;
        METIS_PAR(x, s, reach + 1) {
            const int start = s == 0 ? 0 : (int)(w.fe[s - 1] & kPos) + ((w.fe[s - 1] & kBroke) ? 1 : 0);
            if (!((int)(w.fe[s] & kPos) > start)) irregular = true;
        }
        irregular = x.any(irregular);
        if (irregular) {
            x.note(kPathIrregular);
            if (x.leader()) mail.err = seq_skipped<MAXS, MAXL>(T, S, w);
            x.sync();
            if (mail.err) return mail.err;
        } else if (reach >= 0) {
            int carry = 0;                                    // did the previous stage's sub-layer go to this stage?
#pragma unroll 1
            for (int base = 0; base <= last; base += x.width()) {
                const int s = base + x.lane();
                bool has = false, o0 = false, o1 = false, has_prev = false;
                double c = 0.0, d = 0.0, d_prev = 0.0;
                int pos = 0;
                if (s <= last) {
                    c = w.capa[s];
                    if (s > 0 && s - 1 < last) {
                        const uint16_t ep = w.fe[s - 1];
                        has_prev = (ep & (kBroke | kTaken)) == kBroke;
                        if (has_prev) d_prev = dlay[(ep & kPos) / kH];
                    }
                    if (s < last) {
                        const uint16_t e = w.fe[s];
                        has = (e & (kBroke | kTaken)) == kBroke;
                        if (has) {
                            pos = e & kPos;
                            d = dlay[pos / kH];
                            const double cn = w.capa[s + 1];
                            o0 = cn > c;
                            o1 = has_prev ? cn > (c - d_prev) : o0;
                        }
                    }
                }
                // pick_s = s+1 ?  constant stages (o0 == o1) decide themselves, the others copy the stage below
                const unsigned kmask = x.ballot(o0 == o1), vmask = x.ballot(o0);
                const unsigned below_me = x.lane() ? (0xFFFFFFFFu >> (32 - x.lane())) : 0u;     // lanes < mine
                const unsigned kin = kmask & below_me;
                const bool in = kin ? ((vmask >> (31 - clz32(kin))) & 1u) != 0u : carry != 0;
                const bool up = (o0 == o1) ? o0 : in;          // this stage's sub-layer goes to s + 1
                carry = x.bcast_last(up ? 1 : 0);
                x.sync();                                     // every lane has read its neighbours' capacities
                if (s <= last) {
                    double cc = c;
                    const bool got_prev = has_prev && in;     // (in is false when the stage below has no sub-layer to give)
                    if (got_prev) cc -= d_prev;
                    if (has && !up) cc -= d;
                    if (got_prev || (has && !up)) w.capa[s] = cc;
                    if (has) w.lstk[s] = (uint8_t)(up ? s + 1 : s);
                }
            }
            x.sync();
        }
        // ---- middle block: any length up to 7 * L, one byte per sub-layer in w.subw (unused by the balancer else) ----
        if (m > st.k) {
            x.note(kPathMiddle);
            if (x.leader()) mail.flag = middle_lo<MAXS, MAXL>(S, w, st);
            x.sync();
            int lo = mail.flag;
#pragma unroll 1
            for (int j = st.k; j < m; ++j) {
                int pick = 0x7FFFFFFF;
                double best = -INFINITY;
#pragma unroll 1
                for (int t = lo + x.lane(); t <= last; t += x.width())
                    if (w.capa[t] > best || (w.capa[t] == best && t < pick)) { best = w.capa[t]; pick = t; }
                x.argmax_first(best, pick);
                x.sync();                                     // every lane has read the capacities
                if (x.leader()) {
                    w.capa[pick] = best - dlay[j / kH];
                    reinterpret_cast<uint8_t *>(w.subw)[j - st.k] = (uint8_t)pick;
                }
                x.sync();
                if (pick != last) lo = pick;                  // the nearest block item below that is not on `last`
            }
        }
        return METIS_FATAL_NONE;
    }

    // LayerComputeBalancer.run (model/load_balancer.py:197-207): w.perf -> w.part, w.cnt
    MB_HD int balance_coop() {
        const int S = pd.S;
        const int L = T.p.num_layers;
        if (T.p.norm_len < L) return METIS_FATAL_INDEX;       // expand_lc_demand[layer_id] IndexError (:219/:238)
        const double *lc = T.norm_lc;
        const int last = S - 1;
        x.sync();                                            // earlier readers of capa / got are done
        METIS_PAR(x, s, S) { w.capa[s] = w.perf[s]; w.got[s] = 0; }
        x.sync();
        x.mark(10);
        const int rc_tail = fill_coop();
        if (rc_tail) return rc_tail;
        const int m = mail.m;
        x.mark(13);
        // ---- majority vote back to real layers (:290-308), one layer per lane ----
        // Stage of sub-layer j, from the interval ends: j >= m -> last stage (backward tail); k <= j < m -> where
        // the middle block put it (bytes of subw); below k the forward slot t = #{u : start of stage u+1 <= j}, and if j is
        // that slot's skipped sub-layer: last stage when the backward pass took it, else where it was placed (lstk).
        const int kfwd = mail.k;
        METIS_PAR(x, r, L) {
            const int j0 = kH * r;
            int own = kDropped;
            if (j0 >= m) {
                own = last;
            } else {
                int t = 0;
                if (j0 < kfwd) {                             // first slot whose successor starts above j0
                    int lo = 0, hi = last - 1;               // (j0 < k: such a slot exists among 0 .. last-1)
#pragma unroll 1
                    while (lo < hi) {
                        const int mid = (lo + hi) >> 1;
                        const uint16_t e = w.fe[mid];
                        if ((int)(e & kPos) + ((e & kBroke) ? 1 : 0) <= j0) lo = mid + 1; else hi = mid;
                    }
                    t = lo;
                }
                uint64_t v = 0xFF00000000000000ULL;
                uint16_t e = w.fe[t];                        // slot t: its end, and where stage t + 1 starts
                int nxt = (int)(e & kPos) + ((e & kBroke) ? 1 : 0);
#pragma unroll 1
                for (int q = 0; q < kH; ++q) {
                    const int j = j0 + q;
                    int st;
                    if (j >= m) st = last;
                    else if (j >= kfwd) st = reinterpret_cast<const uint8_t *>(w.subw)[j - kfwd];
                    else {
#pragma unroll 1
                        while (nxt <= j) { ++t; e = w.fe[t]; nxt = (int)(e & kPos) + ((e & kBroke) ? 1 : 0); }
                        st = t;
                        if (nxt - 1 == j && (e & kBroke)) st = (e & kTaken) ? last : (int)w.lstk[t];
                    }
                    v |= (uint64_t)st << (8 * q);
                }
                own = layer_owner(v, (T.p.corrected & METIS_FIX_Q5) != 0);
            }
            reinterpret_cast<uint8_t *>(w.ownerw)[r] = (uint8_t)own;
        }
        METIS_PAR(x, s, S) w.cnt[s] = 0;
        x.sync();
        x.mark(14);
        // ---- first / last / count of the layers of each stage: lanes holding layers of one stage form a group
        //      (match), its lowest lane folds the group into the stage's entry; blocks of `width` layers in turn ----
#pragma unroll 1
        for (int base = 0; base < L; base += x.width()) {
            const int r = base + x.lane();
            const int own = r < L ? (int)reinterpret_cast<const uint8_t *>(w.ownerw)[r] : (int)kDropped;
            const unsigned peers = x.match_any(own);
            if (own != (int)kDropped && x.lane() == ctz32(peers)) {
                const int n = popc32(peers), lo_r = r, hi_r = base + 31 - clz32(peers);
                const int have = w.cnt[own];
                if (have == 0 || lo_r < (int)w.first[own]) w.first[own] = (uint16_t)lo_r;
                if (have == 0 || hi_r > (int)w.lastl[own]) w.lastl[own] = (uint16_t)hi_r;
                w.cnt[own] = (uint16_t)(have + n);
            }
            x.sync();
        }
        // ---- spare capacity (:300-306) ----
        METIS_PAR(x, s, S) {
            const int n = w.cnt[s];
            w.capa[s] = n ? w.perf[s] - range_sum<SerialUniform>(T, kRangeNorm, 0, lc, w.first[s], (int)w.lastl[s] + 1) : w.perf[s];
        }
        x.sync();
        x.mark(15);
        // ---- boundary adjustment (:310-356): at most three committed single-layer moves ----
        uint8_t *owner = reinterpret_cast<uint8_t *>(w.ownerw);
#pragma unroll 1
        for (int n = 1; n <= 3; ++n) {
            int top = 0x7FFFFFFF;
            double maxc = -INFINITY;
            METIS_PAR(x, t, S)                               // stable: lowest index among equal maxima (:329-331)
                if (w.capa[t] > maxc || (w.capa[t] == maxc && t < top)) { maxc = w.capa[t]; top = t; }
            x.argmax_first(maxc, top);
            if (top == 0x7FFFFFFF) top = 0;
            int nb = -1;
            double val = INFINITY;
            if (top - 1 >= 0 && w.capa[top - 1] < val) { nb = top - 1; val = w.capa[top - 1]; }
            if (top + 1 < S && w.capa[top + 1] < val) { nb = top + 1; }
            if (nb < 0 || w.cnt[nb] <= 1) break;             // no-op rounds leave the state unchanged
            const int layer = (top > nb) ? w.lastl[nb] : w.first[nb];
            const double dl = lc[layer];
            const double ntop = w.capa[top] - dl;
            const double nnb = w.capa[nb] + dl;
            double newmax = -INFINITY;
            METIS_PAR(x, t, S) {
                const double v = (t == top) ? ntop : (t == nb) ? nnb : w.capa[t];
                if (v > newmax) newmax = v;
            }
            newmax = x.max_all(newmax);
            if (newmax > maxc) break;                        // :352 (not committed)
            x.sync();                                        // every lane has read the state of this round
            if (x.leader()) {
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
            }
            x.sync();
        }
        x.mark(16);
        // ---- partition = cumulative layer counts (:358-364) ----
        int carry = 0;
#pragma unroll 1
        for (int base = 0; base < S; base += x.width()) {
            const int s = base + x.lane();
            const int v = s < S ? (int)w.cnt[s] : 0;
            const int inc = x.incl_scan(v);
            if (s < S) w.part[s + 1] = (uint16_t)(carry + inc);
            carry += x.last_lane(inc);
        }
        if (x.leader()) w.part[0] = 0;
        x.sync();
        return METIS_FATAL_NONE;
    }

    // LayerLoadBalancer._adj_compute_performance (model/load_balancer.py:71-107)
    // in: w.perf (c_capa), w.extra (m_demand); out: w.perf; returns 1 = None, 0 ok, <0 fatal (negated code)
    MB_HD int adjust_performance_coop() {
        const int S = pd.S;
        const bool one_type = ONE || T.p.num_types == 1;
        double *ratio = reinterpret_cast<double *>(w.subw);      // free after the vote (MAXL >= MAXS)
        double *mcap = ratio + MAXS / 2;                          // stage memory capacity; subw has MAXL >= 2*(MAXS/2).. see static_assert
        static_assert(MAXL >= MAXS, "subw doubles as two S-sized fp64 arrays only when MAXL >= 2 * MAXS / 2");
        (void)mcap;
        x.sync();
        METIS_PAR(x, s, S) {                                     // independent per stage (:80-89)
            const int a = one_type ? 0 : this->rank_start(s), b = a + this->group(s);
            const double c = w.perf[s], md = w.extra[s];
            const double mc = one_type ? T.type_memory[0] * (double)this->group(s) : this->memory_capacity(a, b);
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
            ratio[s] = (mc > md) ? 0.0 : (c - adj);          // this stage's term of extra_required_capacity (:89)
        }
        x.sync();
        if (x.leader()) {                                        // order-dependent accumulations (:89-91)
            double need = 0.;
#pragma unroll 4
            for (int s = 0; s < S; ++s)
                if (w.capa[s] == 0.0 && ratio[s] != 0.0) need += ratio[s];
                else if (ratio[s] != 0.0) need += ratio[s];
            mail.val = need;
            mail.flag = seq_py_sum(w.capa, S) < need ? 1 : 0;
        }
        x.sync();
        if (mail.flag) return 1;
        METIS_PAR(x, s, S) w.extra[s] = 0.;
        x.sync();
        if (x.leader()) {                                        // :96-104, sequential: `need` changes as it goes
            double need = mail.val;
            int guard = 0;
            mail.err = 0;
#pragma unroll 1
            while (need > 0.01) {
                PySum tot;
#pragma unroll 4
                for (int s = 0; s < S; ++s) tot.add(w.capa[s] > 0.001 ? w.perf[s] : 0.0);
                const double tmp_total = tot.result();
#pragma unroll 4
                for (int s = 0; s < S; ++s)                      // c_capa_ratio list (:98), before the updates
                    ratio[s] = w.capa[s] > 0.001 ? w.perf[s] / tmp_total : 0.0;
#pragma unroll 4
                for (int s = 0; s < S; ++s) {
                    const double av = w.capa[s];
                    const double want = need * ratio[s];
                    const double give = want > av ? av : want;
                    w.extra[s] += give;
                    w.capa[s] -= give;
                    need -= give;
                }
                if (++guard > 4096) { mail.err = METIS_FATAL_HANG; break; }
            }
        }
        x.sync();
        if (mail.err) return -mail.err;
        METIS_PAR(x, s, S) w.perf[s] = w.extra[s] + w.mstate[s];
        x.sync();
        return 0;
    }

    // One attempt of LayerLoadBalancer.partition_layer after the balancer (model/load_balancer.py:127-143):
    // memory demand (:29-55), OOM test (:57-63), capacity re-weighting.  Returns like PlanEvaluator::memory_phase.
    MB_HD int memory_phase_coop(int attempt) {
        const int S = pd.S;
        const bool one_type = ONE || T.p.num_types == 1;
        const int type0 = T.run_type[pd.ns * T.p.num_types];
        const bool q10_short = T.p.q10_devices < T.p.total_devices;   // node 0 has fewer GPUs than the average (Q10)
        const bool own_type = (T.p.corrected & METIS_FIX_Q6) != 0;
        bool failed = false, oom = false;
        x.sync();                                            // the balancer's last readers of capa / extra / mstate are done
        METIS_PAR(x, s, S) {
            const int g = w.gcode[s], tpc = w.tpc[s];
            const int a = this->rank_start(s), b = a + (1 << g);
            double md = 0.001, err = 0.0;
            if (!ONE && own_type) {                          // opt-in METIS_FIX_Q6 (not the reference; single type: no change)
                const int rc = this->memory_demand_own_type(s, md);
                if (rc) err = (double)rc + (double)aux * 256.0;
            } else if (q10_short && !own_type && b > T.p.q10_devices) {
                err = (double)METIS_FATAL_INDEX;             // device_types[rank]: IndexError (load_balancer.py:36, Q10)
            } else if (one_type || type_of_q10(T, pd.ns, a) == type_of_q10(T, pd.ns, b - 1)) {
                const int bs = bs_total >> (g - tpc);
                const int key = key_of(T, type0, tpc, bs);
                if (key < 0) err = (double)METIS_FATAL_KEY_MEMORY + (double)(((uint32_t)tpc << 16) | (uint32_t)bs) * 256.0;
                else md += range_sum<SerialUniform>(T, kRangeMem, key, T.mem + (size_t)key * T.p.lpad, w.part[s], w.part[s + 1]) * kMemCoef;
            } else {
                const int rc = this->hetero_memory_demand(s, type0, md);
                if (rc) err = (double)rc + (double)aux * 256.0;
            }
            const double state = one_type ? T.type_memory[0] * (double)(1 << g) - md : this->memory_capacity(a, b) - md;
            w.extra[s] = md;
            w.capa[s] = state;
            w.mstate[s] = err;
            failed = failed || err != 0.0;
            oom = oom || state < 0;
        }
        failed = x.any(failed);
        oom = x.any(oom);
        if (failed) return -first_error(w.mstate, S);
        x.sync();
        if (!oom) {
            METIS_PAR(x, s, S) w.mstate[s] = w.capa[s];
            x.sync();
            return 1;
        }
        if (attempt >= 3) return 0;
        x.mark(21);
        const int rc = adjust_performance_coop();
        if (rc < 0) return rc;
        return rc == 1 ? 0 : 2;
    }

    // HeteroCostEstimator.get_cost (model/cost_estimator.py:199-244); returns 0 ok, 1 KeyError.  The cost lands in
    // mail.val (every lane reads it after the final sync).
    MB_HD int get_cost_coop(double &cost_out) {
        const int per = T.p.devices_per_node;
        const int Lm = T.p.num_layers;
        const bool one_type = ONE || T.p.num_types == 1;
        const bool ubw = T.p.uniform_bw != 0;
        const int nstage = pd.label < pd.S ? pd.label : pd.S;  // zip(range(plan.num_stage), strategies)
        // rank_node_map holds num_nodes * devices(node 0) ranks (cluster_bandwidth.py:34-47, Q10): beyond -> KeyError
        if (T.p.q10_devices < T.p.total_devices && this->rank_start(nstage) > T.p.q10_devices) return 1;
        double *ppterm = reinterpret_cast<double *>(w.subw);  // free after the vote (MAXL >= MAXS)
        bool bad = false;
        double max_len = -INFINITY, max_upd = -INFINITY, max_dp = -INFINITY;
        x.sync();
        METIS_PAR(x, s, nstage) {
            const int g = w.gcode[s], tpc = w.tpc[s];
            const int a = one_type ? 0 : this->rank_start(s), b = a + (1 << g);
            const int la = w.part[s], lb = w.part[s + 1];
            const int ldp = g - tpc;
            const int mbs = bs_total >> ldp;
            const int ta = one_type ? 0 : type_of_rank(T, pd.ns, a);
            const int tb = one_type ? 0 : type_of_rank(T, pd.ns, b - 1);
            double len = 0.0;
            if (ta == tb) {                                   // _get_execution_cost :175-188
                const int key = key_of(T, ta, tpc, mbs);
                if (key < 0) bad = true;
                else len = range_sum<SerialUniform>(T, kRangeLc, key, T.lc + (size_t)key * T.p.lpad, la, lb);
            } else if (this->hetero_exec_cost(a, b, 1 << ldp, tpc, la, lb, len)) {
                bad = true;
            }
            w.capa[s] = len;
            if (len > max_len) max_len = len;
            const double inv_tp = pow2_neg(tpc);              // 1 / tp, exact power of two
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
                    const int a2 = this->rank_start(s), b2 = this->rank_start(s + 2);
                    pp = act / (this->bw_of_node_range(a2 / per, (b2 - 1) / per) * 1048576.0);
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
                dpc = (double)(2 * (dp - 1)) / ((double)dp * (this->dp_bandwidth(this->rank_start(s), dp, 1 << tpc) * 1048576.0)) * params;
            }
            if (dpc > max_dp) max_dp = dpc;
            const double upd = T.p.optimizer_time * inv_tp * T.ratio[lb - la];   // :145-147
            if (upd > max_upd) max_upd = upd;
        }
        if (x.any(bad)) return 1;                             // KeyError raised while costing a stage
        max_len = x.max_all(max_len);
        max_upd = x.max_all(max_upd);
        max_dp = x.max_all(max_dp);
        x.sync();
        x.mark(23);
        if (x.leader()) {                                     // order-dependent sums, stage order
            double pp_cost = 0.;
#pragma unroll 4
            for (int s = 0; s + 1 < nstage; ++s) pp_cost += ppterm[s];
            const double lens = seq_py_sum(w.capa, nstage);
            const int s = nstage - 1;                         // _get_fb_sync_cost of the last costed stage
            const int a = one_type ? 0 : this->rank_start(s), b = a + this->group(s);
            double v = 0.0;
            mail.flag = this->fb_sync_cost(a, b, w.tpc[s], bs_total >> (w.gcode[s] - w.tpc[s]), v);
            const double fb_sync = v * (double)pd.batches;
            const double exec = ((double)(pd.batches - 1) * max_len) + lens;            // :235-236
            const double bg = T.p.batch_generator * (double)pd.batches;
            mail.val = exec + fb_sync + max_upd + max_dp + pp_cost + bg;                // :241-242
        }
        x.sync();
        if (mail.flag) return 1;
        cost_out = mail.val;
        return 0;
    }

    // cost_het_cluster.py:31-48 for one inter-stage plan with IntraStagePlanGenerator.has_next
    // (search_space/plan.py:192-226) inlined: the whole chain, depth first.
    // How the chain starts (the bulk round of the search evaluates the first partition attempt of every plan):
    //   kFresh   nothing was done yet
    //   kReplay  the first attempt was counted by the bulk round; it is recomputed here, not recounted
    //   kRetry   the first attempt ran out of memory and the bulk round re-weighted the stage performance
    //            (load_balancer.py:137-141): continue with attempt 2 from `perf[s * perf_stride]`
    //   kAdvance the first attempt ran out of memory and no re-weighting exists (:142-143): the first strategy is
    //            over, continue with the next one (memory_state None, plan.py:225)
    enum Start { kFresh = 0, kReplay = 1, kRetry = 2, kAdvance = 3 };
    template <class Sink>
    MB_HD void run_chain(const PlanDesc &plan, Sink &sink, int start, const double *perf = nullptr, size_t perf_stride = 0) {
        begin_coop(plan);
        bool started = false, have_state = false;
        bool skip_first = start == kReplay;
        int nrep = 0, step = 0;
        if (start == kRetry) {
            METIS_PAR(x, s, pd.S) w.perf[s] = perf[(size_t)s * perf_stride];
            x.sync();
        }
#pragma unroll 1
        for (;;) {
            if (nrep == 1) return;                            // plan.py:194-195
            int attempt = 0;
#pragma unroll 1
            for (;;) {
                int first_attempt = 1;
                if (!started) {                               // first strategy that can be valid (see begin)
                    started = true;
                    if (start == kAdvance && !next_strategy_coop(false)) return;
                    if (start == kRetry) first_attempt = 2;
                } else if (!next_strategy_coop(have_state)) return;   // :203-204
                if (!this->valid()) continue;
                int rc = 0;
                if (first_attempt == 1) {
                    if (!skip_first) sink.partition_call();
                    x.mark(2);
                    rc = compute_performance_coop();
                    if (rc) { sink.fatal(pd.ordinal, rc, aux); return; }
                }
                attempt = 0;
#pragma unroll 1
                for (int a = first_attempt; a <= 3; ++a) {    // LayerLoadBalancer.partition_layer (:121-144)
                    if (!skip_first) sink.balancer_run();
                    skip_first = false;
                    x.gate();                                 // (device) the block's warps start their runs together
                    rc = balance_coop();
                    if (rc) { sink.fatal(pd.ordinal, rc, aux); return; }
                    x.mark(20);
                    const int r = memory_phase_coop(a);
                    if (r < 0) { sink.fatal(pd.ordinal, -r, aux); return; }
                    if (r == 1) { attempt = a; break; }
                    if (r == 0) break;
                }
                skip_first = false;
                have_state = attempt > 0;                     // memory_state is None after a failure (:225)
                if (attempt > 0) break;
            }
            nrep = attempt;
            x.mark(22);
            double cost = 0.0;
            if (get_cost_coop(cost) == 0) sink.emit(pd, step, nrep, cost, w.tpc, w.part);
            else sink.keyerror();
            x.sync();                                         // the leader's record is written before the state changes
            x.mark(24);
            ++step;
        }
    }
};

}  // namespace metis
