// metis_enum.cpp - host-side enumeration of device-group rows in the reference's order.
//
// Restates gen_dgroups_for_stages_with_variance (search_space/device_group.py:93-107):
// power-of-two shapes filtered by the variance floor, non-decreasing compositions of
// num_gpus in lexicographic shape order (:58-81), pair-merging of the smallest groups down
// to max_permute_len (:7-55) and the multiset permutations of the merged groups in the
// prefix-shift order of Williams' algorithm (search_space/utils.py:56-88).  `dg_idx` in the
// reference is the position in this list, so the order is part of the contract.
//
// Structure: (1) list the compositions, (2) merge each one and count its permutations in closed
// form (n! / prod mult!), (3) prefix-sum the counts into row offsets, (4) generate the
// permutations of disjoint composition ranges on several host threads straight into the output.
// This is enumeration (integer tuples) - the candidate evaluation itself only runs on the GPU.
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <functional>
#include <mutex>
#include <thread>
#include <unistd.h>
#include <vector>

#include "../../include/metis_b200.h"

namespace {

using Group = std::vector<int>;   // one merged group = tuple of device-group sizes

uint8_t ilog2(int v) {
    uint8_t c = 0;
    while ((1 << c) < v) ++c;
    return c;
}

// permute() of search_space/device_group.py:7-55 without the final permutations: the merged groups.
// Every merge concatenates two NEIGHBOURS (:40-41), so a group is always a contiguous slice of the
// composition: the passes run on (offset, length, sum) triples without touching the heap.
std::vector<Group> merge_groups(const std::vector<int> &comp, int max_permute_len) {
    struct Slice { int off, len, sum; };
    const int n0 = (int)comp.size();
    std::vector<Slice> cur(n0), nxt;
    nxt.reserve(n0);
    for (int i = 0; i < n0; ++i) cur[i] = Slice{i, 1, comp[i]};
    auto same = [&](const Slice &a, const Slice &b) {
        return a.len == b.len && std::equal(comp.begin() + a.off, comp.begin() + a.off + a.len, comp.begin() + b.off);
    };
    int num_reduce = n0 - max_permute_len;
    while (num_reduce > 0) {
        const int count = (int)cur.size();
        const int min_size = cur[0].sum;
        int num_min = count;                               // find_num_min (:8-12)
        for (int idx = 0; idx < count; ++idx)
            if (!same(cur[idx], cur[0])) { num_min = idx + 1; break; }
        if (num_min / 2 > num_reduce) num_reduce = num_min / 2;      // :26-27
        nxt.clear();
        for (int i = 0; i < count; i += 2) {                          // :31-45
            if (num_reduce <= i / 2) {
                nxt.insert(nxt.end(), cur.begin() + i, cur.end());
                break;
            }
            if (i + 1 >= count) {
                nxt.push_back(cur[i]);
            } else if (cur[i].sum == min_size && cur[i].sum == cur[i + 1].sum) {
                nxt.push_back(Slice{cur[i].off, cur[i].len + cur[i + 1].len, cur[i].sum + cur[i + 1].sum});
            } else {
                nxt.push_back(cur[i]);
                nxt.push_back(cur[i + 1]);
            }
        }
        cur.swap(nxt);
        if (num_reduce == (int)cur.size() - max_permute_len) break;   // :48-50
        num_reduce = (int)cur.size() - max_permute_len;
    }
    std::vector<Group> groups;
    groups.reserve(cur.size());
    for (const Slice &g : cur) groups.emplace_back(comp.begin() + g.off, comp.begin() + g.off + g.len);
    std::sort(groups.begin(), groups.end());               // utils.py:57 (tuple comparison == lexicographic)
    return groups;
}

// number of distinct permutations of a sorted multiset: n! / prod(multiplicity!)
int64_t multiset_permutation_count(const std::vector<Group> &sorted_items) {
    int64_t total = 1, placed = 0;
    size_t i = 0;
    while (i < sorted_items.size()) {
        size_t j = i;
        while (j < sorted_items.size() && sorted_items[j] == sorted_items[i]) ++j;
        for (int64_t k = 1; k <= (int64_t)(j - i); ++k) total = total * (placed + k) / k;   // *= C(placed+k, k)
        placed += (int64_t)(j - i);
        i = j;
    }
    return total;
}

// multiset permutations of the sorted groups (search_space/utils.py:72-88), visiting order preserved;
// rows (log2 codes, `stages` bytes each) are written consecutively starting at dst
void williams_rows(const std::vector<Group> &items, int stages, uint8_t *dst) {
    const int n = (int)items.size();
    std::vector<int> rank(n), nxt(n, -1), off(n), len(n);
    std::vector<uint8_t> codes;
    for (int k = 0; k < n; ++k) {
        rank[k] = (k > 0 && items[k] == items[k - 1]) ? rank[k - 1] : k;   // equal tuples compare equal
        off[k] = (int)codes.size();
        len[k] = (int)items[k].size();
        for (int v : items[k]) codes.push_back(ilog2(v));
    }
    int head = 0;
    for (int k = 1; k < n; ++k) { nxt[k] = head; head = k; }              // prepend => non-increasing chain
    auto visit = [&]() {
        uint8_t *p = dst;
        for (int h = head; h != -1; h = nxt[h]) { memcpy(p, codes.data() + off[h], (size_t)len[h]); p += len[h]; }
        dst += stages;
    };
    auto nth = [&](int h, int k) {
        while (k > 0 && nxt[h] != -1) { h = nxt[h]; --k; }
        return h;
    };
    int i = nth(head, n - 2), j = nth(head, n - 1);
    visit();
    while (nxt[j] != -1 || rank[j] < rank[head]) {
        const int s = (nxt[j] != -1 && rank[i] >= rank[nxt[j]]) ? j : i;
        const int t = nxt[s];
        nxt[s] = nxt[t];
        nxt[t] = head;
        if (rank[t] < rank[head]) i = t;
        j = nxt[i];
        head = t;
        visit();
    }
}

// gen_dgroups_recursive (:58-81): the non-decreasing sequences of `stages` shapes that sum to `gpus`, in
// the order of the reference's depth-first search (lexicographic in the shape index).  The shapes are
// consecutive powers of two, so a sequence is a vector of counts per shape, lexicographic order is "more
// of the smaller shape first", and feasibility of a remainder is exact: R is a sum of exactly m powers of
// two from 2^a..2^b iff 2^a | R and  floor(R / 2^b) + popcount(R mod 2^b)  <=  m  <=  R / 2^a  (splitting
// one term into halves adds one term at a time).  Only live branches are visited - the reference's own
// pruning (:61-66, :73-74) discards the same dead branches later, at up to 10^2x the cost for 128 stages.
void list_compositions(int stages, int gpus, const std::vector<int> &shapes, std::vector<std::vector<int>> &out) {
    if (shapes.empty()) return;
    const int K = (int)shapes.size();
    for (int k = 1; k < K; ++k)
        if (shapes[k] != 2 * shapes[k - 1]) return;          // (list_stage only passes consecutive powers of two)
    const int top = shapes[K - 1];
    auto feasible = [&](int R, int m, int k) {                // R gpus in exactly m groups of shapes[k..K-1]
        if (k >= K) return R == 0 && m == 0;
        if (R == 0 || m == 0) return R == 0 && m == 0;
        if (R % shapes[k]) return false;
        const int fewest = R / top + __builtin_popcount((unsigned)(R % top));
        return fewest <= m && m <= R / shapes[k];
    };
    std::vector<int> count(K, 0), sol(stages);
    // depth-first over shapes; count[k] runs from its largest feasible value down
    struct Frame { int R, m, c; };
    std::vector<Frame> st(K + 1);
    int k = 0;
    st[0] = Frame{gpus, stages, -1};
    if (!feasible(gpus, stages, 0)) return;
    auto first_count = [&](const Frame &f, int kk) { return std::min(f.m, f.R / shapes[kk]); };
    st[0].c = first_count(st[0], 0) + 1;
    while (k >= 0) {
        Frame &f = st[k];
        int c = f.c - 1;
        while (c >= 0 && !feasible(f.R - c * shapes[k], f.m - c, k + 1)) --c;
        if (c < 0) { --k; continue; }
        f.c = c;
        count[k] = c;
        if (k + 1 == K || (f.R - c * shapes[k] == 0 && f.m - c == 0)) {
            for (int j = k + 1; j < K; ++j) count[j] = 0;
            int p = 0;
            for (int j = 0; j < K; ++j)
                for (int r = 0; r < count[j]; ++r) sol[p++] = shapes[j];
            out.push_back(sol);
            continue;                                          // next (smaller) count at this depth
        }
        st[k + 1] = Frame{f.R - c * shapes[k], f.m - c, 0};
        st[k + 1].c = first_count(st[k + 1], k + 1) + 1;
        ++k;
    }
}

// One stage count: prepare (compositions, merged groups, row offsets), then fill rows.
struct StageTable {
    int stages = 0;
    std::vector<std::vector<int>> comps;
    std::vector<std::vector<Group>> merged;
    std::vector<int64_t> offset;          // row offset of each composition, size merged.size()+1
    int64_t rows() const { return offset.empty() ? 0 : offset.back(); }
};

void list_stage(StageTable &t, int num_stages, int num_gpus, double variance) {
    t.stages = num_stages;
    const int share = std::max(num_gpus / num_stages, num_stages / num_gpus);   // :96-98
    const double floor_share = (double)share * variance;
    std::vector<int> shapes;
    for (int s = 1; s <= num_gpus; s <<= 1)
        if ((double)s >= floor_share) shapes.push_back(s);
    list_compositions(num_stages, num_gpus, shapes, t.comps);
    t.merged.resize(t.comps.size());
    t.offset.assign(t.comps.size() + 1, 0);
}

// Persistent host workers: the three parallel sections of one enumeration would otherwise pay a thread
// spawn + join each (24 spawns per call at 8 threads, a measurable share of a 3-4 ms enumeration).  The
// pool is created on first use, never destroyed (its threads are detached and die with the process) and
// rebuilt in a forked child, where the parent's threads do not exist.  Chunks are handed out through an
// atomic counter; the caller works too.
class WorkerPool {
  public:
    static WorkerPool &get() {
        static WorkerPool *pool = nullptr;
        static std::mutex guard;
        std::lock_guard<std::mutex> lk(guard);
        if (!pool || pool->pid_ != getpid()) pool = new WorkerPool();
        return *pool;
    }
    unsigned size() const { return nworkers_ + 1; }

    void run(int64_t chunks, const std::function<void(int64_t)> &chunk_body) {
        std::lock_guard<std::mutex> serial(run_mutex_);      // one parallel section at a time
        {
            std::lock_guard<std::mutex> lk(m_);
            body_ = &chunk_body;
            chunks_ = chunks;
            next_.store(0);
            pending_ = nworkers_;
            ++epoch_;
        }
        cv_work_.notify_all();
        drain();
        std::unique_lock<std::mutex> lk(m_);
        cv_done_.wait(lk, [&] { return pending_ == 0; });
        body_ = nullptr;
    }

  private:
    WorkerPool() : pid_(getpid()) {
        const char *env = getenv("METIS_ENUM_THREADS");
        unsigned v = env ? (unsigned)atoi(env) : 8u;         // 8 host threads unless METIS_ENUM_THREADS says otherwise
        const unsigned hw = std::thread::hardware_concurrency();
        if (hw && v > hw) v = hw;
        if (v < 1) v = 1;
        nworkers_ = v - 1;
        for (unsigned t = 0; t < nworkers_; ++t) std::thread([this] { loop(); }).detach();
    }
    void drain() {
        for (;;) {
            const int64_t c = next_.fetch_add(1);
            if (c >= chunks_) break;
            (*body_)(c);
        }
    }
    void loop() {
        uint64_t seen = 0;
        for (;;) {
            {
                std::unique_lock<std::mutex> lk(m_);
                cv_work_.wait(lk, [&] { return epoch_ != seen; });
                seen = epoch_;
            }
            drain();
            std::lock_guard<std::mutex> lk(m_);
            if (--pending_ == 0) cv_done_.notify_one();
        }
    }
    pid_t pid_;
    unsigned nworkers_ = 0;
    std::mutex m_, run_mutex_;
    std::condition_variable cv_work_, cv_done_;
    const std::function<void(int64_t)> *body_ = nullptr;
    int64_t chunks_ = 0;
    std::atomic<int64_t> next_{0};
    unsigned pending_ = 0;
    uint64_t epoch_ = 0;
};

template <class F>
void parallel_for(int64_t n, int64_t grain, F body) {        // body(begin, end) on chunks of `grain` items
    const int64_t chunks = (n + grain - 1) / grain;
    WorkerPool &pool = WorkerPool::get();
    if (pool.size() < 2 || chunks < 2) { if (n > 0) body((int64_t)0, n); return; }
    const std::function<void(int64_t)> chunk_body = [&](int64_t c) { body(c * grain, std::min(n, (c + 1) * grain)); };
    pool.run(chunks, chunk_body);
}

// All stage counts of a range: compositions per stage count, then merge + count and row generation
// over the flattened (stage count, composition) list so the host threads are evenly loaded.
struct TableSet {
    int first = 0;
    std::vector<StageTable> tables;
    std::vector<std::pair<int, int>> items;                  // (table index, composition index)

    void prepare(int first_stage, int last_stage, int num_gpus, double variance, int max_permute_len) {
        first = first_stage;
        const int n = last_stage - first_stage + 1;
        tables.assign(n, StageTable());
        parallel_for(n, 1, [&](int64_t b, int64_t e) {
            for (int64_t i = b; i < e; ++i) list_stage(tables[i], first_stage + (int)i, num_gpus, variance);
        });
        items.clear();
        for (int i = 0; i < n; ++i)
            for (int c = 0; c < (int)tables[i].comps.size(); ++c) items.emplace_back(i, c);
        parallel_for((int64_t)items.size(), 256, [&](int64_t b, int64_t e) {
            for (int64_t k = b; k < e; ++k) {
                StageTable &t = tables[items[k].first];
                const int c = items[k].second;
                t.merged[c] = merge_groups(t.comps[c], max_permute_len);
                t.offset[c + 1] = multiset_permutation_count(t.merged[c]);   // count; prefix-summed below
            }
        });
        for (StageTable &t : tables)
            for (size_t c = 0; c < t.merged.size(); ++c) t.offset[c + 1] += t.offset[c];
    }

    void fill(const std::vector<int64_t> &byte_off, uint8_t *out) const {
        parallel_for((int64_t)items.size(), 64, [&](int64_t b, int64_t e) {
            for (int64_t k = b; k < e; ++k) {
                const StageTable &t = tables[items[k].first];
                const int c = items[k].second;
                williams_rows(t.merged[c], t.stages, out + byte_off[items[k].first] + t.offset[c] * t.stages);
            }
        });
    }
};

}  // namespace

extern "C" int64_t metis_enum_device_groups(int32_t num_stages, int32_t num_gpus, double variance,
                                            int32_t max_permute_len, uint8_t *out, int64_t capacity_rows) {
    if (num_stages < 1 || num_gpus < 1 || max_permute_len < 1) return METIS_E_ARG;
    TableSet set;
    set.prepare(num_stages, num_stages, num_gpus, variance, max_permute_len);
    const int64_t rows = set.tables[0].rows();
    if (!out) return rows;
    if (rows > capacity_rows) return METIS_E_CAPACITY;
    set.fill(std::vector<int64_t>{0, rows * num_stages}, out);
    return rows;
}

extern "C" int64_t metis_enum_device_group_tables(int32_t first_stage, int32_t last_stage, int32_t num_gpus,
                                                  double variance, int32_t max_permute_len, int64_t *rows_per_stage,
                                                  uint8_t *out, int64_t capacity_bytes) {
    if (first_stage < 1 || last_stage < first_stage || num_gpus < 1 || max_permute_len < 1 || !rows_per_stage)
        return METIS_E_ARG;
    const int n = last_stage - first_stage + 1;
    // the sizing call (out == NULL) and the filling call that follows it share the prepared tables
    struct Prepared { int first, last, gpus, mpl; double variance; TableSet set; };
    static thread_local Prepared cache{0, 0, 0, 0, 0.0, {}};
    const bool hit = cache.first == first_stage && cache.last == last_stage && cache.gpus == num_gpus &&
                     cache.mpl == max_permute_len && cache.variance == variance && (int)cache.set.tables.size() == n;
    if (!hit) {
        cache.first = first_stage; cache.last = last_stage; cache.gpus = num_gpus; cache.mpl = max_permute_len;
        cache.variance = variance;
        cache.set.prepare(first_stage, last_stage, num_gpus, variance, max_permute_len);
    }
    const TableSet &set = cache.set;
    std::vector<int64_t> byte_off(n + 1, 0);
    for (int i = 0; i < n; ++i) {
        rows_per_stage[i] = set.tables[i].rows();
        byte_off[i + 1] = byte_off[i] + set.tables[i].rows() * (first_stage + i);
    }
    if (!out) return byte_off[n];
    if (byte_off[n] > capacity_bytes) return METIS_E_CAPACITY;
    set.fill(byte_off, out);
    const int64_t total_bytes = byte_off[n];
    cache.first = cache.last = 0;                            // release the prepared tables
    cache.set = TableSet();
    return total_bytes;
}


// ---------------------------------------------------------------------------------------------------------------
// Compact form of the same enumeration for DEVICE-side generation of the rows (SURVEY.md 8(f)-1): the host lists
// the compositions and merges their groups (cheap: thousands of compositions for millions of rows); the
// permutations - the bulk of the bytes - are written by het_rows_kernel (metis_search.cu), one thread per
// composition running the same prefix-shift walk as williams_rows above.
//   recs  [ncomp] MetisCompRec: byte offset of the composition's first row in the row blob, stage count, number of
//         merged groups, offset of its entry in `pool`
//   pool  bytes: per composition n group lengths followed by the log2 codes of the groups in SORTED order
//         (search_space/utils.py:57), `stages` bytes in total
// Call with recs == NULL to size (returns the number of compositions, *pool_bytes receives the pool size).
// ---------------------------------------------------------------------------------------------------------------
extern "C" int64_t metis_enum_compositions(int32_t first_stage, int32_t last_stage, int32_t num_gpus, double variance,
                                           int32_t max_permute_len, int64_t *rows_per_stage, MetisCompRec *recs,
                                           int64_t recs_capacity, uint8_t *pool, int64_t pool_capacity,
                                           int64_t *pool_bytes, int32_t *max_groups) {
    if (first_stage < 1 || last_stage < first_stage || num_gpus < 1 || max_permute_len < 1 || !rows_per_stage || !pool_bytes)
        return METIS_E_ARG;
    const int n = last_stage - first_stage + 1;
    struct Prepared { int first, last, gpus, mpl; double variance; TableSet set; };
    static thread_local Prepared cache{0, 0, 0, 0, 0.0, {}};
    const bool hit = cache.first == first_stage && cache.last == last_stage && cache.gpus == num_gpus &&
                     cache.mpl == max_permute_len && cache.variance == variance && (int)cache.set.tables.size() == n;
    if (!hit) {
        cache.first = first_stage; cache.last = last_stage; cache.gpus = num_gpus; cache.mpl = max_permute_len;
        cache.variance = variance;
        cache.set.prepare(first_stage, last_stage, num_gpus, variance, max_permute_len);
    }
    const TableSet &set = cache.set;
    int64_t nrec = 0, pbytes = 0, byte_off = 0;
    int most = 0;
    for (int i = 0; i < n; ++i) {
        const StageTable &t = set.tables[i];
        rows_per_stage[i] = t.rows();
        for (size_t c = 0; c < t.merged.size(); ++c) {
            pbytes += (int64_t)t.merged[c].size() + t.stages;
            most = std::max(most, (int)t.merged[c].size());
            const int64_t perms = t.offset[c + 1] - t.offset[c];
            nrec += (perms + METIS_COMP_SLICE_ROWS - 1) / METIS_COMP_SLICE_ROWS;
        }
    }
    *pool_bytes = pbytes;
    if (max_groups) *max_groups = most;
    if (!recs) return nrec;
    if (nrec > recs_capacity || pbytes > pool_capacity || !pool) return METIS_E_CAPACITY;
    int64_t k = 0, po = 0;
    for (int i = 0; i < n; ++i) {
        const StageTable &t = set.tables[i];
        for (size_t c = 0; c < t.merged.size(); ++c) {
            const int64_t perms = t.offset[c + 1] - t.offset[c];
            const uint32_t entry = (uint32_t)po;
            for (const Group &g : t.merged[c]) pool[po++] = (uint8_t)g.size();
            for (const Group &g : t.merged[c])
                for (int v : g) pool[po++] = ilog2(v);
            for (int64_t first = 0; first < perms; first += METIS_COMP_SLICE_ROWS) {
                MetisCompRec &r = recs[k++];
                r.row_offset = byte_off + (t.offset[c] + first) * t.stages;
                r.pool_offset = entry;
                r.stages = (uint16_t)t.stages;
                r.num_groups = (uint16_t)t.merged[c].size();
                r.first_row = (uint32_t)first;
                r.num_rows = (uint32_t)std::min<int64_t>(METIS_COMP_SLICE_ROWS, perms - first);
            }
        }
        byte_off += t.rows() * t.stages;
    }
    const int64_t ncomp = nrec;
    cache.first = cache.last = 0;
    cache.set = TableSet();
    return ncomp;
}
