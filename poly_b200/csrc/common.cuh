// common.cuh -- shared declarations of libpolyb200 (internal; the public surface is
// include/poly_b200.h).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <functional>
#include <vector>

#include "../../include/poly_b200.h"

namespace pg {

// thread-local error string + helpers (runtime.cu)
void set_error(const char *fmt, ...);
int cuda_fail(cudaError_t e, const char *what, const char *file, int line);
void note_launch(const char *kernel_name);

#define PG_CUDA(call)                                                     \
    do {                                                                  \
        cudaError_t _e = (call);                                          \
        if (_e != cudaSuccess) return ::pg::cuda_fail(_e, #call, __FILE__, __LINE__); \
    } while (0)

#define PG_LAUNCH_CHECK(name)                                             \
    do {                                                                  \
        ::pg::note_launch(name);                                          \
        cudaError_t _e = cudaGetLastError();                              \
        if (_e != cudaSuccess) return ::pg::cuda_fail(_e, name, __FILE__, __LINE__); \
    } while (0)

int sm_count();
// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) cached per (device, kernel); thread-safe (runtime.cu)
int func_smem(const void *kernel, size_t bytes);
// Grid of a kernel that loops over its work items: func_smem, then as many CTAs as are resident at once (at least
// one per SM), but no more than `work` (runtime.cu)
int resident_blocks(const void *kernel, int threads, size_t smem, uint64_t work, uint64_t *blocks);
// The n_reads + 1 offsets of a ragged batch copied to the host, for launchers that cut a batch into launch groups by
// row length; synchronises st (runtime.cu)
int host_row_starts(const uint64_t *d_offsets, uint64_t n_reads, cudaStream_t st, std::vector<uint64_t> &off);

// transform.complementTable (transform.go:78-109): every unlisted byte maps to 0, including the DNA
// letters U and Z.  Seqhash reads it on upper-cased bytes; the clone ligation on fragments as given.
__host__ __device__ __forceinline__ uint8_t complement(uint8_t c) {
    switch (c) {
        case 'A': return 'T'; case 'B': return 'V'; case 'C': return 'G'; case 'D': return 'H';
        case 'G': return 'C'; case 'H': return 'D'; case 'K': return 'M'; case 'M': return 'K';
        case 'N': return 'N'; case 'R': return 'Y'; case 'S': return 'S'; case 'T': return 'A';
        case 'V': return 'B'; case 'W': return 'W'; case 'Y': return 'R';
        case 'a': return 't'; case 'b': return 'v'; case 'c': return 'g'; case 'd': return 'h';
        case 'g': return 'c'; case 'h': return 'd'; case 'k': return 'm'; case 'm': return 'k';
        case 'n': return 'n'; case 'r': return 'y'; case 's': return 's'; case 't': return 'a';
        case 'v': return 'b'; case 'w': return 'w'; case 'y': return 'r';
        default: return 0;
    }
}

// Stream-ordered temporaries that are released together when the scope ends -- also on the early
// returns of PG_CUDA -- with cudaFreeAsync on the stream they were allocated on.
struct StreamScratch {
    cudaStream_t st;
    std::vector<void *> ptr;
    explicit StreamScratch(cudaStream_t s) : st(s) {}
    StreamScratch(const StreamScratch &) = delete;
    StreamScratch &operator=(const StreamScratch &) = delete;
    ~StreamScratch() {
        for (void *p : ptr) cudaFreeAsync(p, st);
    }
    template <typename T>
    cudaError_t alloc(T **p, uint64_t count) {  // at least one element, so the pointer is always valid
        ptr.push_back(nullptr);  // the slot first, so that keeping the buffer cannot throw and leak it
        cudaError_t e = cudaMallocAsync(&ptr.back(), (count ? count : 1) * sizeof(T), st);
        if (e != cudaSuccess) ptr.pop_back();
        else *p = (T *)ptr.back();
        return e;
    }
    void adopt(void *p) {  // take ownership of a buffer allocated elsewhere on the same stream
        if (p) ptr.push_back(p);
    }
};

// destinations of a sketch row block: the local buffer, or the gathered buffers of all ranks
struct SketchDst {
    uint32_t *ptr[PG_MAX_PEERS];
    int n;
};

// ---- per-row pieces of the sketch kernels (sketch_fill.cu, sketch_select.cu, sketch_select_large.cu) ----
// Row `row` of a batch is bytes [beg, beg + len) of the bases and has n = max(len - k, 0) k-mers (mash.go:73).
struct RowSpan {
    uint64_t beg, len, n;
};
__device__ __forceinline__ RowSpan row_span(const uint64_t *offsets, uint32_t uniform_len, uint64_t row, uint32_t k) {
    RowSpan r;
    if (offsets) {
        r.beg = offsets[row];
        r.len = offsets[row + 1] - r.beg;
    } else {
        r.beg = row * (uint64_t)uniform_len;
        r.len = uniform_len;
    }
    r.n = r.len > k ? r.len - k : 0;
    return r;
}
// the select regime of mash.go:87-102 (s == 0 included: it panics there); other rows are filled positionally
__host__ __device__ __forceinline__ bool select_regime(uint64_t n, uint64_t s) { return n >= s && n > 0; }

// Thread 0 writes the status and count of a finished select-regime row.  `panic`: the row reaches the
// reference's Sketches[-1] index (mash.go:96-98); each kernel tests that its own way.
__device__ __forceinline__ void put_row_status(int32_t *status, uint32_t *count, uint64_t row, uint32_t cnt, bool panic) {
    if (threadIdx.x != 0) return;
    if (status) status[row] = panic ? PG_ITEM_PANIC : PG_ITEM_OK;
    if (count) count[row] = cnt;
}
// s == 0: mash.go:96 reads Sketches[-1] on the first k-mer of a select-regime row.  True when that settled the row.
__device__ __forceinline__ bool empty_sketch_panics(uint32_t s, int32_t *status, uint32_t *count, uint64_t row) {
    if (s != 0) return false;
    put_row_status(status, count, row, 0, true);
    return true;
}

// Fused all-gather: the CTA copies the finished row src[0, s) to the row of every destination except
// dst, which already holds it.  Static indices keep `extra` in parameter space.
template <int NT>
__device__ __forceinline__ void replicate_row(const SketchDst &extra, uint64_t row, uint64_t row_stride, const uint32_t *src,
                                              const uint32_t *dst, uint32_t s) {
    if (extra.n > 0) {
        __syncthreads();  // src is complete
#pragma unroll
        for (int pr = 0; pr < PG_MAX_PEERS; ++pr) {
            if (pr >= extra.n) continue;
            uint32_t *peer = extra.ptr[pr] + row * row_stride;
            if (peer == dst) continue;
            for (uint32_t i = threadIdx.x; i < s; i += NT) peer[i] = src[i];
        }
    }
}

// Ascending bitonic sort of key[0, P) in shared memory by the NT threads of the CTA, P a power of two.  The
// keys must be in place before the call (a CTA barrier behind their stores); all threads call, and the
// sorted keys are visible to the whole CTA on return.
template <typename T, int NT>
__device__ void block_bitonic_sort(T *key, uint32_t P) {
    // Pair t of a stage with distance j touches elements inside the 64-element block [64 * (t / 32), +64)
    // whenever j <= 32, and a warp owns 32 consecutive pairs t: those stages only need a warp barrier.
    static_assert(NT % 32 == 0, "a warp must own 32 consecutive pairs of every stage");
    for (uint32_t k2 = 2; k2 <= P; k2 <<= 1) {
        for (uint32_t j = k2 >> 1; j > 0; j >>= 1) {
            for (uint32_t t = threadIdx.x; t < (P >> 1); t += NT) {
                const uint32_t i = ((t & ~(j - 1)) << 1) | (t & (j - 1)), ixj = i | j;
                const bool up = (i & k2) == 0;
                const T a = key[i], c = key[ixj];
                if ((a > c) == up) { key[i] = c; key[ixj] = a; }
            }
            if (j > 32) __syncthreads();  // this stage wrote outside the warp's own 64-element block
            else __syncwarp();            // stages with distance <= 32 read and write inside it
        }
        __syncthreads();  // the next k2 starts with a distance that may cross warps
    }
}

// ---- kernel launchers (one per .cu) -------------------------------------------
// sketch_fill.cu
int launch_sketch_uniform(const uint8_t *d_bases, uint64_t n_reads, uint32_t read_len, int k, int s,
                          uint32_t flags, uint32_t *d_out, uint64_t row_stride, int32_t *d_status,
                          cudaStream_t st, const SketchDst *extra = nullptr);
int launch_sketch_ragged(const uint8_t *d_bases, const uint64_t *d_offsets, uint64_t n_reads,
                         uint64_t max_read_len, int k, int s, uint32_t flags, uint32_t *d_out,
                         uint64_t row_stride, uint32_t *d_count, int32_t *d_status, cudaStream_t st);
// sketch_select.cu  (reads with n >= s; uniform: read_len != 0 and d_offsets == nullptr)
int launch_sketch_select(const uint8_t *d_bases, const uint64_t *d_offsets, uint32_t read_len,
                         uint64_t n_reads, int k, int s, uint32_t *d_out,
                         uint64_t row_stride, uint32_t *d_count, int32_t *d_status, cudaStream_t st,
                         const SketchDst *extra = nullptr, uint64_t max_read_len = 0);
// sketch_select_large.cu: the select regime for s > 16384 or k > 1024 (hashes through global memory)
int launch_sketch_select_large(const uint8_t *d_bases, const uint64_t *d_offsets, uint32_t read_len, uint64_t n_reads, int k, int s,
                               uint32_t *d_out, uint64_t row_stride, uint32_t *d_count, int32_t *d_status, cudaStream_t st,
                               const SketchDst &ex);
// distance.cu
int launch_similarity_pairs(const uint32_t *d_sk, const uint64_t *d_off, uint64_t n_sk,
                            const uint32_t *d_a, const uint32_t *d_b, uint64_t n_pairs,
                            int64_t *d_same, double *d_sim, double *d_dist, int32_t *d_status,
                            cudaStream_t st);
int launch_distance_block(const uint32_t *d_sk, uint64_t n, int s, uint64_t row_begin,
                          uint64_t row_end, uint32_t *d_same, double *d_dist, cudaStream_t st);
int launch_distance_sparse(const uint32_t *d_sk, uint64_t n, int s, uint64_t row_begin, uint64_t row_end, uint32_t flags,
                           uint32_t *d_i, uint32_t *d_j, uint32_t *d_same, uint64_t cap, unsigned long long *d_n_pairs,
                           cudaStream_t st);
// distance_join.cu (ascending sketches only): bucketed (value, id) index, built once per sketch
// set and reused for every row block
struct JoinIndex {
    uint64_t *entries = nullptr, *start = nullptr;
    uint32_t *vmax = nullptr;  // device word: the largest value, which sets the bucket scale (hist_kernel)
    uint64_t nb = 0, n = 0;
    uint64_t largest = 0;  // entries of the largest bucket: join_emit needs <= JOIN_CAP, the probe has no limit
    int s = 0;
    bool ok = false;
};
// The bucket of value v: values scaled to [0, nb) by the set's largest value vmax.  The index is built
// (hist_kernel, scatter_kernel) and probed (index_probe_kernel) with this one mapping.
__device__ __forceinline__ uint64_t join_bucket_scale(uint32_t nb, uint32_t vmax) {
    return (((uint64_t)nb) << 32) / ((uint64_t)vmax + 1);
}
__device__ __forceinline__ uint32_t join_bucket(uint32_t v, uint64_t scale, uint32_t nb) {
    return min((uint32_t)(((uint64_t)v * scale) >> 32), nb - 1);
}
// The keys (v << 32 | id0 + e / s) of the `total` words d_sk[e] of rows of s words, in any order, and atomicMax of
// their largest value into *d_vmax
int launch_batch_keys(const uint32_t *d_sk, uint64_t total, uint32_t s, uint64_t id0, uint64_t *d_keys, uint32_t *d_vmax, cudaStream_t st);
int join_build(const uint32_t *d_sk, uint64_t n, int s, cudaStream_t st, JoinIndex *ix);
int join_merge(const JoinIndex &old, const uint32_t *d_batch, uint64_t m, cudaStream_t st, JoinIndex *out);
int join_emit(const JoinIndex &ix, uint64_t row_begin, uint64_t row_end, uint32_t *d_same, double *d_dist, cudaStream_t st);
void join_free(JoinIndex &ix, cudaStream_t st);
// distance.cu: a plan = sortedness flags (+ join index when every sketch is ascending)
struct DistancePlan {
    const uint32_t *d_sk = nullptr;
    uint64_t n = 0;
    int s = 0;
    uint8_t *d_flag = nullptr;
    JoinIndex join;
};
int distance_plan_create(const uint32_t *d_sk, uint64_t n, int s, cudaStream_t st, DistancePlan *plan);
int distance_plan_rows(const DistancePlan &plan, uint64_t row_begin, uint64_t row_end, uint32_t *d_same, double *d_dist, cudaStream_t st);
void distance_plan_destroy(DistancePlan &plan, cudaStream_t st);
// The plan over n + m sketches of size s whose first n are plan's: d_sk holds all n + m rows.  Flags of the new
// rows; the join merged (every new row ascending), dropped (one is not) or still absent; an empty plan is created
// afresh.  plan is not changed; on an error nothing of *out remains allocated.
int distance_plan_grow(const DistancePlan &plan, const uint32_t *d_sk, uint64_t m, int s, cudaStream_t st, DistancePlan *out);
// distance.cu: rows per dense tile of the passes that consume a plan's tiles on the device (sparse pairs, cluster,
// dereplicate); n > 0
uint64_t distance_tile_rows(uint64_t n, uint64_t rows);
// distance.cu: rows [row_begin, row_end) (row_begin < row_end, n > 0) of n equal-size sketches as dense tiles of at most rows_per rows, over one
// DistancePlan and one tile buffer (counts if want_same, distances if want_dist).  consume(same, dist, rb, re) runs
// once each tile of rows [rb, re) is enqueued, with the unwanted buffer NULL; it may return early on an error.  The
// plan and the tile are released on every way out; the result is the first code other than PG_OK.
int distance_plan_tiles(const uint32_t *d_sk, uint64_t n, int s, uint64_t row_begin, uint64_t row_end, uint64_t rows_per,
                        bool want_same, bool want_dist, cudaStream_t st,
                        const std::function<int(const uint32_t *same, const double *dist, uint64_t rb, uint64_t re)> &consume);
// Counts p[i .. i + 3] of an array of `end` counts: one 16-byte load when vec (rows of a multiple of 4 counts, so
// every quad of a row-major tile is 16-byte aligned) and the quad is in range, else one by one with zeros past end.
__device__ __forceinline__ void load_count_quad(const uint32_t *p, uint64_t i, uint64_t end, bool vec, uint32_t (&v)[4]) {
    if (vec && i + 3 < end) {
        const uint4 q = *reinterpret_cast<const uint4 *>(p + i);
        v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
    } else {
        for (int t = 0; t < 4; ++t) v[t] = i + t < end ? p[i + t] : 0;
    }
}
// mash_cluster.cu: single-linkage groups at same >= min_same; label[i] = smallest index of i's group, the
// counters (either may be NULL) = number of groups and of linked pairs i < j.  mash_cluster_check is the
// argument rule of pg_mash_cluster, which the host entry point applies before it copies anything.
int mash_cluster_check(uint64_t n, int s, uint32_t min_same);
int launch_mash_cluster(const uint32_t *d_sk, uint64_t n, int s, uint32_t min_same, uint32_t *d_label,
                        unsigned long long *d_n_groups, unsigned long long *d_n_links, cudaStream_t st);
// mash_cluster.cu: the one scan of a rows x n array of counts into the union-find forest d_parent: entry (t, j)
// with count >= min_same (>= 1) unites sketches row0 + t and col0 + j and adds one to *d_n_links; with upper only
// where col0 + j > row0 + t.
int launch_cluster_link(const uint32_t *d_counts, uint64_t rows, uint64_t n, uint64_t row0, uint64_t col0, bool upper, uint32_t min_same,
                        uint32_t *d_parent, unsigned long long *d_n_links, cudaStream_t st);
// mash_cluster.cu: one batch of a growing clustering.  plan holds the n sketches before it, d_old their labels;
// the m x s batch d_b takes ids n .. n + m - 1.  d_label (n + m entries) gets the labels of all n + m sketches,
// d_cnt[0] the links found (cross pairs counted with the batch row as the receiver, inner pairs with the lower
// row), d_cnt[1] the groups, d_cnt[2] the earlier groups absorbed into another.  d_old is only read.  Argument
// checks are the caller's.
int launch_mash_cluster_add(const DistancePlan &plan, const uint32_t *d_old, const uint32_t *d_b, uint64_t m, int s, uint32_t min_same,
                            uint32_t *d_label, unsigned long long *d_cnt, cudaStream_t st);
// mash_derep.cu: greedy representatives at same >= min_same; rep[i] = i's representative (first or, with
// PG_DEREP_NEAREST, nearest), the counter (may be NULL) = number of representatives.  mash_derep_check is the
// argument rule of pg_mash_dereplicate: the flags, then mash_cluster_check.
int mash_derep_check(uint64_t n, int s, uint32_t min_same, uint32_t flags);
int launch_mash_derep(const uint32_t *d_sk, uint64_t n, int s, uint32_t min_same, uint32_t flags, uint32_t *d_rep,
                      unsigned long long *d_n_reps, cudaStream_t st);
// distance.cu: flag[r] = 1 if sketch r is non-decreasing; *d_n_unsorted = number of other sketches
int launch_sorted_flags(const uint32_t *d_sk, uint64_t n, int s, uint8_t *d_flag, uint32_t *d_n_unsorted, cudaStream_t st);
// mash_index.cu: the top_k most similar sketches of plan's set for each of nq query sketches of size sq
// (receiver = query); outputs nq x top_k on the device, any may be NULL
constexpr uint32_t INDEX_MAX_TOP_K = 1024;
int launch_index_query(const DistancePlan &plan, const uint32_t *d_q, uint64_t nq, int sq, uint32_t top_k, uint32_t min_same,
                       uint32_t *d_ref, uint32_t *d_same, double *d_dist, uint32_t *d_n_hits, cudaStream_t st);
// mash_index.cu: every reference with same >= min_same for each query, as CSR lists in reference order: offsets
// d_off[0 .. nq] (d_off[nq] = the total), entries at positions >= cap not stored, the lists and d_total may be NULL.
// Argument rules and their order are those of pg_mash_index_query_within_dev.
int launch_index_within(const DistancePlan &plan, const uint32_t *d_q, uint64_t nq, int sq, uint32_t min_same, uint64_t *d_off,
                        uint32_t *d_ref, uint32_t *d_same, double *d_dist, uint64_t cap, uint64_t *d_total, cudaStream_t st);
// mash_index.cu: for each of nq query sketches of size sq > 0, the first reference of plan's set with same >= min_same
// (min_same >= 1; the query is the receiver) as d_rep[q] = d_ids[p], or with `nearest` the one with the largest
// same, ties to the first, as d_key[q] = same << 32 | ~d_ids[p].  d_ids ascends with p.  Rows that link to no
// reference are written 0xFFFFFFFF / 0; nothing is written when the set is empty (the caller initialises).
int launch_index_link(const DistancePlan &plan, const uint32_t *d_q, uint64_t nq, int sq, uint32_t min_same, const uint32_t *d_ids,
                      bool nearest, uint32_t *d_rep, unsigned long long *d_key, cudaStream_t st);
// mash_index.cu: for each of nq query sketches of size sq > 0, every reference p of plan's set with same >= min_same
// (min_same >= 1; the query is the receiver) united with query q as sketch first + q in the forest d_parent
// (launch_cluster_link), and the links counted into *d_n_links.  Nothing is done when the set is empty.
int launch_index_cluster(const DistancePlan &plan, const uint32_t *d_q, uint64_t nq, int sq, uint32_t min_same, uint64_t first,
                         uint32_t *d_parent, unsigned long long *d_n_links, cudaStream_t st);
// mash_derep.cu: one batch of a growing dereplication.  The m x s batch d_b takes ids base .. base + m - 1; plan
// holds the kept representatives (ids d_ids, ascending) of the rows before it.  Rows linked to a kept
// representative are seeded from it (launch_index_link), then the batch is dereplicated on its own with the seeded
// rows covered: d_rep[i] = the global id of batch row i's representative (base + i for a new one), and
// *d_n_new = the number of new representatives.  Argument checks are the caller's.
int launch_mash_derep_add(const DistancePlan &plan, const uint32_t *d_ids, const uint32_t *d_b, uint64_t m, int s, uint32_t min_same,
                          uint32_t flags, uint32_t base, uint32_t *d_rep, unsigned long long *d_n_new, cudaStream_t st);
// mash_derep.cu: the n_new rows of the batch with d_rep[i] == base + i, in order: their sketches to d_rows
// (n_new x s) and their ids to d_ids
int launch_derep_gather(const uint32_t *d_b, uint64_t m, int s, uint32_t base, const uint32_t *d_rep, uint64_t n_new, uint32_t *d_rows,
                        uint32_t *d_ids, cudaStream_t st);
// mash_screen.cu: a screen's device state.  keys: the n x s (value << 32 | id) keys of the reference words, sorted;
// vals: the D distinct values, ascending; cnt: the pool count of each value in each of the `samples` samples,
// value-major (cnt[d * samples + q]), and one sink counter after them; dir: nb + 1 entries, dir[b] = the first distinct value in bucket b of
// join_bucket over [0, vmax].
struct ScreenIndex {
    uint64_t *keys = nullptr, *dir = nullptr;
    uint32_t *vals = nullptr;
    unsigned long long *cnt = nullptr;
    uint64_t n = 0, D = 0;
    int s = 0;
    uint32_t nb = 0, vmax = 0;
    uint32_t samples = 1;
    bool canon = false;  // adds count canonical k-mers (PG_KMER_CANONICAL)
};
// Builds the screen of n reference rows of s > 0 words (any order, zero tails included) with zero counts for
// samples >= 1 samples; synchronises st.  On an error nothing of *out is allocated.
int screen_build(const uint32_t *d_sk, uint64_t n, int s, uint32_t samples, cudaStream_t st, ScreenIndex *out);
// Counts every window of reads [0, n_reads) of the ragged pool (d_bases, d_off) into ix.cnt, read i into sample
// d_ids[i] (sample 0 when d_ids is null; a read whose id is >= ix.samples counts nowhere); only enqueues, and
// reads no byte outside [d_off[0], d_off[n_reads]) whatever the offsets hold.
int screen_add(const ScreenIndex &ix, int k, const uint8_t *d_bases, const uint64_t *d_off, const uint32_t *d_ids, uint64_t n_reads,
               cudaStream_t st);
int screen_reset(const ScreenIndex &ix, cudaStream_t st);
// shared, containment and multiplicity of every reference for samples [first, first + count), row-major
// (out[(q - first) * n + r]; any output may be NULL; first + count <= ix.samples); only enqueues
int screen_results(const ScreenIndex &ix, uint32_t first, uint32_t count, uint32_t *d_shared, double *d_cont, uint64_t *d_mult,
                   cudaStream_t st);
// the same three arrays over the words each value's winner-take-all vote gave their reference: a value a sample holds
// goes to the reference that holds it with the largest first-pass shared of that sample (ties to the smallest id);
// only enqueues
int screen_winners(const ScreenIndex &ix, uint32_t first, uint32_t count, uint32_t *d_shared, double *d_cont, uint64_t *d_mult,
                   cudaStream_t st);
void screen_free(ScreenIndex &ix, cudaStream_t st);
// sketch_groups.cu: row g of d_out (row_stride words, zeroed past its count) = the smallest min(q_g, s) distinct window
// hashes of group g's records [d_goff[g], d_goff[g + 1]) that occur at least m times, ascending; d_count[g] = how many.
// canon: canonical k-mers (PG_KMER_CANONICAL).  Decides its passes on the host, so it synchronises st.  Argument checks
// are the caller's.
int sketch_groups(const uint8_t *d_bases, const uint64_t *d_off, uint64_t n_records, const uint64_t *d_goff, uint64_t n_groups, int k, int s,
                  uint32_t m, bool canon, uint32_t *d_out, uint64_t row_stride, uint32_t *d_count, cudaStream_t st);
// The state of a grouped sketch grown in place (pg_mash_sketcher): per group g its cap C_g and every value v < C_g
// seen so far with min(c_g(v), m), ascending in segment [seg[g], seg[g + 1]) of val / cnt.  The host keeps seg and
// cap too, to plan the passes.
struct SketcherState {
    uint64_t G = 0, B = 0;  // groups, most values a group keeps
    int k = 0, s = 0;
    uint32_t m = 1;
    bool canon = false;  // canonical k-mers (PG_KMER_CANONICAL)
    std::vector<uint64_t> seg, cap;
    uint32_t *d_val = nullptr, *d_cnt = nullptr;  // seg[G] entries
    uint64_t *d_seg = nullptr, *d_cap = nullptr;  // G + 1 and G
};
// an empty state of G groups (every cap 2^32); synchronises st
int sketcher_init(SketcherState &S, cudaStream_t st);
// Adds records [d_goff[i], d_goff[i + 1]) of the batch to group first + i, i < nb (d_goff[0] = 0, d_goff[nb] =
// n_records).  Builds the new state in new buffers and takes it only on success; synchronises st.
int sketcher_add(SketcherState &S, const uint8_t *d_bases, const uint64_t *d_off, uint64_t n_records, const uint64_t *d_goff, uint64_t first,
                 uint64_t nb, cudaStream_t st);
// rows [first, first + count): the first s qualifying values of each state segment, then zeros to row_stride, their
// number, complete and held (either may be null); only enqueues
int sketcher_rows(const SketcherState &S, uint64_t first, uint64_t count, uint32_t *d_out, uint64_t row_stride, uint32_t *d_n, uint8_t *d_complete,
                  uint64_t *d_held, cudaStream_t st);
void sketcher_free(SketcherState &S, cudaStream_t st);
// mash_dist.cu: Mash distance of a block of queries against references (pg_mash_dist / pg_mash_dist_within).  Query q of
// the block is global query q0 + q; rows are row-major at `stride` words, count[i] values each (<= s, ascending).
// q_len / r_len are read only when a p-value is needed.  Dense: outputs at q * nr + r (each may be null).  List: the
// pairs with distance <= max_distance and p <= max_p_value (r > q0 + q with upper) go to slots of an atomic counter, the
// first cap of them stored.
struct DistArgs {
    const uint32_t *q_rows, *q_count, *r_rows, *r_count;
    uint64_t nq, nr, stride, q0;
    int s, k;
    const uint64_t *q_len, *r_len;
    uint32_t *common, *denom;
    double *distance, *p_value;
    double max_distance, max_p_value;
    bool upper;
    uint32_t *pair_q, *pair_r;
    uint64_t cap;
    unsigned long long *n_pairs;
};
// only enqueues
int launch_mash_dist(const DistArgs &g, bool list, cudaStream_t st);
// Alignment launchers: the scoring (byte LUTs, table, gap, local / global) is an AlignScoring of host
// pointers (align_core.cuh).
struct AlignScoring;
// sw_score.cu
int launch_sw_score(const uint8_t *d_q, const uint64_t *d_qoff, uint64_t nq, uint64_t max_qlen, const uint8_t *d_t, uint64_t tlen,
                    int query_is_a, const AlignScoring &s, int64_t *d_score, int32_t *d_err, int64_t *d_errpos, cudaStream_t st);
// sw_align.cu (score + aligned strings; queries <= 64 symbols, 32-bit scores)
int launch_sw_align(const uint8_t *d_q, const uint64_t *d_qoff, uint64_t nq, uint64_t max_qlen, const uint8_t *d_t, uint64_t tlen,
                    int query_is_a, const AlignScoring &s, int64_t *d_score, int32_t *d_err, int64_t *d_errpos, uint8_t *d_align_a,
                    uint8_t *d_align_b, uint64_t out_stride, uint32_t *d_len, int32_t *d_status, cudaStream_t st);
// sw_align_long.cu (both strings longer than 64 symbols: full matrix in HBM).  With d_toff, item k
// aligns query d_pq[k] against template d_pt[k] of the ragged set (d_t, d_toff) and tlen is the
// longest template; without it every query meets the one template d_t[0, tlen).
int launch_sw_align_long(const uint8_t *d_q, const uint64_t *d_qoff, uint64_t nq, uint64_t max_qlen, const uint8_t *d_t,
                         uint64_t tlen, int query_is_a, const AlignScoring &s, const int64_t *d_score, const int32_t *d_err,
                         uint8_t *d_align_a, uint8_t *d_align_b, uint64_t out_stride, uint32_t *d_len, int32_t *d_status,
                         cudaStream_t st, const uint64_t *d_toff = nullptr, const uint32_t *d_pq = nullptr,
                         const uint32_t *d_pt = nullptr);
// sw_pairs.cu: scores of n_pairs (A[d_pa[k]], B[d_pb[k]]) pairs; only enqueues work on st
int launch_sw_score_pairs(const uint8_t *d_a, const uint64_t *d_aoff, uint64_t na, uint64_t max_la, const uint8_t *d_b,
                          const uint64_t *d_boff, uint64_t nb, uint64_t max_lb, const uint32_t *d_pa, const uint32_t *d_pb,
                          uint64_t n_pairs, const AlignScoring &s, int64_t *d_score, int32_t *d_err, int64_t *d_errpos,
                          cudaStream_t st);
// tm.cu
int launch_tm(const uint8_t *d_bases, const uint64_t *d_off, uint64_t n, double cp, double na,
              double mg, double *d_tm, double *d_dh, double *d_ds, int32_t *d_status,
              cudaStream_t st);
int launch_design_primers(const uint8_t *d_bases, const uint64_t *d_off, uint64_t n, double target,
                          uint32_t *d_fwd, uint32_t *d_rev, int32_t *d_status, cudaStream_t st);
int launch_minimal_primer(const uint8_t *d_bases, const uint64_t *d_off, uint64_t n, double target,
                          uint32_t *d_min_len, int32_t *d_status, cudaStream_t st);
// find_sites.cu
int launch_find_sites(const uint8_t *d_seqs, const uint64_t *d_seq_off, uint64_t n_seq, uint64_t total_bytes,
                      const uint8_t *d_pats, const uint64_t *d_pat_off, uint32_t n_pat, uint64_t pat_bytes, uint32_t flags,
                      uint32_t *d_hit_seq, uint64_t *d_hit_pos, uint32_t *d_hit_pat, uint64_t cap,
                      unsigned long long *d_n_hits, cudaStream_t st);
// fastq_ingest.cu
int launch_fastq_ingest(const uint8_t *d_text, uint64_t nbytes, uint8_t *d_bases, uint64_t bases_cap,
                        uint64_t *d_offsets, uint64_t records_cap, uint64_t *n_records,
                        uint64_t *total_bases, int32_t *err_code, uint64_t *err_line, cudaStream_t st,
                        uint64_t *d_spans = nullptr);
// fasta_ingest.cu
int launch_fasta_ingest(const uint8_t *d_text, uint64_t nbytes, uint32_t max_line_size, uint32_t flags,
                        uint8_t *d_bases, uint64_t bases_cap, uint64_t *d_offsets, uint8_t *d_names,
                        uint64_t names_cap, uint64_t *d_name_offsets, uint64_t records_cap, uint64_t *n_records,
                        uint64_t *total_bases, uint64_t *total_name_bytes, int32_t *err_code, uint64_t *err_line,
                        cudaStream_t st);
// seqhash.cu: digests (n x 32 bytes), error codes and positions of pg_seqhash_batch for sequences of at most
// max_len bytes, total = off[n] - off[0]
int launch_seqhash(const uint8_t *d_in, const uint64_t *d_off, uint64_t n, uint64_t max_len, uint64_t total, int seq_type,
                   uint32_t flags, uint8_t *d_digest, int32_t *d_err, uint64_t *d_pos, cudaStream_t st);
int launch_least_rotation(const uint8_t *d_in, const uint64_t *d_off, uint64_t n, uint64_t max_len, uint64_t *d_rotation,
                          cudaStream_t st);
// fold.cu: per-item device scratch of pg_fold_zuker_batch (0 for items that are not folded), the DNA and RNA
// energy tables at temp degrees Celsius (uploaded as is), and the kernel over items [0, n)
uint64_t fold_scratch_bytes(uint64_t len);
std::vector<uint8_t> fold_tables(double temp);
int launch_fold_zuker(const uint8_t *d_seqs, const uint64_t *d_off, uint64_t n, const uint8_t *d_tables, uint8_t *d_scratch,
                      const uint64_t *d_scr_off, double *d_mfe, uint8_t *d_db, uint64_t *d_db_len, int32_t *d_status, cudaStream_t st);
// fragment.cu: poly's synthesis/fragment.  fragment_host turns the batch-wide exclude and include lists
// into what the kernel reads (the fidelity table, R and the keys of the excludes, the A/C/G/T masks and the
// other 4-byte words with their reverse complements); fragment_max_ends bounds an item's fragment count.
struct FragmentHost {
    std::vector<uint8_t> fid;  // the kernel's table: 120 x 120 counts, then the code -> key map
    std::vector<long long> r_ex;
    std::vector<uint32_t> ex_mask, inc_mask, ex_other, inc_other;
    std::vector<uint8_t> ex_keys;
};
struct FragmentArgs {
    const uint8_t *seqs;
    const uint64_t *off;
    uint64_t n;
    int64_t min_size, max_size;
    const uint8_t *fid;
    const long long *r_ex;
    const uint32_t *ex_mask, *inc_mask;
    const uint8_t *ex_keys;
    uint64_t n_ex_keys;
    const uint32_t *ex_other, *inc_other;
    uint64_t n_ex_other, n_inc_other;
    int has_include;
    uint32_t *scratch;  // set by launch_fragment
    uint64_t slot_words;
    int32_t *status;
    double *eff;
    int64_t *err_min, *err_max;
    uint64_t *n_ends, *ends;    // item i's ends at ends[ends_off[i] ..], room for fragment_max_ends(L_i)
    const uint64_t *ends_off;
};
struct SetArgs {
    const uint8_t *fid;
    const uint8_t *ov;          // overhang bytes, indexed with ov_off
    const uint64_t *ov_off, *set_off;
    uint64_t first, n_sets;     // sets first .. first + n_sets; outputs are indexed from 0
    int next;                   // 0: SetEfficiency, 1: NextOverhangs
    uint8_t *scratch;           // set by launch_overhang_sets
    uint64_t slot_bytes;
    double *eff;                // n_sets (SetEfficiency) or n_sets x 256 (NextOverhangs)
    uint8_t *cands;             // n_sets x 256 x 4
    uint32_t *n_cands;
};
uint64_t fragment_max_ends(uint64_t len);
FragmentHost fragment_host(const uint8_t *ex, const uint64_t *ex_off, uint64_t n_ex, const uint8_t *inc, const uint64_t *inc_off, uint64_t n_inc);
int launch_fragment(FragmentArgs a, uint64_t max_len, uint64_t scratch_budget, StreamScratch &tmp, cudaStream_t st);
int launch_fragment_compact(const uint64_t *d_region, const uint64_t *d_region_off, const uint64_t *d_n_ends, const uint64_t *d_out_off, uint64_t n,
                            uint64_t *d_out, cudaStream_t st);
// max_keys: the most keyed members of any set in the launch
int launch_overhang_sets(SetArgs a, uint64_t max_keys, uint64_t scratch_budget, StreamScratch &tmp, cudaStream_t st);
// synth.cu
int launch_synth_reads(uint8_t *d_bases, uint64_t first_read, uint64_t n_reads, uint32_t read_len,
                       uint64_t seed, int kind, uint32_t family, cudaStream_t st);

}  // namespace pg
