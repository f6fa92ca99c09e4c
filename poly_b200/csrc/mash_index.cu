// mash_index.cu -- K3 index queries: for each sketch of a query batch, the top_k most similar sketches of a
// stored reference set (receiver = query, mash.go:107-135), ranked on the device.
//
// The reference set is a DistancePlan (distance.cu): sortedness flags and, when every reference is ascending,
// the bucketed (value, id) join index of distance_join.cu.  A query batch is cut into row blocks whose dense
// matching-count accumulator [rows][n] fits a memory budget; each block runs
//   index_probe_kernel    ascending query x join index: for every distinct query value v (multiplicity cq),
//                         binary search of v's bucket and min(cq, cr) for each reference id of v's run (cr its
//                         multiplicity) -- same = sum over values of min(c_q, c_r), exact for ascending pairs
//                         of any sizes because the range early-out only fires when that sum is 0;
//   index_pairwise_kernel the other rows (an unsorted query, an unsorted reference, or a set the join declined):
//                         query tile x reference tile in shared memory with the literal size / early-out / walk
//                         rules of distance_block_kernel;
//   index_select_kernel   one CTA per row: exact top_k by (same desc, reference index asc) with a count
//                         histogram, a threshold count and an index-ordered pass over the ties.
// Radius queries (launch_index_within) consume the same blocks with two other kernels:
//   index_within_count_kernel  one CTA per row: the number of counts >= min_same, scanned in place into the
//                              CSR offsets (the entry before the block already holds the earlier blocks' total);
//   index_within_fill_kernel   one CTA per row: an index-ordered compaction of the row into its CSR slice.
// A growing dereplication (launch_index_link) seeds a batch from its kept representatives with a third:
//   index_link_kernel<Nearest> one CTA per row: the first reference (or the closest, ties to the first) with
//                              same >= min_same, written as the row's assignment or nearest key.
// A growing clustering (launch_index_cluster) unites each batch row with every reference it links to with a
// fourth, the scan of mash_cluster.cu (launch_cluster_link without its upper-triangle rule: each entry of the
// block is one pair of a batch row and an earlier sketch).
#include <algorithm>
#include <cstdlib>

#include <cub/device/device_scan.cuh>

#include "common.cuh"

namespace pg {

namespace {

constexpr int PROBE_THREADS = 128;
constexpr int PAIR_BT = 8;            // sketches per tile side of the pairwise kernel
constexpr int SEL_THREADS = 256;
constexpr int SEL_BITS = 12;          // histogram digit: counts are selected 12 bits at a time
constexpr int SEL_BINS = 1 << SEL_BITS;
constexpr uint32_t NO_REF = 0xffffffffu;

// One CTA per query row of the block; rows whose query is not ascending are left to the pairwise kernel.
// Lanes search 32 distinct query values at once, then the warp walks each found run with its lanes along the
// run, so the reductions of one instruction go to neighbouring words of the accumulator row.
__global__ void __launch_bounds__(PROBE_THREADS)
index_probe_kernel(const uint32_t *__restrict__ q, uint32_t sq, uint64_t row0, const uint8_t *__restrict__ qflag,
                   const uint64_t *__restrict__ entries, const uint64_t *__restrict__ start, uint32_t nb,
                   const uint32_t *__restrict__ vmax_p, uint64_t n, uint32_t *__restrict__ acc) {
    const uint64_t row = row0 + blockIdx.x;
    if (!qflag[row]) return;
    const uint32_t *Q = q + row * sq;
    uint32_t *A = acc + (uint64_t)blockIdx.x * n;
    const uint32_t vmax = *vmax_p;
    const uint64_t scale = join_bucket_scale(nb, vmax);
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    for (uint32_t base = warp * 32; base < sq; base += PROBE_THREADS) {
        const uint32_t i = base + lane;
        bool found = false;
        uint64_t p = 0, hi = 0;
        uint32_t v = 0, cq = 0;
        if (i < sq) {
            v = __ldg(Q + i);
            if ((i == 0 || __ldg(Q + i - 1) != v) && v <= vmax) {  // head of a value; larger values match nothing
                cq = 1;
                while (i + cq < sq && __ldg(Q + i + cq) == v) ++cq;
                const uint32_t b = join_bucket(v, scale, nb);
                uint64_t lo = start[b];
                hi = start[b + 1];
                const uint64_t key = (uint64_t)v << 32;
                uint64_t h = hi;
                while (lo < h) { const uint64_t m = (lo + h) >> 1; if (__ldg(entries + m) < key) lo = m + 1; else h = m; }
                p = lo;
                found = p < hi && (uint32_t)(__ldg(entries + p) >> 32) == v;
            }
        }
        uint32_t pending = __ballot_sync(0xffffffffu, found);
        while (pending) {
            const int src = __ffs(pending) - 1;
            pending &= pending - 1;
            const uint64_t r0 = __shfl_sync(0xffffffffu, p, src), r1 = __shfl_sync(0xffffffffu, hi, src);
            const uint32_t rv = __shfl_sync(0xffffffffu, v, src), rc = __shfl_sync(0xffffffffu, cq, src);
            for (uint64_t c0 = r0;; c0 += 32) {
                const uint64_t pos = c0 + lane;
                const uint64_t k = pos < r1 ? __ldg(entries + pos) : ~0ull;
                const bool in = pos < r1 && (uint32_t)(k >> 32) == rv;
                if (in && (pos == r0 || __ldg(entries + pos - 1) != k)) {  // head of a (value, id) group
                    uint32_t cr = 1;
                    while (pos + cr < r1 && __ldg(entries + pos + cr) == k) ++cr;
                    atomicAdd(A + (uint32_t)k, min(rc, cr));
                }
                if (__ballot_sync(0xffffffffu, in) != 0xffffffffu) break;  // the run ended inside this chunk
            }
        }
    }
}

// Query tile x reference tile, both staged in shared memory; one warp per pair.  Receiver = query: the larger
// sketch by SketchSize, the query on ties (mash.go:109-115).  Rows the probe kernel serves are skipped.
__global__ void __launch_bounds__(256)
index_pairwise_kernel(const uint32_t *__restrict__ q, uint32_t sq, uint64_t row0, uint64_t row_end,
                      const uint8_t *__restrict__ qflag, int probe_sorted, const uint32_t *__restrict__ ref, uint64_t n,
                      uint32_t sr, const uint8_t *__restrict__ rflag, uint32_t *__restrict__ acc) {
    extern __shared__ __align__(16) uint32_t tile[];  // queries [BT][sq] then references [BT][sr]
    uint32_t *sqt = tile, *srt = tile + (size_t)PAIR_BT * sq;
    const uint64_t q0 = row0 + (uint64_t)blockIdx.y * PAIR_BT;
    const uint64_t c0 = (uint64_t)blockIdx.x * PAIR_BT;
    const uint32_t nr = (uint32_t)min((uint64_t)PAIR_BT, row_end - q0);
    const uint32_t nc = (uint32_t)min((uint64_t)PAIR_BT, n - c0);
    const bool Qlarge = sq >= sr;
    const uint32_t sl = Qlarge ? sq : sr, ss = Qlarge ? sr : sq;
    // mash.go:117-119 needs only the first and last word of each sketch: skip the staging when every pair of
    // the tile early-outs (always the case for zero-padded fill-regime sketches) -- the accumulator is zeroed
    {
        bool work = false;
        if (threadIdx.x < nr * nc) {
            const uint32_t ri = threadIdx.x / nc, ci = threadIdx.x % nc;
            if (!(probe_sorted && qflag[q0 + ri])) {
                const uint32_t *Qs = q + (q0 + ri) * sq, *Rs = ref + (c0 + ci) * sr;
                const uint32_t *L = Qlarge ? Qs : Rs, *S = Qlarge ? Rs : Qs;
                work = !(__ldg(L + sl - 1) < __ldg(S) || __ldg(S + ss - 1) < __ldg(L));
            }
        }
        if (!__syncthreads_or(work)) return;
    }
    for (uint32_t i = threadIdx.x; i < nr * sq; i += blockDim.x) sqt[i] = __ldg(q + q0 * sq + i);
    for (uint32_t i = threadIdx.x; i < nc * sr; i += blockDim.x) srt[i] = __ldg(ref + c0 * sr + i);
    __syncthreads();
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u, nwarps = blockDim.x >> 5;
    for (uint32_t pr = warp; pr < nr * nc; pr += nwarps) {
        const uint32_t ri = pr / nc, ci = pr % nc;
        if (probe_sorted && qflag[q0 + ri]) continue;
        const uint32_t *Qs = sqt + (size_t)ri * sq, *Rs = srt + (size_t)ci * sr;
        const uint32_t *L = Qlarge ? Qs : Rs, *S = Qlarge ? Rs : Qs;
        uint32_t same = 0;
        if (!(L[sl - 1] < S[0] || S[ss - 1] < L[0])) {  // mash.go:117
            if (qflag[q0 + ri] && rflag[c0 + ci]) {
                // element i of S (its t-th copy) matches iff L holds more than t copies of its value
                uint32_t local = 0;
                for (uint32_t i = lane; i < ss; i += 32) {
                    const uint32_t v = S[i];
                    uint32_t lo = 0, hi = i;
                    while (lo < hi) { const uint32_t m = (lo + hi) >> 1; if (S[m] < v) lo = m + 1; else hi = m; }
                    const uint32_t t = i - lo;
                    uint32_t l0 = 0, l1 = sl;
                    while (l0 < l1) { const uint32_t m = (l0 + l1) >> 1; if (L[m] < v) l0 = m + 1; else l1 = m; }
                    if (l0 + t < sl && L[l0 + t] == v) ++local;
                }
                for (int d = 16; d > 0; d >>= 1) local += __shfl_xor_sync(0xffffffffu, local, d);
                same = local;
            } else if (lane == 0) {  // literal walk, mash.go:121-132
                uint32_t si = 0, li = 0;
                while (si < ss && li < sl) {
                    const uint32_t a = S[si], b = L[li];
                    if (a == b) { ++same; ++si; ++li; }
                    else if (a < b) ++si;
                    else ++li;
                }
            }
        }
        if (lane == 0 && same) acc[(q0 + ri - row0) * n + (c0 + ci)] = same;
    }
}

// Bins of a SEL_BINS histogram from the top: the bin where the running count from above reaches `want`
// (*bin) and the count strictly above it (*above).  All threads of the CTA call it.
__device__ void hist_cut(const uint32_t *hist, uint32_t want, uint32_t *s_part, uint32_t *bin, uint32_t *above) {
    constexpr int PER = SEL_BINS / SEL_THREADS;
    const uint32_t t = threadIdx.x, lane = t & 31u, warp = t >> 5;
    uint32_t mine = 0;
    for (int j = 0; j < PER; ++j) mine += hist[t * PER + j];
    // exclusive suffix sum over threads: counts in the bins of threads > t
    uint32_t incl = mine;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t y = __shfl_down_sync(0xffffffffu, incl, d);
        if (lane + d < 32) incl += y;
    }
    if (lane == 0) s_part[warp] = incl;
    __syncthreads();
    uint32_t cum = incl - mine;
    for (uint32_t w = warp + 1; w < SEL_THREADS / 32; ++w) cum += s_part[w];
    for (int j = PER - 1; j >= 0; --j) {
        const uint32_t h = hist[t * PER + j];
        if (cum < want && cum + h >= want) { *bin = t * PER + j; *above = cum; }
        cum += h;
    }
    __syncthreads();
}

// One CTA per query row: the references with same >= min_same, ordered by same descending and then index
// ascending, cut to top_k.  The threshold count t is found digit by digit (12 bits of the count per level,
// counts are <= den); every reference above t is taken, and the ties at t in index order until top_k is full.
__global__ void __launch_bounds__(SEL_THREADS)
index_select_kernel(const uint32_t *__restrict__ acc, uint64_t n, uint64_t row0, uint32_t den, uint32_t top_k,
                    uint32_t min_same, uint32_t *__restrict__ hit_ref, uint32_t *__restrict__ hit_same,
                    double *__restrict__ hit_dist, uint32_t *__restrict__ n_hits) {
    __shared__ uint32_t hist[SEL_BINS];
    __shared__ uint64_t key[INDEX_MAX_TOP_K];  // (UINT32_MAX - same) << 32 | ref: ascending = output order
    __shared__ uint32_t s_part[SEL_THREADS / 32];
    __shared__ uint32_t s_bin, s_above, s_taken, s_ties;
    const uint32_t *A = acc + (uint64_t)blockIdx.x * n;
    const uint64_t row = row0 + blockIdx.x;
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    // levels: digit shift 12 when counts can reach 2^12, then 0 (den < 2^24 is checked by the launcher)
    uint32_t t = 0, need = top_k, prefix = 0, prefix_shift = 32;
    bool take_all = false;
    for (int shift = den >= (uint32_t)SEL_BINS ? SEL_BITS : 0; shift >= 0; shift -= SEL_BITS) {
        for (uint32_t i = threadIdx.x; i < SEL_BINS; i += SEL_THREADS) hist[i] = 0;
        __syncthreads();
        for (uint64_t j0 = 0; j0 < n; j0 += SEL_THREADS) {
            const uint64_t j = j0 + threadIdx.x;
            const uint32_t c = j < n ? A[j] : 0;
            if (j < n && c >= min_same && (prefix_shift >= 32 || (c >> prefix_shift) == prefix)) {
                const uint32_t b = (c >> shift) & (SEL_BINS - 1);
                const uint32_t peers = __match_any_sync(__activemask(), b);  // mostly one bin (count 0) per warp
                if ((int)lane == __ffs(peers) - 1) atomicAdd(&hist[b], __popc(peers));
            }
        }
        __syncthreads();
        if (threadIdx.x == 0) { s_bin = NO_REF; s_above = 0; }
        __syncthreads();
        hist_cut(hist, need, s_part, &s_bin, &s_above);
        if (s_bin == NO_REF) {  // fewer than `need` candidates left: take every one of them
            take_all = true;
            break;
        }
        need -= s_above;
        prefix = (prefix_shift >= 32 ? 0 : prefix << SEL_BITS) | s_bin;
        prefix_shift = shift;
        t = prefix;
        __syncthreads();
    }
    // take_all: every count >= min_same (at most top_k of them); else every count > t and `need` ties at t
    const uint32_t lo_cut = take_all ? min_same : t;
    if (take_all) need = 0xffffffffu;
    if (threadIdx.x == 0) { s_taken = 0; s_ties = 0; }
    __syncthreads();
    for (uint64_t j0 = 0; j0 < n; j0 += SEL_THREADS) {
        const uint64_t j = j0 + threadIdx.x;
        const uint32_t c = j < n ? A[j] : 0;
        const bool ok = j < n && c >= min_same;
        const bool gt = ok && c > lo_cut, eq = ok && c == lo_cut;
        // index-ordered rank of the ties of this chunk
        const uint32_t eb = __ballot_sync(0xffffffffu, eq);
        if (lane == 0) s_part[warp] = __popc(eb);
        __syncthreads();
        uint32_t rank = s_ties + __popc(eb & ((1u << lane) - 1u)), total = 0;
        for (uint32_t w = 0; w < SEL_THREADS / 32; ++w) { if (w < warp) rank += s_part[w]; total += s_part[w]; }
        if (gt || (eq && rank < need)) key[atomicAdd(&s_taken, 1u)] = ((uint64_t)(0xffffffffu - c) << 32) | (uint32_t)j;
        __syncthreads();
        if (threadIdx.x == 0) s_ties += total;
        __syncthreads();
    }
    const uint32_t m = s_taken;  // <= top_k
    uint32_t P = 1;
    while (P < m) P <<= 1;
    for (uint32_t i = m + threadIdx.x; i < P; i += SEL_THREADS) key[i] = ~0ull;
    __syncthreads();
    block_bitonic_sort<uint64_t, SEL_THREADS>(key, P);
    for (uint32_t i = threadIdx.x; i < top_k; i += SEL_THREADS) {
        const uint64_t o = row * top_k + i;
        const uint32_t same = i < m ? 0xffffffffu - (uint32_t)(key[i] >> 32) : 0;
        if (hit_ref) hit_ref[o] = i < m ? (uint32_t)key[i] : NO_REF;
        if (hit_same) hit_same[o] = same;
        if (hit_dist) hit_dist[o] = i < m ? 1 - (double)same / (double)den : 1.0;  // mash.go:134,139
    }
    if (threadIdx.x == 0 && n_hits) n_hits[row] = m;
}

// One CTA per query row: off[row + 1] = the number of references with same >= min_same (min_same >= 1, so the
// zeros load_count_quad returns past n never count).
__global__ void __launch_bounds__(SEL_THREADS)
index_within_count_kernel(const uint32_t *__restrict__ acc, uint64_t n, uint64_t row0, uint32_t min_same, uint64_t *__restrict__ off) {
    __shared__ uint32_t s_part[SEL_THREADS / 32];
    const uint32_t *A = acc + (uint64_t)blockIdx.x * n;
    const bool vec = (n & 3) == 0;
    uint32_t c = 0;
    for (uint64_t j = 4ull * threadIdx.x; j < n; j += 4ull * SEL_THREADS) {
        uint32_t v[4];
        load_count_quad(A, j, n, vec, v);
#pragma unroll
        for (int t = 0; t < 4; ++t) c += v[t] >= min_same;
    }
    for (int d = 16; d > 0; d >>= 1) c += __shfl_xor_sync(0xffffffffu, c, d);
    if ((threadIdx.x & 31u) == 0) s_part[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint64_t total = 0;
        for (int w = 0; w < SEL_THREADS / 32; ++w) total += s_part[w];
        off[row0 + blockIdx.x + 1] = total;
    }
}

// One CTA per query row: the references with same >= min_same in index order, stored from off[row] on; only
// positions below cap are written.  Each thread takes four neighbouring counts of a chunk, so a thread's hits are
// consecutive: a warp scan of the per-thread counts, the warps' totals in shared memory and a running base (the
// same for every thread) give each hit its position.
__global__ void __launch_bounds__(SEL_THREADS)
index_within_fill_kernel(const uint32_t *__restrict__ acc, uint64_t n, uint64_t row0, uint32_t den, uint32_t min_same,
                         const uint64_t *__restrict__ off, uint64_t cap, uint32_t *__restrict__ hit_ref, uint32_t *__restrict__ hit_same,
                         double *__restrict__ hit_dist) {
    __shared__ uint32_t s_part[SEL_THREADS / 32];
    const uint32_t *A = acc + (uint64_t)blockIdx.x * n;
    const uint64_t row = row0 + blockIdx.x;
    const uint64_t end = min(off[row + 1], cap);
    uint64_t base = off[row];
    if (base >= end) return;  // an empty list, or one wholly past the cap
    const bool vec = (n & 3) == 0;
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    for (uint64_t j0 = 0; j0 < n; j0 += 4ull * SEL_THREADS) {
        const uint64_t j = j0 + 4ull * threadIdx.x;
        uint32_t v[4];
        load_count_quad(A, j, n, vec, v);
        uint32_t mask = 0;
#pragma unroll
        for (int t = 0; t < 4; ++t) mask |= (uint32_t)(v[t] >= min_same) << t;
        const uint32_t mine = __popc(mask);
        uint32_t incl = mine;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t y = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= (uint32_t)d) incl += y;
        }
        if (lane == 31) s_part[warp] = incl;
        __syncthreads();
        uint64_t pos = base + incl - mine;
        uint32_t total = 0;
        for (uint32_t w = 0; w < SEL_THREADS / 32; ++w) { if (w < warp) pos += s_part[w]; total += s_part[w]; }
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            if (!((mask >> t) & 1u)) continue;
            if (pos < end) {
                if (hit_ref) hit_ref[pos] = (uint32_t)(j + t);
                if (hit_same) hit_same[pos] = v[t];
                if (hit_dist) hit_dist[pos] = 1 - (double)v[t] / (double)den;  // mash.go:134,139
            }
            ++pos;
        }
        base += total;
        if (base >= end) break;  // the rest of the row lies past the cap (base is the same in every thread)
        __syncthreads();         // s_part is read before the next chunk writes it
    }
}

// One CTA per query row: the best reference with same >= min_same as a 64-bit key, larger is better.  First
// mode: 1 << 32 | ~p, so the smallest position p wins, and the scan stops after the first chunk that holds one;
// nearest: same << 32 | ~p, the largest count and then the smallest position.  ids[p] is position p's id and
// ascends with p, so position order is id order.  Row `row` gets rep[row] = ids[p] (first; 0xFFFFFFFF when
// nothing links) or key[row] = same << 32 | ~ids[p] (nearest; 0 when nothing links): the slots derep_walk_kernel
// reads as "covered by an earlier representative".
template <bool Nearest>
__global__ void __launch_bounds__(SEL_THREADS)
index_link_kernel(const uint32_t *__restrict__ acc, uint64_t n, uint64_t row0, uint32_t min_same, const uint32_t *__restrict__ ids,
                  uint32_t *__restrict__ rep, unsigned long long *__restrict__ key) {
    __shared__ unsigned long long s_part[SEL_THREADS / 32];
    const uint32_t *A = acc + (uint64_t)blockIdx.x * n;
    const uint64_t row = row0 + blockIdx.x;
    const bool vec = (n & 3) == 0;
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    unsigned long long best = 0;  // min_same >= 1: the zeros load_count_quad returns past n never count
    for (uint64_t j0 = 0; j0 < n; j0 += 4ull * SEL_THREADS) {
        const uint64_t j = j0 + 4ull * threadIdx.x;
        uint32_t v[4];
        load_count_quad(A, j, n, vec, v);
#pragma unroll
        for (int t = 0; t < 4; ++t)
            if (v[t] >= min_same) best = max(best, (unsigned long long)(Nearest ? v[t] : 1u) << 32 | (uint32_t)~(j + t));
        if (!Nearest && __syncthreads_or(best != 0)) break;  // the loop bounds are the same in every thread
    }
    for (int d = 16; d > 0; d >>= 1) best = max(best, (unsigned long long)__shfl_xor_sync(0xffffffffu, best, d));
    if (lane == 0) s_part[warp] = best;
    __syncthreads();
    if (threadIdx.x != 0) return;
    for (int w = 0; w < SEL_THREADS / 32; ++w) best = max(best, s_part[w]);
    const uint32_t id = best ? ids[~(uint32_t)best] : NO_REF;
    if (Nearest) key[row] = best ? (best & ~0xffffffffull) | (uint32_t)~id : 0ull;
    else rep[row] = id;
}

// The accumulation loop of both query kinds (nq > 0, sq > 0): the queries' sortedness (the one host sync), the
// probe / pairwise choice, and row blocks whose dense [rows][n] counts fit a 2 GiB budget.  consume(acc, rb, re)
// runs once the counts of rows [rb, re) are enqueued into acc; the first code other than PG_OK is the result.
int index_blocks(const DistancePlan &plan, const uint32_t *d_q, uint64_t nq, int sq, cudaStream_t st,
                 const std::function<int(const uint32_t *acc, uint64_t rb, uint64_t re)> &consume) {
    const uint64_t n = plan.n;
    const uint32_t sr = (uint32_t)plan.s;
    StreamScratch sc(st);
    uint8_t *d_qflag = nullptr;
    uint32_t *d_unsorted = nullptr;
    PG_CUDA(sc.alloc(&d_qflag, nq));
    PG_CUDA(sc.alloc(&d_unsorted, 1));
    { const int rc_ = launch_sorted_flags(d_q, nq, sq, d_qflag, d_unsorted, st); if (rc_ != PG_OK) return rc_; }
    uint32_t n_unsorted = 0;
    PG_CUDA(cudaMemcpyAsync(&n_unsorted, d_unsorted, 4, cudaMemcpyDeviceToHost, st));
    PG_CUDA(cudaStreamSynchronize(st));
    // ascending queries against a joined set take the probe, every other row the pairwise kernel
    const bool probe = n && plan.join.ok && n_unsorted < nq;
    const bool pairwise = n && (!plan.join.ok || n_unsorted > 0);
    const size_t pair_smem = (size_t)PAIR_BT * ((size_t)sq + sr) * 4;
    if (pairwise) {
        if (pair_smem > 200 * 1024) {
            set_error("sketch sizes %d + %u too large for the pairwise tile kernel", sq, sr);
            return PG_ERR_UNSUPPORTED;
        }
        const int rc_ = func_smem((const void *)index_pairwise_kernel, pair_smem);
        if (rc_ != PG_OK) return rc_;
    }
    // row blocks: the accumulator of a block is rows x n words, within 2 GiB; each block costs one pass of the
    // join index's buckets per query value (probe) or of the reference tiles (pairwise), independent of rows
    const uint64_t budget_words = 512ull << 20;
    uint64_t rows_per = std::max<uint64_t>(1, std::min<uint64_t>(nq, n ? budget_words / n : nq));
    if (const char *e = getenv("PG_INDEX_QUERY_ROWS")) rows_per = std::max<uint64_t>(1, std::min<uint64_t>(rows_per, strtoull(e, nullptr, 10)));
    rows_per = std::min<uint64_t>(rows_per, 65535ull * PAIR_BT);  // one pairwise launch per block (gridDim.y)
    uint32_t *d_acc = nullptr;
    PG_CUDA(sc.alloc(&d_acc, rows_per * n));
    for (uint64_t rb = 0; rb < nq; rb += rows_per) {
        const uint64_t re = std::min(nq, rb + rows_per), rows = re - rb;
        if (n) PG_CUDA(cudaMemsetAsync(d_acc, 0, rows * n * 4, st));
        if (probe) {
            index_probe_kernel<<<(unsigned)rows, PROBE_THREADS, 0, st>>>(d_q, (uint32_t)sq, rb, d_qflag, plan.join.entries, plan.join.start,
                                                                         (uint32_t)plan.join.nb, plan.join.vmax, n, d_acc);
            PG_LAUNCH_CHECK("index_probe_kernel");
        }
        if (pairwise) {
            const uint64_t gx = (n + PAIR_BT - 1) / PAIR_BT;
            if (gx > 0x7fffffffull) { set_error("too many reference sketches"); return PG_ERR_ARG; }
            dim3 grid((unsigned)gx, (unsigned)((rows + PAIR_BT - 1) / PAIR_BT));
            index_pairwise_kernel<<<grid, 256, pair_smem, st>>>(d_q, (uint32_t)sq, rb, re, d_qflag, plan.join.ok ? 1 : 0, plan.d_sk, n, sr,
                                                                 plan.d_flag, d_acc);
            PG_LAUNCH_CHECK("index_pairwise_kernel");
        }
        const int rc_ = consume(d_acc, rb, re);
        if (rc_ != PG_OK) return rc_;
    }
    return PG_OK;
}

}  // namespace

int launch_index_query(const DistancePlan &plan, const uint32_t *d_q, uint64_t nq, int sq, uint32_t top_k, uint32_t min_same,
                       uint32_t *d_ref, uint32_t *d_same, double *d_dist, uint32_t *d_n_hits, cudaStream_t st) {
    if (top_k == 0 || top_k > INDEX_MAX_TOP_K) {
        set_error("top_k %u outside [1, %u]", top_k, INDEX_MAX_TOP_K);
        return PG_ERR_ARG;
    }
    if (nq == 0) return PG_OK;
    if (sq <= 0) {
        set_error("query sketches of size %d: the reference panics (Sketches[-1])", sq);
        return PG_ERR_PANIC;
    }
    const uint64_t n = plan.n;
    const uint32_t den = std::min<uint32_t>((uint32_t)sq, (uint32_t)plan.s);
    if (n && den >= (1u << 24)) { set_error("sketch size %u above the selection's 2^24 limit", den); return PG_ERR_UNSUPPORTED; }
    return index_blocks(plan, d_q, nq, sq, st, [&](const uint32_t *d_acc, uint64_t rb, uint64_t re) {
        index_select_kernel<<<(unsigned)(re - rb), SEL_THREADS, 0, st>>>(d_acc, n, rb, std::max<uint32_t>(den, 1), top_k, min_same, d_ref,
                                                                         d_same, d_dist, d_n_hits);
        PG_LAUNCH_CHECK("index_select_kernel");
        return PG_OK;
    });
}

int launch_index_within(const DistancePlan &plan, const uint32_t *d_q, uint64_t nq, int sq, uint32_t min_same, uint64_t *d_off,
                        uint32_t *d_ref, uint32_t *d_same, double *d_dist, uint64_t cap, uint64_t *d_total, cudaStream_t st) {
    if (min_same == 0) {
        set_error("min_same 0 would list all %llu x %llu pairs", (unsigned long long)nq, (unsigned long long)plan.n);
        return PG_ERR_ARG;
    }
    if (nq == 0) {
        if (d_off) PG_CUDA(cudaMemsetAsync(d_off, 0, 8, st));
        if (d_total) PG_CUDA(cudaMemsetAsync(d_total, 0, 8, st));
        return PG_OK;
    }
    if (sq <= 0) {
        set_error("query sketches of size %d: the reference panics (Sketches[-1])", sq);
        return PG_ERR_PANIC;
    }
    if (!d_off) { set_error("null hit_offsets"); return PG_ERR_ARG; }
    const uint64_t n = plan.n;
    const uint32_t den = std::max<uint32_t>(std::min<uint32_t>((uint32_t)sq, (uint32_t)plan.s), 1);
    StreamScratch sc(st);
    uint8_t *d_scan = nullptr;  // CUB's scan storage, allocated for the first block (the largest)
    size_t have = 0;
    PG_CUDA(cudaMemsetAsync(d_off, 0, 8, st));
    const int rc = index_blocks(plan, d_q, nq, sq, st, [&](const uint32_t *d_acc, uint64_t rb, uint64_t re) {
        const unsigned rows = (unsigned)(re - rb);
        index_within_count_kernel<<<rows, SEL_THREADS, 0, st>>>(d_acc, n, rb, min_same, d_off);
        PG_LAUNCH_CHECK("index_within_count_kernel");
        // d_off[rb] holds the total of the rows before the block: the inclusive scan makes the counts global offsets
        size_t bytes = 0;
        PG_CUDA(cub::DeviceScan::InclusiveSum(nullptr, bytes, d_off + rb, d_off + rb, (int64_t)rows + 1, st));
        if (bytes > have) {
            PG_CUDA(sc.alloc(&d_scan, bytes));
            have = bytes;
        }
        PG_CUDA(cub::DeviceScan::InclusiveSum(d_scan, bytes, d_off + rb, d_off + rb, (int64_t)rows + 1, st));
        index_within_fill_kernel<<<rows, SEL_THREADS, 0, st>>>(d_acc, n, rb, den, min_same, d_off, cap, d_ref, d_same, d_dist);
        PG_LAUNCH_CHECK("index_within_fill_kernel");
        return PG_OK;
    });
    if (rc != PG_OK) return rc;
    if (d_total) PG_CUDA(cudaMemcpyAsync(d_total, d_off + nq, 8, cudaMemcpyDeviceToDevice, st));
    return PG_OK;
}

int launch_index_link(const DistancePlan &plan, const uint32_t *d_q, uint64_t nq, int sq, uint32_t min_same, const uint32_t *d_ids,
                      bool nearest, uint32_t *d_rep, unsigned long long *d_key, cudaStream_t st) {
    if (nq == 0 || plan.n == 0) return PG_OK;
    const uint64_t n = plan.n;
    return index_blocks(plan, d_q, nq, sq, st, [&](const uint32_t *d_acc, uint64_t rb, uint64_t re) {
        if (nearest) {
            index_link_kernel<true><<<(unsigned)(re - rb), SEL_THREADS, 0, st>>>(d_acc, n, rb, min_same, d_ids, d_rep, d_key);
            PG_LAUNCH_CHECK("index_link_kernel<true>");
        } else {
            index_link_kernel<false><<<(unsigned)(re - rb), SEL_THREADS, 0, st>>>(d_acc, n, rb, min_same, d_ids, d_rep, d_key);
            PG_LAUNCH_CHECK("index_link_kernel<false>");
        }
        return PG_OK;
    });
}

int launch_index_cluster(const DistancePlan &plan, const uint32_t *d_q, uint64_t nq, int sq, uint32_t min_same, uint64_t first,
                         uint32_t *d_parent, unsigned long long *d_n_links, cudaStream_t st) {
    if (nq == 0 || plan.n == 0) return PG_OK;
    const uint64_t n = plan.n;
    return index_blocks(plan, d_q, nq, sq, st, [&](const uint32_t *d_acc, uint64_t rb, uint64_t re) {
        return launch_cluster_link(d_acc, re - rb, n, first + rb, 0, false, min_same, d_parent, d_n_links, st);
    });
}

}  // namespace pg
