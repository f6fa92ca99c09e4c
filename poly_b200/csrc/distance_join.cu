// distance_join.cu -- K3 fast path: all-pairs matching counts over ASCENDING sketches as an
// inverted-index join instead of N^2 pairwise merges.
//
// For two ascending sketches the reference's walk (/root/reference/search/mash/mash.go:121-132)
// counts sum over values v of min(cnt_A(v), cnt_B(v)) (SURVEY.md 8a a5), and its early-out
// (mash.go:117-119) only fires when that sum is 0 anyway.  So
//     same[i][j] = sum over values v present in both i and j of min(c_i(v), c_j(v))
// and the whole matrix is the sum over values of the outer product of that value's posting
// list.  Work is N*s + (number of matching pairs), not N^2*s:
//   1. histogram of value buckets over all N*s (value, sketch id) entries
//   2. exclusive scan of the bucket counts
//   3. scatter of the entries into their buckets
//   4. one CTA per bucket: sort the bucket's entries by (value, id) in shared memory, collapse
//      duplicates into (id, count), and for every run of one value add min(count_a, count_b)
//      to same[a][b] for all a in the row block, b in the run (global atomics).
// Buckets are value ranges scaled to the largest value present, sized for ~2k entries.  If the
// data is so skewed that a bucket cannot fit shared memory even with the finest bucketing, the
// caller falls back to the pairwise kernel (distance.cu).
#include <algorithm>
#include <cstdlib>
#include <vector>

#include <cub/device/device_merge.cuh>
#include <cub/device/device_radix_sort.cuh>

#include "common.cuh"

namespace pg {

namespace {

constexpr int JOIN_CAP = 4096;      // entries a bucket CTA can hold (32 KB of keys + 24 KB of run tables)
constexpr int JOIN_SMEM = JOIN_CAP * (8 + 3 * 2);
constexpr int JOIN_THREADS = 256;

__global__ void max_value_kernel(const uint32_t *__restrict__ sk, uint64_t n, uint32_t s,
                                 uint32_t *__restrict__ vmax) {
    // ascending rows: the maximum of a row is its last element
    uint32_t m = 0;
    for (uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (uint64_t)gridDim.x * blockDim.x)
        m = max(m, __ldg(sk + r * s + (s - 1)));
    for (int d = 16; d > 0; d >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, d));
    if ((threadIdx.x & 31) == 0) atomicMax(vmax, m);
}

// the value of a sketch word, or of a (value << 32 | id) join key
__device__ __forceinline__ uint32_t join_value(uint32_t v) { return v; }
__device__ __forceinline__ uint32_t join_value(uint64_t key) { return (uint32_t)(key >> 32); }

// bucket counts of `total` values: the words of a sketch set (join_build) or the keys of a merged index (join_merge)
template <typename T>
__global__ void hist_kernel(const T *__restrict__ src, uint64_t total, const uint32_t *__restrict__ vmax,
                            uint32_t nbuckets, uint32_t *__restrict__ hist) {
    const uint64_t scale = join_bucket_scale(nbuckets, *vmax);
    for (uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t b = join_bucket(join_value(__ldg(src + e)), scale, nbuckets);
        // consecutive elements of an ascending row mostly share a bucket: aggregate per warp
        const uint32_t peers = __match_any_sync(__activemask(), b);
        if ((int)(threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&hist[b], __popc(peers));
    }
}

// single-CTA exclusive scan (nbuckets <= 2^22); also reports the largest bucket
__global__ void scan_kernel(const uint32_t *__restrict__ hist, uint32_t nbuckets, uint64_t *__restrict__ start,
                            uint32_t *__restrict__ largest) {
    __shared__ uint64_t s_part[1024];
    __shared__ uint32_t s_max[1024];
    const uint32_t tid = threadIdx.x, per = (nbuckets + 1023) / 1024;
    const uint32_t lo = min(tid * per, nbuckets), hi = min(lo + per, nbuckets);
    uint64_t sum = 0;
    uint32_t mx = 0;
    for (uint32_t i = lo; i < hi; ++i) { sum += hist[i]; mx = max(mx, hist[i]); }
    s_part[tid] = sum;
    s_max[tid] = mx;
    __syncthreads();
    if (tid == 0) {
        uint64_t run = 0;
        uint32_t m = 0;
        for (int i = 0; i < 1024; ++i) { const uint64_t t = s_part[i]; s_part[i] = run; run += t; m = max(m, s_max[i]); }
        *largest = m;
        start[nbuckets] = run;
    }
    __syncthreads();
    uint64_t run = s_part[tid];
    for (uint32_t i = lo; i < hi; ++i) { start[i] = run; run += hist[i]; }
}

// The keys (v << 32 | id0 + row) of `total` words of rows of s words, and their largest value into *vmax.
__global__ void batch_keys_kernel(const uint32_t *__restrict__ sk, uint64_t total, uint32_t s, uint64_t id0,
                                  uint64_t *__restrict__ keys, uint32_t *__restrict__ vmax) {
    uint32_t m = 0;
    for (uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t v = __ldg(sk + e);
        keys[e] = ((uint64_t)v << 32) | (id0 + e / s);
        m = max(m, v);
    }
    for (int d = 16; d > 0; d >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, d));
    if ((threadIdx.x & 31) == 0) atomicMax(vmax, m);
}

// Merge-path cut points of the merge of the sorted keys a[0, na) and b[0, nb) (no key in both): cut[k] = the
// number of a's keys among the first min(k * piece, na + nb) keys of the merged order.
__global__ void merge_cuts_kernel(const uint64_t *__restrict__ a, uint64_t na, const uint64_t *__restrict__ b, uint64_t nb, uint64_t piece,
                                  uint64_t ncuts, uint64_t *__restrict__ cut) {
    for (uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; k < ncuts; k += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t d = min(k * piece, na + nb);
        uint64_t lo = d > nb ? d - nb : 0, hi = min(d, na);
        while (lo < hi) {
            const uint64_t mid = (lo + hi) >> 1;
            if (a[mid] < b[d - 1 - mid]) lo = mid + 1;
            else hi = mid;
        }
        cut[k] = lo;
    }
}

__global__ void scatter_kernel(const uint32_t *__restrict__ sk, uint64_t total, uint32_t s,
                               const uint32_t *__restrict__ vmax, uint32_t nbuckets,
                               const uint64_t *__restrict__ start, uint32_t *__restrict__ cursor,
                               uint64_t *__restrict__ entries) {
    const uint64_t scale = join_bucket_scale(nbuckets, *vmax);
    for (uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t v = __ldg(sk + e);
        const uint32_t id = (uint32_t)(e / s);
        const uint32_t b = join_bucket(v, scale, nbuckets);
        const uint32_t peers = __match_any_sync(__activemask(), b);
        const int leader = __ffs(peers) - 1;
        uint32_t base = 0;
        if ((int)(threadIdx.x & 31) == leader) base = atomicAdd(&cursor[b], __popc(peers));
        base = __shfl_sync(peers, base, leader);
        const uint32_t rank = __popc(peers & ((1u << (threadIdx.x & 31)) - 1u));
        entries[start[b] + base + rank] = ((uint64_t)v << 32) | id;
    }
}

// One CTA per value bucket, once per index: sort the bucket's (value << 32 | id) keys in shared memory and
// write them back, so that every later row-block pass only loads them.
__global__ void __launch_bounds__(JOIN_THREADS)
bucket_sort_kernel(uint64_t *__restrict__ entries, const uint64_t *__restrict__ start, uint32_t nbuckets) {
    extern __shared__ __align__(16) uint64_t key[];  // [JOIN_CAP]
    for (uint32_t b = blockIdx.x; b < nbuckets; b += gridDim.x) {
        const uint64_t lo = start[b];
        const uint32_t m = (uint32_t)(start[b + 1] - lo);
        if (m < 2) continue;
        uint32_t P = 1;
        while (P < m) P <<= 1;
        for (uint32_t i = threadIdx.x; i < P; i += JOIN_THREADS) key[i] = i < m ? entries[lo + i] : ~0ull;
        __syncthreads();
        block_bitonic_sort<uint64_t, JOIN_THREADS>(key, P);
        for (uint32_t i = threadIdx.x; i < m; i += JOIN_THREADS) entries[lo + i] = key[i];
        __syncthreads();
    }
}

// One CTA per value bucket: load the bucket's sorted (value, id) keys, then every value run of g >= 2 distinct
// ids contributes min(c_a, c_b) to same[a][b] for its ordered pairs a != b (the diagonal is s for every
// ascending sketch and is written by diag_kernel).  Emission is warp-cooperative: for one row a the lanes
// run ALONG the run, i.e. along row a of the matrix, so the reductions of one instruction fall into
// neighbouring words (ids of a run are ascending; related sketches tend to have neighbouring ids) and
// coalesce into few L2 transactions instead of 32.
__global__ void __launch_bounds__(JOIN_THREADS)
bucket_join_kernel(const uint64_t *__restrict__ entries, const uint64_t *__restrict__ start, uint32_t nbuckets,
                   uint64_t n, uint64_t row_begin, uint64_t row_end, uint32_t *__restrict__ same) {
    extern __shared__ __align__(16) uint64_t key[];                  // [JOIN_CAP] sorted (value << 32 | id)
    uint16_t *rs = reinterpret_cast<uint16_t *>(key + JOIN_CAP);     // [JOIN_CAP] first position of my value run
    uint16_t *re = rs + JOIN_CAP;                                    // [JOIN_CAP] one past its last position
    uint16_t *mult = re + JOIN_CAP;                                  // [JOIN_CAP] multiplicity at a (value, id) head, 0 elsewhere
    __shared__ uint32_t s_scan[2 * (JOIN_THREADS / 32)];
    __shared__ uint32_t s_next;
    const uint32_t lane = threadIdx.x & 31u;
    for (uint32_t b = blockIdx.x; b < nbuckets; b += gridDim.x) {
        const uint64_t lo = start[b];
        const uint32_t m = (uint32_t)(start[b + 1] - lo);
        if (m == 0) continue;
        for (uint32_t i = threadIdx.x; i < m; i += JOIN_THREADS) key[i] = entries[lo + i];  // sorted by bucket_sort_kernel
        __syncthreads();
        // run bounds by two scans over the head flags of the value runs (a run of g ids used to be walked by
        // ONE thread: g serial steps with 31 idle lanes), multiplicities by a short forward look (duplicates
        // of one (value, id) are rare)
        {
            constexpr int PER = JOIN_CAP / JOIN_THREADS;  // 16 consecutive positions per thread
            const uint32_t p0 = threadIdx.x * PER;
            const uint32_t lane_ = threadIdx.x & 31u, warp_ = threadIdx.x >> 5;
            // forward: rs[i] = last run head at or before i
            uint32_t last = 0;
            bool any = false;
            for (int t = 0; t < PER; ++t) {
                const uint32_t i = p0 + t;
                if (i < m && (i == 0 || (uint32_t)(key[i - 1] >> 32) != (uint32_t)(key[i] >> 32))) { last = i; any = true; }
            }
            uint32_t carry = any ? last + 1 : 0;  // 0 = no head in my span (positions are >= 0: shift by one)
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const uint32_t y = __shfl_up_sync(0xffffffffu, carry, d);
                if ((int)lane_ >= d) carry = max(carry, y);
            }
            if (lane_ == 31) s_scan[warp_] = carry;
            uint32_t before = __shfl_up_sync(0xffffffffu, carry, 1);
            if (lane_ == 0) before = 0;
            __syncthreads();
            for (uint32_t w = 0; w < warp_; ++w) before = max(before, s_scan[w]);
            uint32_t run_head = before ? before - 1 : 0;
            for (int t = 0; t < PER; ++t) {
                const uint32_t i = p0 + t;
                if (i >= m) break;
                if (i == 0 || (uint32_t)(key[i - 1] >> 32) != (uint32_t)(key[i] >> 32)) run_head = i;
                rs[i] = (uint16_t)run_head;
                uint32_t c = 0;
                if (i == 0 || key[i - 1] != key[i]) {  // head of a (value, id) group
                    c = 1;
                    while (i + c < m && key[i + c] == key[i]) ++c;
                }
                mult[i] = (uint16_t)c;
            }
            __syncthreads();
            // backward: re[i] = first run head after i (m if none)
            uint32_t nxt = m;
            for (int t = PER - 1; t >= 0; --t) {
                const uint32_t i = p0 + t;
                if (i < m && rs[i] == i) nxt = i;  // smallest head in my span
            }
            uint32_t c2 = nxt;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const uint32_t y = __shfl_down_sync(0xffffffffu, c2, d);
                if ((int)lane_ + d < 32) c2 = min(c2, y);
            }
            if (lane_ == 0) s_scan[8 + warp_] = c2;
            uint32_t after = __shfl_down_sync(0xffffffffu, c2, 1);
            if (lane_ == 31) after = m;
            __syncthreads();
            for (uint32_t w = warp_ + 1; w < JOIN_THREADS / 32; ++w) after = min(after, s_scan[8 + w]);
            uint32_t next_head = after;
            for (int t = PER - 1; t >= 0; --t) {
                const uint32_t i = p0 + t;
                if (i >= m) continue;
                re[i] = (uint16_t)next_head;
                if (rs[i] == i) next_head = i;
            }
            if (threadIdx.x == 0) s_next = 0;
        }
        __syncthreads();
        // emission, one value run at a time: chunks of 32 positions are handed out dynamically (runs cluster: a
        // static split leaves most warps waiting at the barrier); the warp that owns a run's first position serves
        // the whole run.  The b side of a 32-wide tile sits in registers (lane = one member), the a side is
        // broadcast member by member with shuffles, so one (a, tile) step is a handful of instructions and its
        // reductions go to neighbouring words of row a.
        for (;;) {
            uint32_t chunk = 0;
            if (lane == 0) chunk = atomicAdd(&s_next, 1u);
            chunk = __shfl_sync(0xffffffffu, chunk, 0);
            const uint32_t c0 = chunk * 32u;
            if (c0 >= m) break;
            const uint32_t pos = c0 + lane;
            uint32_t heads = __ballot_sync(0xffffffffu, pos < m && rs[pos] == pos && (uint32_t)re[pos] - pos > mult[pos]);  // runs with >= 2 members
            while (heads) {
                const uint32_t h = c0 + (__ffs(heads) - 1);
                heads &= heads - 1;
                const uint32_t r0 = h, r1 = re[h];
                for (uint32_t b0 = r0; b0 < r1; b0 += 32) {       // tile of b members in registers
                    const uint32_t jb = b0 + lane;
                    const uint32_t cb = jb < r1 ? mult[jb] : 0u;
                    const uint32_t idb = jb < r1 ? (uint32_t)key[jb] : 0u;
                    for (uint32_t a0 = r0; a0 < r1; a0 += 32) {   // tile of a members, broadcast one by one
                        const uint32_t ja = a0 + lane;
                        const uint32_t ca_l = ja < r1 ? mult[ja] : 0u;
                        const uint32_t ida_l = ja < r1 ? (uint32_t)key[ja] : 0u;
                        uint32_t amask = __ballot_sync(0xffffffffu, ca_l != 0 && ida_l >= row_begin && ida_l < row_end);
                        while (amask) {
                            const uint32_t src = __ffs(amask) - 1;
                            amask &= amask - 1;
                            const uint32_t ca = __shfl_sync(0xffffffffu, ca_l, src);
                            const uint32_t ida = __shfl_sync(0xffffffffu, ida_l, src);
                            if (cb != 0 && idb != ida)  // a (value, id) group never pairs with itself
                                atomicAdd(same + (ida - row_begin) * n + idb, min(ca, cb));
                        }
                    }
                }
            }
        }
        __syncthreads();
    }
}

// same[a][a] = s: the walk of a sketch against itself matches every element (ascending sketches only)
__global__ void diag_kernel(uint32_t *__restrict__ same, uint64_t n, uint64_t row_begin, uint64_t row_end, uint32_t s) {
    for (uint64_t r = row_begin + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; r < row_end; r += (uint64_t)gridDim.x * blockDim.x)
        same[(r - row_begin) * n + r] = s;
}

__global__ void same_to_distance_kernel(const uint32_t *__restrict__ same, uint64_t count, uint32_t s,
                                        double *__restrict__ dist) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (uint64_t)gridDim.x * blockDim.x)
        dist[i] = 1 - (double)same[i] / (double)s;  // mash.go:134,139
}

// the first bucket count tried for `total` entries: ~2k entries a bucket, at most 2^22 buckets
uint64_t join_first_nb(uint64_t total) {
    uint64_t nb = 1;
    while (nb * 2048 < total) nb <<= 1;
    return std::min<uint64_t>(nb, 1u << 22);
}

}  // namespace

int launch_batch_keys(const uint32_t *d_sk, uint64_t total, uint32_t s, uint64_t id0, uint64_t *d_keys, uint32_t *d_vmax, cudaStream_t st) {
    if (total == 0) return PG_OK;
    batch_keys_kernel<<<(unsigned)std::min<uint64_t>((total + 255) / 256, (uint64_t)sm_count() * 16), 256, 0, st>>>(d_sk, total, s, id0, d_keys, d_vmax);
    PG_LAUNCH_CHECK("batch_keys_kernel");
    return PG_OK;
}

// Builds the bucketed (value, id) index of n ascending sketches.  ix->ok == false means "not
// applicable" (skewed data: a bucket would not fit shared memory) and the caller must use the
// pairwise kernel.
int join_build(const uint32_t *d_sk, uint64_t n, int s, cudaStream_t st, JoinIndex *ix) {
    ix->ok = false; ix->entries = nullptr; ix->start = nullptr; ix->vmax = nullptr; ix->nb = 0; ix->n = n; ix->s = s;
    const uint64_t total = n * (uint64_t)s;
    if (total == 0 || n > 0xffffffffull) return PG_OK;
    uint32_t *d_scalars = nullptr;  // [0] vmax, [1] largest bucket
    PG_CUDA(cudaMallocAsync(&d_scalars, 8, st));
    PG_CUDA(cudaMemsetAsync(d_scalars, 0, 8, st));
    const unsigned sms = (unsigned)sm_count();
    max_value_kernel<<<sms * 4, 256, 0, st>>>(d_sk, n, (uint32_t)s, d_scalars);
    note_launch("max_value_kernel");
    uint64_t nb = join_first_nb(total);
    for (int attempt = 0; attempt < 3 && !ix->ok; ++attempt) {
        uint32_t *d_hist = nullptr, *d_cursor = nullptr;
        uint64_t *d_start = nullptr;
        PG_CUDA(cudaMallocAsync(&d_hist, nb * 4, st));
        PG_CUDA(cudaMallocAsync(&d_cursor, nb * 4, st));
        PG_CUDA(cudaMallocAsync(&d_start, (nb + 1) * 8, st));
        PG_CUDA(cudaMemsetAsync(d_hist, 0, nb * 4, st));
        PG_CUDA(cudaMemsetAsync(d_cursor, 0, nb * 4, st));
        hist_kernel<uint32_t><<<sms * 16, 256, 0, st>>>(d_sk, total, d_scalars, (uint32_t)nb, d_hist);
        note_launch("hist_kernel");
        scan_kernel<<<1, 1024, 0, st>>>(d_hist, (uint32_t)nb, d_start, d_scalars + 1);
        note_launch("scan_kernel");
        uint32_t largest = 0;
        PG_CUDA(cudaMemcpyAsync(&largest, d_scalars + 1, 4, cudaMemcpyDeviceToHost, st));
        PG_CUDA(cudaStreamSynchronize(st));
        if (largest <= JOIN_CAP) {
            uint64_t *d_entries = nullptr;
            PG_CUDA(cudaMallocAsync(&d_entries, total * 8, st));
            scatter_kernel<<<sms * 16, 256, 0, st>>>(d_sk, total, (uint32_t)s, d_scalars, (uint32_t)nb, d_start, d_cursor, d_entries);
            note_launch("scatter_kernel");
            { const int rc_ = func_smem((const void *)bucket_sort_kernel, JOIN_CAP * 8); if (rc_ != PG_OK) return rc_; }
            bucket_sort_kernel<<<(unsigned)std::min<uint64_t>(nb, (uint64_t)sms * 24), JOIN_THREADS, JOIN_CAP * 8, st>>>(d_entries, d_start, (uint32_t)nb);
            note_launch("bucket_sort_kernel");
            ix->entries = d_entries; ix->start = d_start; ix->nb = nb; ix->largest = largest; ix->ok = true;
        } else {
            cudaFreeAsync(d_start, st);
        }
        cudaFreeAsync(d_hist, st);
        cudaFreeAsync(d_cursor, st);
        if (!ix->ok) {
            if (nb >= (1u << 22)) break;
            nb = std::min<uint64_t>(nb * 8, 1u << 22);
        }
    }
    if (ix->ok) ix->vmax = d_scalars;  // the bucket scale, for lookups of values that are not in the set
    else cudaFreeAsync(d_scalars, st);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(e, "distance join build", __FILE__, __LINE__);
    return PG_OK;
}

// The index of n + m ascending sketches from old's n and the m rows of d_batch (ascending, ids n .. n + m - 1):
// the batch's keys sorted, merged with old's entries (the entries are globally sorted by key, bucket after bucket,
// and no batch key equals an old one), then bucketed afresh for the new total with the first-choice bucket count
// and vmax = max(old, batch).  Buckets are not bounded by JOIN_CAP: the probe searches them in global memory, and
// join_emit refuses such an index.  CUB's merge counts keys in int, so the merged order is cut into pieces of at
// most 2^31 - 1 keys (PG_JOIN_MERGE_PIECE: fewer) at merge-path cut points, each merged by one call; reading the
// cut points is one more synchronisation when there is more than one piece.  old is not changed; on an error
// nothing of *out remains allocated.  One synchronisation at the end, to read the largest bucket.
int join_merge(const JoinIndex &old, const uint32_t *d_batch, uint64_t m, cudaStream_t st, JoinIndex *out) {
    *out = JoinIndex();
    const uint64_t T = old.n * (uint64_t)old.s, M = m * (uint64_t)old.s, total = T + M;
    uint64_t piece = 0x7fffffffull;
    if (const char *e = getenv("PG_JOIN_MERGE_PIECE")) piece = std::max<uint64_t>(1, std::min<uint64_t>(piece, strtoull(e, nullptr, 10)));
    StreamScratch tmp(st), keep(st);  // keep: the new index's buffers, released unless the merge succeeds
    const uint64_t nb = join_first_nb(total);
    uint64_t *d_entries = nullptr, *d_start = nullptr, *d_keys = nullptr, *d_sorted = nullptr;
    uint32_t *d_scalars = nullptr, *d_hist = nullptr;  // [0] vmax, [1] largest bucket
    PG_CUDA(keep.alloc(&d_entries, total));
    PG_CUDA(keep.alloc(&d_start, nb + 1));
    PG_CUDA(keep.alloc(&d_scalars, 2));
    PG_CUDA(tmp.alloc(&d_keys, M));
    PG_CUDA(tmp.alloc(&d_sorted, M));
    PG_CUDA(tmp.alloc(&d_hist, nb));
    PG_CUDA(cudaMemcpyAsync(d_scalars, old.vmax, 4, cudaMemcpyDeviceToDevice, st));
    PG_CUDA(cudaMemsetAsync(d_scalars + 1, 0, 4, st));
    PG_CUDA(cudaMemsetAsync(d_hist, 0, nb * 4, st));
    const unsigned sms = (unsigned)sm_count();
    { const int rc_ = launch_batch_keys(d_batch, M, (uint32_t)old.s, old.n, d_keys, d_scalars, st); if (rc_ != PG_OK) return rc_; }
    size_t bytes = 0, have = 0;
    uint8_t *d_cub = nullptr;
    PG_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, bytes, d_keys, d_sorted, M, 0, 64, st));
    PG_CUDA(tmp.alloc(&d_cub, bytes));
    have = bytes;
    PG_CUDA(cub::DeviceRadixSort::SortKeys(d_cub, bytes, d_keys, d_sorted, M, 0, 64, st));
    // piece k of the merged order is old.entries[cut[k], cut[k + 1]) and d_sorted[k * piece - cut[k], ...)
    const uint64_t pieces = (total + piece - 1) / piece;
    std::vector<uint64_t> cut(pieces + 1);
    cut[0] = 0;
    cut[pieces] = T;
    if (pieces > 1) {
        uint64_t *d_cut = nullptr;
        PG_CUDA(tmp.alloc(&d_cut, pieces + 1));
        merge_cuts_kernel<<<(unsigned)std::min<uint64_t>((pieces + 256) / 256, (uint64_t)sms * 4), 256, 0, st>>>(old.entries, T, d_sorted, M, piece,
                                                                                                                pieces + 1, d_cut);
        PG_LAUNCH_CHECK("merge_cuts_kernel");
        PG_CUDA(cudaMemcpyAsync(cut.data(), d_cut, (pieces + 1) * 8, cudaMemcpyDeviceToHost, st));
        PG_CUDA(cudaStreamSynchronize(st));
    }
    for (uint64_t k = 0; k < pieces; ++k) {
        const uint64_t d0 = k * piece, d1 = std::min(total, d0 + piece);
        const uint64_t a0 = cut[k], a1 = cut[k + 1], b0 = d0 - a0, b1 = d1 - a1;
        PG_CUDA(cub::DeviceMerge::MergeKeys(nullptr, bytes, old.entries + a0, (int)(a1 - a0), d_sorted + b0, (int)(b1 - b0), d_entries + d0,
                                            ::cuda::std::less<uint64_t>(), st));
        if (bytes > have) {
            PG_CUDA(tmp.alloc(&d_cub, bytes));
            have = bytes;
        }
        PG_CUDA(cub::DeviceMerge::MergeKeys(d_cub, bytes, old.entries + a0, (int)(a1 - a0), d_sorted + b0, (int)(b1 - b0), d_entries + d0,
                                            ::cuda::std::less<uint64_t>(), st));
    }
    hist_kernel<uint64_t><<<sms * 16, 256, 0, st>>>(d_entries, total, d_scalars, (uint32_t)nb, d_hist);
    PG_LAUNCH_CHECK("hist_kernel");
    scan_kernel<<<1, 1024, 0, st>>>(d_hist, (uint32_t)nb, d_start, d_scalars + 1);
    PG_LAUNCH_CHECK("scan_kernel");
    uint32_t largest = 0;
    PG_CUDA(cudaMemcpyAsync(&largest, d_scalars + 1, 4, cudaMemcpyDeviceToHost, st));
    PG_CUDA(cudaStreamSynchronize(st));
    out->entries = d_entries; out->start = d_start; out->vmax = d_scalars;
    out->nb = nb; out->n = old.n + m; out->s = old.s; out->largest = largest; out->ok = true;
    keep.ptr.clear();
    return PG_OK;
}

// Rows [row_begin, row_end) of the matching-count matrix from a built index.
int join_emit(const JoinIndex &ix, uint64_t row_begin, uint64_t row_end, uint32_t *d_same, double *d_dist, cudaStream_t st) {
    if (ix.largest > JOIN_CAP) {  // a merged index (join_merge): its buckets need not fit bucket_join_kernel's tile
        set_error("join index bucket of %llu entries exceeds the join kernel's %d", (unsigned long long)ix.largest, JOIN_CAP);
        return PG_ERR_UNSUPPORTED;
    }
    const uint64_t rows = row_end - row_begin;
    const unsigned sms = (unsigned)sm_count();
    PG_CUDA(cudaMemsetAsync(d_same, 0, rows * ix.n * 4, st));
    { const int rc_ = func_smem((const void *)bucket_join_kernel, JOIN_SMEM); if (rc_ != PG_OK) return rc_; }
    bucket_join_kernel<<<(unsigned)std::min<uint64_t>(ix.nb, (uint64_t)sms * 16), JOIN_THREADS, JOIN_SMEM, st>>>(
        ix.entries, ix.start, (uint32_t)ix.nb, ix.n, row_begin, row_end, d_same);
    PG_LAUNCH_CHECK("bucket_join_kernel");
    diag_kernel<<<(unsigned)std::min<uint64_t>((rows + 255) / 256, (uint64_t)sms * 8), 256, 0, st>>>(d_same, ix.n, row_begin, row_end, (uint32_t)ix.s);
    PG_LAUNCH_CHECK("diag_kernel");
    if (d_dist) {
        same_to_distance_kernel<<<sms * 8, 256, 0, st>>>(d_same, rows * ix.n, (uint32_t)ix.s, d_dist);
        PG_LAUNCH_CHECK("same_to_distance_kernel");
    }
    return PG_OK;
}

void join_free(JoinIndex &ix, cudaStream_t st) {
    if (ix.entries) cudaFreeAsync(ix.entries, st);
    if (ix.start) cudaFreeAsync(ix.start, st);
    if (ix.vmax) cudaFreeAsync(ix.vmax, st);
    ix.entries = nullptr; ix.start = nullptr; ix.vmax = nullptr; ix.ok = false;
}

}  // namespace pg
