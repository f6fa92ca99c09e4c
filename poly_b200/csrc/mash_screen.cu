// mash_screen.cu -- the screen: for each reference sketch of a set, how many of its hashes a pool of reads
// contains and how often (Mash Screen's containment and median multiplicity, Ondov et al. 2019), counted from
// every k-mer window of the pool.
//
// Create (screen_build, once per reference set):
//   1. the (value << 32 | id) keys of the n x s reference words (launch_batch_keys), their largest value vmax;
//   2. one CUB radix sort of the keys; the D distinct values, ascending (CUB Unique), and a directory of
//      nb = ceil(D / 4) value buckets over [0, vmax] (join_bucket, the join index's mapping): dir[b] is the first
//      distinct value in bucket b, so a lookup is two directory reads and a binary search over ~4 values;
//   3. one 64-bit pool counter per distinct value and sample, zeroed.
// Several samples: every read of an add carries a sample id, and each distinct value has one counter per sample,
// value-major (cnt[d * S + q]), so a tally reads the samples of a group at one value from one line.
// Add (the hot path, screen_add): the pool's bytes are cut into fixed chunks, whatever the read lengths; a
// CTA stages a chunk (plus the k - 1 byte halo) in shared memory and each thread walks W consecutive windows
// of it with the register-ring murmur3 walk of K1 (kmer_walk.cuh).  A window hash above vmax is dropped by one
// compare, which is almost every window when the references are bottom-s sketches of large genomes.  The
// rest are checked against the read boundaries (a binary search over the offsets, then a cursor) and looked
// up; a hit takes its read's sample id and is aggregated per warp on equal counters (__match_any_sync) before one
// atomicAdd.  k outside the walk's instantiated set hashes each window from global memory.
// Results (screen_results): one pass over the sorted keys.  The c_r(v) words of reference r equal to v are one
// run of equal keys, and the first min(c_r(v), c_pool(v)) of them count; each counted word appends c_pool(v)
// to its reference's segment of s slots.  A CUB segmented sort of the segments then gives the lower median.
// Samples are tallied in groups whose slots stay under SCREEN_GROUP_SLOTS: one count pass, one segmented sort and
// one final kernel per group.
// Winners (screen_winners, Mash Screen's winner-take-all): the same count pass without the segments gives each
// reference's first-pass shared; then every value the pool holds votes among its contenders, one run of keys
// (screen_vote_kernel, per sample), and the count pass above runs again over the won words only.
// A canonical screen (PG_KMER_CANONICAL, ix.canon) adds with the CANON instantiations of the walk and generic kernels:
// windows 0 .. L - k of each read, each the smaller of itself and its reverse complement (walk_chunk.cuh).
#include <algorithm>
#include <climits>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_segmented_sort.cuh>
#include <cub/device/device_select.cuh>

#include "common.cuh"
#include "kmer_walk.cuh"
#include "murmur3.cuh"
#include "walk_chunk.cuh"

namespace pg {

namespace {

constexpr int SCREEN_THREADS = 256;
// A tally's multiplicity slots (8 bytes each, twice: unsorted and sorted) for one group of samples: the group is as
// many samples as fit, at least one.  The segmented sort counts its items in int, so the bound stays below INT_MAX.
constexpr uint64_t SCREEN_GROUP_SLOTS = 1ull << 28;
static_assert(SCREEN_GROUP_SLOTS <= (uint64_t)INT_MAX, "a sample group is one segmented sort");

// what the add and tally kernels read of a screen
struct ScreenLookup {
    const uint32_t *vals;     // [D] distinct reference values, ascending
    const uint64_t *dir;      // [nb + 1]
    unsigned long long *cnt;  // [D][samples] pool counts, value-major, then the sink
    const uint32_t *ids;      // the add's per-read sample ids; null: every read is sample 0
    uint64_t sink;            // D samples: the counter of windows whose read's id is not a sample, never read
    uint32_t nb, vmax, samples;
};

// the index d of value h among the distinct values, if h is one of them
__device__ __forceinline__ bool screen_find(const ScreenLookup &L, uint64_t scale, uint32_t h, uint64_t *d) {
    const uint32_t b = join_bucket(h, scale, L.nb);
    uint64_t lo = L.dir[b], hi = L.dir[b + 1];
    const uint64_t end = hi;
    while (lo < hi) {
        const uint64_t mid = (lo + hi) >> 1;
        if (L.vals[mid] < h) lo = mid + 1;
        else hi = mid;
    }
    *d = lo;
    return lo < end && L.vals[lo] == h;
}

// One window of every lane of a converged warp; cand: the lane's hash h is <= vmax.  With SAMPLES, a hit counts into
// its read's sample, ids[j - 1] (j: the first offset above p; sample 0 when ids is null), or into the sink when that
// id is not a sample: a select rather than one more condition on the hit, which keeps the walk kernels at their
// registers.  Without SAMPLES (one sample, no ids) d is the counter, as in a single-sample screen.  Lanes that hit
// the same counter add to it once, with their number.
template <bool SAMPLES, bool CANON>
__device__ __forceinline__ void screen_hit(const ScreenLookup &L, uint64_t scale, const uint64_t *off, uint64_t n_reads, bool cand, uint64_t p,
                                           uint32_t k, uint32_t h, uint64_t &j) {
    uint64_t d = ~0ull;
    bool hit = cand && window_in_read<CANON>(off, n_reads, p, k, j) && screen_find(L, scale, h, &d);
    if (SAMPLES && hit) {
        const uint32_t q = L.ids ? __ldg(L.ids + (j - 1)) : 0u;
        d = q < L.samples ? d * L.samples + q : L.sink;
    }

    const unsigned peers = __match_any_sync(0xffffffffu, hit ? d : ~0ull);
    if (hit && (int)(threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&L.cnt[d], (unsigned long long)__popc(peers));
}

// EMIT of the walk: the hash of window p0 + i + R_.  The vote keeps the common case (no lane has a candidate) to
// one compare and one vote per window.
#define PG_SCREEN_EMIT(R_, H_)                                                                                              \
    {                                                                                                                       \
        const bool cand_ = (H_) <= L.vmax;                                                                                  \
        if (__any_sync(0xffffffffu, cand_)) screen_hit<SAMPLES, CANON>(L, scale, off, n_reads, cand_, p0 + i + (R_), (uint32_t)K, (H_), j); \
    }

// The walk path (k in WalkKs).  Persistent CTAs take chunks of SCREEN_THREADS x W windows of the pool
// [off[0], off[n_reads]); thread t walks windows [t W, t W + W) of the chunk.  The chunk's bytes, its look-ahead
// and the 16-byte alignment head are staged in shared memory with 16-byte loads; bytes outside the pool are
// zeros and are never read from global memory.
template <int K, bool SAMPLES, bool CANON>
__global__ void __launch_bounds__(SCREEN_THREADS, 2)
screen_walk_kernel(const uint8_t *__restrict__ bases, const uint64_t *__restrict__ off, uint64_t n_reads, const ScreenLookup L,
                   uint32_t lut_stride) {
    PG_WALK_CONSTANTS;
    constexpr uint32_t W = walk_span(NB);
    constexpr uint32_t CHUNK = SCREEN_THREADS * W;
    constexpr uint32_t STAGE = CHUNK + 128;  // + head (< 16) + the walk's look-ahead (< 4 NB + 20 bytes)
    constexpr uint32_t nk = W;               // PG_KMER_STEP's bound; unchecked steps never test it
    // CANON: the complemented copy s_rc and the complement table s_comp follow the chunk
    __shared__ __align__(16) uint8_t s_in[CANON ? 2 * STAGE + 256 : STAGE];
    __shared__ __align__(16) uint32_t s_lut[LUT ? 256 : 4];
    uint8_t *s_rc = nullptr, *s_comp = nullptr;
    const uint32_t tid = threadIdx.x;
    if (LUT)
        for (uint32_t x = tid; x < 256; x += SCREEN_THREADS) s_lut[x] = g_kmix_byte.v[x];
    if constexpr (CANON) {
        s_rc = s_in + STAGE;
        s_comp = s_in + 2 * STAGE;
        for (uint32_t x = tid; x < 256; x += SCREEN_THREADS) s_comp[x] = complement((uint8_t)x);
    }
    const uint64_t lo = off[0], hi = max(off[n_reads], lo);
    const uint64_t chunks = (hi - lo + CHUNK - 1) / CHUNK;
    const uint64_t scale = join_bucket_scale(L.nb, L.vmax);
    const uint32_t lut_base = smem_u32(s_lut);

    for (uint64_t c = blockIdx.x; c < chunks; c += gridDim.x) {
        const uint64_t P0 = lo + c * CHUNK;
        const uint32_t head = chunk_head(bases, P0);
        __syncthreads();  // the previous chunk's walk is done with s_in (and, the first time, s_lut is written)
        if constexpr (CANON) stage_chunk<STAGE, SCREEN_THREADS, true>(s_in, bases, P0, head, lo, hi, s_rc, s_comp);
        else stage_chunk<STAGE, SCREEN_THREADS>(s_in, bases, P0, head, lo, hi);
        __syncthreads();

        const uint32_t b0 = head + tid * W;
        const uint32_t *sw = reinterpret_cast<const uint32_t *>(s_in) + (b0 >> 2);
        const uint32_t sh = (b0 & 3u) * 8u;
        const uint8_t *sb = s_in + b0 + 4 * NB;  // tail byte of window i is sb[i]
        const uint64_t p0 = P0 + tid * W;        // pool position of window 0
        uint64_t j = ~0ull;

        if constexpr (CANON) {
            const uint8_t *sbf = s_in + b0, *sbc = s_rc + b0;
            const uint32_t *cw = reinterpret_cast<const uint32_t *>(s_rc) + ((b0 + TAIL) >> 2);
            const uint32_t csh = ((b0 + TAIL) & 3u) * 8u;
            PG_WALK_PROLOGUE
            PG_CANON_PROLOGUE
            uint32_t i = 0;
            while (i < W) {
#pragma unroll
                for (int u = 0; u < NB; ++u) PG_KMER_STEP_CANON(u, PG_SCREEN_EMIT)
            }
        } else {
            PG_WALK_PROLOGUE
            uint32_t i = 0;
            while (i < W) {  // every lane runs the same steps, so the warp is converged at each window
#pragma unroll
                for (int u = 0; u < NB; ++u) PG_KMER_STEP(u, false, PG_SCREEN_EMIT)
            }
        }
    }
}

// Any other k (0 included, but not in canonical mode): window p of the pool is hashed from global memory by thread p
// of a CTA-uniform grid-stride loop, so that every lane of a warp runs the same iterations.
template <bool SAMPLES, bool CANON>
__global__ void __launch_bounds__(SCREEN_THREADS)
screen_generic_kernel(const uint8_t *__restrict__ bases, const uint64_t *__restrict__ off, uint64_t n_reads, uint32_t k, const ScreenLookup L) {
    const uint64_t lo = off[0], hi = max(off[n_reads], lo);
    const uint64_t scale = join_bucket_scale(L.nb, L.vmax);
    for (uint64_t base = lo + (uint64_t)blockIdx.x * SCREEN_THREADS; base < hi; base += (uint64_t)gridDim.x * SCREEN_THREADS) {
        const uint64_t p = base + threadIdx.x;
        uint32_t h = 0;
        bool cand = false;
        if (p < hi && window_fits<CANON>(hi - p, k)) {
            h = window_hash<CANON>(bases + p, k);
            cand = h <= L.vmax;
        }
        if (__any_sync(0xffffffffu, cand)) {
            uint64_t j = ~0ull;
            screen_hit<SAMPLES, CANON>(L, scale, off, n_reads, cand, p, k, h, j);
        }
    }
}

__global__ void screen_values_kernel(const uint64_t *__restrict__ keys, uint64_t total, uint32_t *__restrict__ vals) {
    for (uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (uint64_t)gridDim.x * blockDim.x)
        vals[e] = (uint32_t)(keys[e] >> 32);
}

// dir[b] = the first distinct value index in bucket b or above, for b in [0, nb]; dir[nb] = D
__global__ void screen_dir_kernel(const uint32_t *__restrict__ vals, uint64_t D, uint32_t nb, uint32_t vmax, uint64_t *__restrict__ dir) {
    const uint64_t scale = join_bucket_scale(nb, vmax);
    for (uint64_t d = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; d < D; d += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t b = join_bucket(vals[d], scale, nb);
        const uint32_t first = d ? join_bucket(vals[d - 1], scale, nb) + 1 : 0;
        for (uint32_t x = first; x <= b; ++x) dir[x] = d;  // buckets (the previous value's, b]
        if (d + 1 == D)
            for (uint64_t x = (uint64_t)b + 1; x <= nb; ++x) dir[x] = D;
    }
}

// The winner of a vote word fill << 32 | (0xFFFFFFFF - id): its largest value has the largest first-pass shared,
// ties to the smallest id.
__device__ __forceinline__ uint32_t vote_id(unsigned long long w) { return 0xFFFFFFFFu - (uint32_t)w; }

// For each sample t of the group [q0, q0 + g): entry e of the sorted keys counts when its rank in its run of equal
// keys (one reference's copies of one value, at most s long) is below the value's pool count in the sample, and,
// given a vote (win != null, [D][g]), when its reference won the value in the sample; it then appends that count to
// its reference's segment of the sample, row t n + id (mult != null).  The run start and the value index are found
// once for every sample.
__global__ void screen_count_kernel(const uint64_t *__restrict__ keys, uint64_t total, uint32_t s, const ScreenLookup L, uint32_t q0, uint32_t g,
                                    uint64_t n, const unsigned long long *__restrict__ win, uint32_t *__restrict__ fill,
                                    unsigned long long *__restrict__ mult) {
    const uint64_t scale = join_bucket_scale(L.nb, L.vmax);
    for (uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t key = keys[e];
        uint64_t lo = e >= s - 1 ? e - (s - 1) : 0, hi = e;  // the run's first entry: the lower bound of key in [e - s + 1, e]
        while (lo < hi) {
            const uint64_t mid = (lo + hi) >> 1;
            if (keys[mid] < key) lo = mid + 1;
            else hi = mid;
        }
        uint64_t d = 0;
        screen_find(L, scale, (uint32_t)(key >> 32), &d);  // every reference value is present
        const unsigned long long *cnt = L.cnt + d * L.samples + q0;
        const uint32_t id = (uint32_t)key;
        for (uint32_t t = 0; t < g; ++t) {
            const unsigned long long c = cnt[t];
            if (e - lo < c && (!win || vote_id(win[d * g + t]) == id)) {
                const uint64_t row = t * n + id;
                const uint32_t pos = atomicAdd(&fill[row], 1u);
                if (mult) mult[row * s + pos] = c;
            }
        }
    }
}

// The winner-take-all vote, for each sample t of the group [q0, q0 + g) apart.  The first entry of each (value, id)
// run whose value the sample holds proposes fill[t n + id] << 32 | (0xFFFFFFFF - id) for the value; win[d g + t]
// keeps the largest, whatever the order of the atomics.
// A value's keys are adjacent, so the lanes of a warp that hold it are consecutive: they reduce to one proposal
// (a segmented max over shuffles) before one atomic, and a proposal no larger than win[d] as read is dropped (win
// only grows, so a stale read drops nothing that could win).  A value held by every reference thus costs at most one
// atomic per warp, and far fewer once its leader is in.
__global__ void screen_vote_kernel(const uint64_t *__restrict__ keys, uint64_t total, const ScreenLookup L, uint32_t q0, uint32_t g, uint64_t n,
                                   const uint32_t *__restrict__ fill, unsigned long long *win) {
    const uint64_t scale = join_bucket_scale(L.nb, L.vmax);
    const int lane = (int)(threadIdx.x & 31);
    // a warp-uniform trip count: every lane reaches the shuffles
    for (uint64_t base = (uint64_t)blockIdx.x * blockDim.x; base < total; base += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t e = base + threadIdx.x;
        uint64_t d = ~0ull;  // past the end: a segment of its own, after every value
        uint32_t id = 0;
        bool lead = false;  // the first entry of its (value, id) run
        if (e < total) {
            const uint64_t key = keys[e];
            screen_find(L, scale, (uint32_t)(key >> 32), &d);
            id = (uint32_t)key;
            lead = e == 0 || keys[e - 1] != key;
        }
        const unsigned peers = __match_any_sync(0xffffffffu, d);
        const int last = 31 - __clz(peers);
        for (uint32_t t = 0; t < g; ++t) {  // g is uniform: every lane reaches the shuffles
            unsigned long long p = 0;
            if (lead && L.cnt[d * L.samples + q0 + t]) p = (unsigned long long)fill[t * n + id] << 32 | (0xFFFFFFFFu - id);
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {  // lane i ends with the max over lanes [i, last]
                const unsigned long long q = __shfl_down_sync(0xffffffffu, p, o);
                if (lane + o <= last) p = max(p, q);
            }
            if (p && lane == __ffs(peers) - 1 && p > win[d * g + t]) atomicMax(&win[d * g + t], p);
        }
    }
}

// segment r of a sort group of rows [g0, g0 + rows): [r s, r s + fill[g0 + r]) of the group's slots
__global__ void screen_segments_kernel(const uint32_t *__restrict__ fill, uint64_t rows, uint32_t s, int *__restrict__ beg, int *__restrict__ end) {
    for (uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += (uint64_t)gridDim.x * blockDim.x) {
        beg[r] = (int)(r * s);
        end[r] = (int)(r * s + fill[r]);
    }
}

__global__ void screen_final_kernel(const uint32_t *__restrict__ fill, const unsigned long long *__restrict__ sorted, uint64_t n, uint32_t s,
                                    uint32_t *__restrict__ shared, double *__restrict__ containment, uint64_t *__restrict__ multiplicity) {
    for (uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t m = fill[r];
        if (shared) shared[r] = m;
        if (containment) containment[r] = (double)m / (double)s;
        if (multiplicity) multiplicity[r] = m ? sorted[r * s + (m - 1) / 2] : 0;  // the lower median
    }
}

ScreenLookup lookup_of(const ScreenIndex &ix, const uint32_t *ids = nullptr) {
    return ScreenLookup{ix.vals, ix.dir, ix.cnt, ids, ix.D * ix.samples, ix.nb, ix.vmax, ix.samples};
}

unsigned grid_of(uint64_t work) { return (unsigned)std::max<uint64_t>(1, std::min<uint64_t>((work + 255) / 256, (uint64_t)sm_count() * 16)); }

template <int K, bool SAMPLES, bool CANON>
int launch_screen_walk(const ScreenIndex &ix, const uint8_t *d_bases, const uint64_t *d_off, const uint32_t *d_ids, uint64_t n_reads,
                       cudaStream_t st) {
    uint64_t grid = 0;  // persistent: the pool's size is on the device, so the grid is what is resident at once
    { const int rc_ = resident_blocks((const void *)screen_walk_kernel<K, SAMPLES, CANON>, SCREEN_THREADS, 0, ~0ull, &grid); if (rc_ != PG_OK) return rc_; }
    screen_walk_kernel<K, SAMPLES, CANON><<<(unsigned)grid, SCREEN_THREADS, 0, st>>>(d_bases, d_off, n_reads, lookup_of(ix, d_ids), 4u);
    PG_LAUNCH_CHECK("screen_walk_kernel");
    return PG_OK;
}

// the add in one mode: screen_walk_kernel for k in WalkKs, screen_generic_kernel for any other k
template <bool CANON>
int screen_add_mode(const ScreenIndex &ix, int k, const uint8_t *d_bases, const uint64_t *d_off, const uint32_t *d_ids, uint64_t n_reads,
                    cudaStream_t st) {
    const bool samples = d_ids || ix.samples != 1;
    int rc = PG_OK;
    if (with_walk_k(k, [&](auto kk) {
            constexpr int K = decltype(kk)::value;
            rc = samples ? launch_screen_walk<K, true, CANON>(ix, d_bases, d_off, d_ids, n_reads, st)
                         : launch_screen_walk<K, false, CANON>(ix, d_bases, d_off, d_ids, n_reads, st);
        }))
        return rc;
    const void *fn = samples ? (const void *)screen_generic_kernel<true, CANON> : (const void *)screen_generic_kernel<false, CANON>;
    uint64_t grid = 0;
    if ((rc = resident_blocks(fn, SCREEN_THREADS, 0, ~0ull, &grid)) != PG_OK) return rc;
    if (samples) screen_generic_kernel<true, CANON><<<(unsigned)grid, SCREEN_THREADS, 0, st>>>(d_bases, d_off, n_reads, (uint32_t)k, lookup_of(ix, d_ids));
    else screen_generic_kernel<false, CANON><<<(unsigned)grid, SCREEN_THREADS, 0, st>>>(d_bases, d_off, n_reads, (uint32_t)k, lookup_of(ix, d_ids));
    PG_LAUNCH_CHECK("screen_generic_kernel");
    return PG_OK;
}

}  // namespace

void screen_free(ScreenIndex &ix, cudaStream_t st) {
    for (void *p : {(void *)ix.keys, (void *)ix.vals, (void *)ix.cnt, (void *)ix.dir})
        if (p) cudaFreeAsync(p, st);
    ix = ScreenIndex();
}

int screen_build(const uint32_t *d_sk, uint64_t n, int s, uint32_t samples, cudaStream_t st, ScreenIndex *out) {
    ScreenIndex ix;
    ix.n = n;
    ix.s = s;
    ix.samples = samples;
    const uint64_t total = n * (uint64_t)std::max(s, 0);
    if (total == 0) {
        *out = ix;
        return PG_OK;
    }
    int rc = [&]() -> int {
        StreamScratch tmp(st);
        uint64_t *d_keys = nullptr;
        uint32_t *d_v = nullptr, *d_u = nullptr;
        unsigned long long *d_scal = nullptr;  // [0]: vmax (low word), [1]: D
        auto nomem = [&](cudaError_t e) { set_error("cudaMallocAsync for the screen failed: %s", cudaGetErrorString(e)); cudaGetLastError(); return PG_ERR_NOMEM; };
        cudaError_t e;
        if ((e = tmp.alloc(&d_keys, total)) != cudaSuccess || (e = tmp.alloc(&d_scal, 2)) != cudaSuccess ||
            (e = cudaMallocAsync(&ix.keys, total * 8, st)) != cudaSuccess)
            return nomem(e);
        PG_CUDA(cudaMemsetAsync(d_scal, 0, 16, st));
        const int krc = launch_batch_keys(d_sk, total, (uint32_t)s, 0, d_keys, (uint32_t *)d_scal, st);
        if (krc != PG_OK) return krc;
        size_t bytes = 0;
        uint8_t *d_cub = nullptr;
        PG_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, bytes, d_keys, ix.keys, total, 0, 64, st));
        if ((e = tmp.alloc(&d_cub, bytes)) != cudaSuccess) return nomem(e);
        PG_CUDA(cub::DeviceRadixSort::SortKeys(d_cub, bytes, d_keys, ix.keys, total, 0, 64, st));
        if ((e = tmp.alloc(&d_v, total)) != cudaSuccess || (e = tmp.alloc(&d_u, total)) != cudaSuccess) return nomem(e);
        screen_values_kernel<<<grid_of(total), 256, 0, st>>>(ix.keys, total, d_v);
        PG_LAUNCH_CHECK("screen_values_kernel");
        bytes = 0;
        PG_CUDA(cub::DeviceSelect::Unique(nullptr, bytes, d_v, d_u, d_scal + 1, (int64_t)total, st));
        if ((e = tmp.alloc(&d_cub, bytes)) != cudaSuccess) return nomem(e);
        PG_CUDA(cub::DeviceSelect::Unique(d_cub, bytes, d_v, d_u, d_scal + 1, (int64_t)total, st));
        unsigned long long h_scal[2] = {0, 0};
        PG_CUDA(cudaMemcpyAsync(h_scal, d_scal, 16, cudaMemcpyDeviceToHost, st));
        PG_CUDA(cudaStreamSynchronize(st));
        ix.vmax = (uint32_t)h_scal[0];
        ix.D = h_scal[1];
        ix.nb = (uint32_t)((ix.D + 3) / 4);
        uint64_t cnt_bytes = 0;
        if (__builtin_mul_overflow(ix.D, (uint64_t)samples, &cnt_bytes) || __builtin_mul_overflow(cnt_bytes + 1, (uint64_t)8, &cnt_bytes)) {
            set_error("%llu values x %u samples of counters overflow 64 bits", (unsigned long long)ix.D, samples);
            return PG_ERR_NOMEM;
        }
        if ((e = cudaMallocAsync(&ix.vals, ix.D * 4, st)) != cudaSuccess || (e = cudaMallocAsync(&ix.cnt, cnt_bytes, st)) != cudaSuccess ||
            (e = cudaMallocAsync(&ix.dir, ((uint64_t)ix.nb + 1) * 8, st)) != cudaSuccess)
            return nomem(e);
        PG_CUDA(cudaMemcpyAsync(ix.vals, d_u, ix.D * 4, cudaMemcpyDeviceToDevice, st));
        PG_CUDA(cudaMemsetAsync(ix.cnt, 0, cnt_bytes, st));
        screen_dir_kernel<<<grid_of(ix.D), 256, 0, st>>>(ix.vals, ix.D, ix.nb, ix.vmax, ix.dir);
        PG_LAUNCH_CHECK("screen_dir_kernel");
        return PG_OK;
    }();
    if (rc == PG_OK) { cudaError_t e = cudaStreamSynchronize(st); if (e != cudaSuccess) rc = cuda_fail(e, "screen build", __FILE__, __LINE__); }
    if (rc != PG_OK) {
        screen_free(ix, st);
        cudaStreamSynchronize(st);
        return rc;
    }
    *out = ix;
    return PG_OK;
}

// One sample and no ids take the kernels without the sample step, the single-sample screen's; anything else the
// kernels with it.
int screen_add(const ScreenIndex &ix, int k, const uint8_t *d_bases, const uint64_t *d_off, const uint32_t *d_ids, uint64_t n_reads,
               cudaStream_t st) {
    if (n_reads == 0 || ix.D == 0) return PG_OK;
    return ix.canon ? screen_add_mode<true>(ix, k, d_bases, d_off, d_ids, n_reads, st) : screen_add_mode<false>(ix, k, d_bases, d_off, d_ids, n_reads, st);
}

int screen_reset(const ScreenIndex &ix, cudaStream_t st) {
    if (ix.D) PG_CUDA(cudaMemsetAsync(ix.cnt, 0, (ix.D * ix.samples + 1) * 8, st));
    return PG_OK;
}

namespace {

// The tail of results and winners for samples [first, first + count): per group of g samples (g n s slots at most
// SCREEN_GROUP_SLOTS, or one sample), the count pass over the words that count (all of them, or given a vote the won
// ones), the segmented sort of each (sample, reference) segment of pool counts and the final arrays, written straight
// into rows [q - first, q - first + g) of the outputs.  One sample is one group: the launches of a single-sample screen.
int screen_tally(const ScreenIndex &ix, bool winners, uint32_t first, uint32_t count, uint32_t *d_shared, double *d_cont, uint64_t *d_mult,
                 cudaStream_t st) {
    const uint64_t n = ix.n, s = (uint64_t)std::max(ix.s, 0), total = n * s;
    if (n == 0 || count == 0 || (!d_shared && !d_cont && !d_mult)) return PG_OK;
    StreamScratch tmp(st);
    uint32_t *d_fill = nullptr;
    unsigned long long *d_m = nullptr, *d_sorted = nullptr, *d_win = nullptr;
    int *d_beg = nullptr, *d_end = nullptr;
    const uint64_t group = std::max<uint64_t>(1, std::min<uint64_t>(count, SCREEN_GROUP_SLOTS / total));
    // the segmented sort counts in int: one sort per chunk of whole rows of at most INT_MAX slots
    const uint64_t chunk = std::min(std::max<uint64_t>(1, (uint64_t)INT_MAX / s), group * n);
    cudaError_t e;
    if ((e = tmp.alloc(&d_fill, group * n)) != cudaSuccess || (e = tmp.alloc(&d_m, group * total)) != cudaSuccess ||
        (e = tmp.alloc(&d_sorted, group * total)) != cudaSuccess || (e = tmp.alloc(&d_beg, chunk)) != cudaSuccess ||
        (e = tmp.alloc(&d_end, chunk)) != cudaSuccess || (winners && (e = tmp.alloc(&d_win, group * ix.D)) != cudaSuccess)) {
        set_error("cudaMallocAsync for the screen results failed: %s", cudaGetErrorString(e));
        cudaGetLastError();
        return PG_ERR_NOMEM;
    }
    size_t have = 0;
    uint8_t *d_cub = nullptr;
    const ScreenLookup L = lookup_of(ix);
    for (uint64_t q0 = first; q0 < (uint64_t)first + count; q0 += group) {
        const uint32_t g = (uint32_t)std::min<uint64_t>(group, (uint64_t)first + count - q0);
        const uint64_t rows = g * n, out = (q0 - first) * n;
        PG_CUDA(cudaMemsetAsync(d_fill, 0, rows * 4, st));
        if (winners) {  // the first pass's shared of every (sample, reference), then the vote
            PG_CUDA(cudaMemsetAsync(d_win, 0, g * ix.D * 8, st));
            screen_count_kernel<<<grid_of(total), 256, 0, st>>>(ix.keys, total, (uint32_t)s, L, (uint32_t)q0, g, n, nullptr, d_fill, nullptr);
            PG_LAUNCH_CHECK("screen_count_kernel");
            screen_vote_kernel<<<grid_of(total), 256, 0, st>>>(ix.keys, total, L, (uint32_t)q0, g, n, d_fill, d_win);
            PG_LAUNCH_CHECK("screen_vote_kernel");
            PG_CUDA(cudaMemsetAsync(d_fill, 0, rows * 4, st));
        }
        screen_count_kernel<<<grid_of(total), 256, 0, st>>>(ix.keys, total, (uint32_t)s, L, (uint32_t)q0, g, n, d_win, d_fill, d_m);
        PG_LAUNCH_CHECK("screen_count_kernel");
        for (uint64_t r0 = 0; r0 < rows; r0 += chunk) {
            const uint64_t rr = std::min(chunk, rows - r0);
            screen_segments_kernel<<<grid_of(rr), 256, 0, st>>>(d_fill + r0, rr, (uint32_t)s, d_beg, d_end);
            PG_LAUNCH_CHECK("screen_segments_kernel");
            size_t bytes = 0;
            PG_CUDA(cub::DeviceSegmentedSort::SortKeys(nullptr, bytes, d_m + r0 * s, d_sorted + r0 * s, (int)(rr * s), (int)rr, d_beg, d_end, st));
            if (bytes > have) {
                if ((e = tmp.alloc(&d_cub, bytes)) != cudaSuccess) {
                    set_error("cudaMallocAsync(%zu) for the screen results failed", bytes);
                    cudaGetLastError();
                    return PG_ERR_NOMEM;
                }
                have = bytes;
            }
            PG_CUDA(cub::DeviceSegmentedSort::SortKeys(d_cub, bytes, d_m + r0 * s, d_sorted + r0 * s, (int)(rr * s), (int)rr, d_beg, d_end, st));
        }
        screen_final_kernel<<<grid_of(rows), 256, 0, st>>>(d_fill, d_sorted, rows, (uint32_t)s, d_shared ? d_shared + out : nullptr,
                                                           d_cont ? d_cont + out : nullptr, d_mult ? d_mult + out : nullptr);
        PG_LAUNCH_CHECK("screen_final_kernel");
    }
    return PG_OK;
}

}  // namespace

int screen_results(const ScreenIndex &ix, uint32_t first, uint32_t count, uint32_t *d_shared, double *d_cont, uint64_t *d_mult,
                   cudaStream_t st) {
    return screen_tally(ix, false, first, count, d_shared, d_cont, d_mult, st);
}

int screen_winners(const ScreenIndex &ix, uint32_t first, uint32_t count, uint32_t *d_shared, double *d_cont, uint64_t *d_mult,
                   cudaStream_t st) {
    return screen_tally(ix, true, first, count, d_shared, d_cont, d_mult, st);
}

}  // namespace pg
