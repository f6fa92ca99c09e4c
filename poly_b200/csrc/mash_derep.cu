// mash_derep.cu -- greedy representatives of a sketch set at a matching-count threshold.
//
// Sketches r < i are linked iff same(r, i) >= min_same (the link rule of mash_cluster.cu: row r, column i of the
// dense pass).  In index order, i is a representative iff no representative r < i is linked to i.  Every other
// sketch is assigned the smallest linked representative (first) or the one with the largest count, ties to the
// smaller index (PG_DEREP_NEAREST).
//
// The dense row-block tiles of distance.cu are consumed on the device in sub-blocks of kDerepRows consecutive rows
// (never straddling a tile).  For sub-block [a, a + b):
//
// derep_links_kernel  : whole grid; the links among the sub-block's own rows as a b x kDerepRows bitmap
// derep_walk_kernel   : one CTA; the serial part.  It reads which rows earlier marks already cover, then walks the
//                       rows in order in shared memory: the next uncovered row is a representative and its link
//                       bits cover the rows after it.  At most kDerepRows steps whatever the input; it writes the
//                       sub-block's representatives as a list.
// derep_mark_kernel   : whole grid; the representatives' tile rows at columns (r, n), and nothing else.  A linked
//                       column j gets atomicMin(rep[j], r) (first) or atomicMax(key[j], same << 32 | ~r) (nearest),
//                       both order-independent.  Columns inside the sub-block get their assignment here too.
// derep_finish_kernel : after the last tile: rep[i] = i for representatives, keys to indices, the count.
//
// A growing dereplication (launch_mash_derep_add) runs the same kernels over one batch whose rows are numbered from
// an id base: rows linked to a kept representative of the earlier batches are seeded first (launch_index_link
// writes rep / key there), the walk reads them as covered, and the marks and the finish write global ids
// base + r.  All comparisons stay in batch rows.  derep_gather_kernel then lists the batch's new
// representatives, in order, for the representative index.
//
// A representative's slot is never written (the marks only reach sketches linked to an earlier representative),
// so "slot still unset" is exactly "representative" and no separate flag array is kept.  Stream order makes every
// earlier mark visible to the next walk; the output depends on the input alone.
#include <algorithm>

#include <cub/device/device_select.cuh>
#include <thrust/iterator/counting_iterator.h>

#include "common.cuh"

namespace pg {

namespace {

constexpr uint32_t kDerepRows = 1024;            // rows per sub-block: one bit per row in a warp's 32 x 32-bit words
constexpr uint32_t kWords = kDerepRows / 32;
constexpr uint32_t kNone = 0xffffffffu;          // first mode: rep[j] not yet assigned
constexpr uint32_t kMarkCols = 4096;             // columns of one mark step: 256 threads x 4 quads

// bits[t * kWords + w], bit x: sub-block row t is linked to sub-block row 32 w + x (only x above t, below b).
// One warp per word: a coalesced 128-byte load and one ballot.
__global__ void __launch_bounds__(256)
derep_links_kernel(const uint32_t *__restrict__ tile, uint64_t n, uint64_t t0, uint64_t a, uint32_t b, uint32_t min_same,
                   uint32_t *__restrict__ bits) {
    const uint32_t lane = threadIdx.x & 31u;
    for (uint32_t it = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; it < b * kWords; it += (gridDim.x * blockDim.x) >> 5) {
        const uint32_t t = it / kWords, c = (it % kWords) * 32 + lane;
        const uint32_t v = c > t && c < b ? tile[(t0 + t) * n + a + c] : 0;  // min_same >= 1: 0 never links
        const uint32_t m = __ballot_sync(0xffffffffu, v >= min_same);
        if (lane == 0) bits[it] = m;
    }
}

// list[0] = number of representatives in [a, a + b), list[1..] = their indices in increasing order.
template <bool Nearest>
__global__ void __launch_bounds__(1024)
derep_walk_kernel(const uint32_t *__restrict__ bits, uint64_t a, uint32_t b, const uint32_t *__restrict__ rep,
                  const unsigned long long *__restrict__ key, uint32_t *__restrict__ list) {
    extern __shared__ uint4 s_bits4[];
    const uint32_t *s_bits = reinterpret_cast<const uint32_t *>(s_bits4);
#pragma unroll 8
    for (uint32_t i = threadIdx.x; i < b * kWords / 4; i += blockDim.x) s_bits4[i] = reinterpret_cast<const uint4 *>(bits)[i];
    __syncthreads();
    if (threadIdx.x >= 32) return;
    const uint32_t lane = threadIdx.x;
    // lane w holds rows 32 w .. 32 w + 31 of the sub-block: covered by an earlier mark (rows past b count as covered)
    bool set[kWords];
#pragma unroll
    for (uint32_t w = 0; w < kWords; ++w) {  // all 32 loads in flight: every lane reads a row of the sub-block
        const uint64_t row = a + min(w * 32 + lane, b - 1);
        set[w] = Nearest ? key[row] != 0 : rep[row] != kNone;
    }
    uint32_t cov = 0;
#pragma unroll
    for (uint32_t w = 0; w < kWords; ++w) {
        const uint32_t m = __ballot_sync(0xffffffffu, set[w] || w * 32 + lane >= b);
        if (lane == w) cov = m;
    }
    // every step takes the first uncovered row: a ballot skips any run of covered rows at once
    uint32_t reps = 0;
    for (;;) {
        const uint32_t open = __ballot_sync(0xffffffffu, cov != 0xffffffffu);
        if (!open) break;
        const uint32_t w = __ffs(open) - 1;
        const uint32_t x = __ffs(~__shfl_sync(0xffffffffu, cov, w)) - 1;
        cov |= s_bits[(w * 32 + x) * kWords + lane];
        if (lane == w) {
            cov |= 1u << x;
            reps |= 1u << x;
        }
    }
    const uint32_t cnt = __popc(reps);
    uint32_t end = cnt;  // inclusive prefix sum over the lanes
    for (uint32_t d = 1; d < 32; d <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, end, d);
        if (lane >= d) end += y;
    }
    uint32_t at = end - cnt;
    for (uint32_t m = reps; m; m &= m - 1) list[1 + at++] = (uint32_t)a + lane * 32 + __ffs(m) - 1;
    if (lane == 31) list[0] = end;
}

// The listed representatives' tile rows (tile row 0 is sketch row0), columns j > r.  One CTA step covers
// kMarkCols columns of one representative with 16-byte loads, four per thread in flight.  Marks carry the
// representative's id base + r.
template <bool Nearest>
__global__ void __launch_bounds__(256)
derep_mark_kernel(const uint32_t *__restrict__ tile, uint64_t n, uint64_t row0, uint32_t min_same, const uint32_t *__restrict__ list,
                  uint32_t base, uint32_t *rep, unsigned long long *key) {
    const uint64_t chunks = (n + kMarkCols - 1) / kMarkCols;
    const uint64_t items = (uint64_t)list[0] * chunks;
    const bool vec = (n & 3) == 0;  // rows are 16-byte aligned
    for (uint64_t it = blockIdx.x; it < items; it += gridDim.x) {
        const uint32_t r = list[1 + it / chunks];
        const uint64_t c0 = (it % chunks) * kMarkCols;
        if (c0 + kMarkCols <= (uint64_t)r + 1) continue;  // all at or left of the diagonal
        const uint32_t *row = tile + (r - row0) * n;
        uint32_t v[4][4];
#pragma unroll
        for (int q = 0; q < 4; ++q) load_count_quad(row, c0 + (q * 256 + threadIdx.x) * 4, n, vec, v[q]);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            if (max(max(v[q][0], v[q][1]), max(v[q][2], v[q][3])) < min_same) continue;
            const uint64_t j0 = c0 + (q * 256 + threadIdx.x) * 4;
#pragma unroll
            for (int t = 0; t < 4; ++t) {
                const uint64_t j = j0 + t;
                if (v[q][t] < min_same || j <= r) continue;
                if (Nearest) atomicMax(key + j, (unsigned long long)v[q][t] << 32 | (uint32_t)~(base + r));
                else atomicMin(rep + j, base + r);
            }
        }
    }
}

template <bool Nearest>
__global__ void __launch_bounds__(256)
derep_finish_kernel(uint32_t *__restrict__ rep, const unsigned long long *__restrict__ key, uint64_t n, uint32_t base,
                    unsigned long long *__restrict__ n_reps) {
    const uint32_t lane = threadIdx.x & 31u;
    uint32_t reps = 0;
    for (uint64_t i0 = (uint64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); i0 < n; i0 += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t i = i0 + lane;
        if (i >= n) continue;
        const bool self = Nearest ? key[i] == 0 : rep[i] == kNone;
        if (self) rep[i] = base + (uint32_t)i;
        else if (Nearest) rep[i] = ~(uint32_t)key[i];
        reps += self;
    }
    reps = __reduce_add_sync(0xffffffffu, reps);
    if (n_reps && lane == 0 && reps) atomicAdd(n_reps, (unsigned long long)reps);
}

template <bool Nearest>
int derep_tiles(const uint32_t *d_sk, uint64_t n, int s, uint32_t min_same, uint32_t base, uint32_t *d_rep, unsigned long long *d_key,
                unsigned long long *d_n_reps, StreamScratch &tmp, cudaStream_t st) {
    uint32_t *d_bits = nullptr, *d_list = nullptr;
    if (tmp.alloc(&d_bits, kDerepRows * kWords + 1 + kDerepRows) != cudaSuccess) {
        cudaGetLastError();
        set_error("cudaMallocAsync for the dereplication sub-block failed");
        return PG_ERR_NOMEM;
    }
    d_list = d_bits + kDerepRows * kWords;
    int rc = func_smem((const void *)derep_walk_kernel<Nearest>, kDerepRows * kWords * 4);
    if (rc != PG_OK) return rc;

    const unsigned grid = (unsigned)sm_count() * 8;
    rc = distance_plan_tiles(d_sk, n, s, 0, n, distance_tile_rows(n, n), true, false, st,
                             [&](const uint32_t *tile, const double *, uint64_t rb, uint64_t re) {
        for (uint64_t a = rb; a < re; a += kDerepRows) {
            const uint32_t b = (uint32_t)std::min<uint64_t>(kDerepRows, re - a);
            derep_links_kernel<<<(b * kWords + 7) / 8, 256, 0, st>>>(tile, n, a - rb, a, b, min_same, d_bits);
            PG_LAUNCH_CHECK("derep_links_kernel");
            derep_walk_kernel<Nearest><<<1, 1024, b * kWords * 4, st>>>(d_bits, a, b, d_rep, d_key, d_list);
            PG_LAUNCH_CHECK("derep_walk_kernel");
            derep_mark_kernel<Nearest><<<grid, 256, 0, st>>>(tile, n, rb, min_same, d_list, base, d_rep, d_key);
            PG_LAUNCH_CHECK("derep_mark_kernel");
        }
        return PG_OK;
    });
    if (rc != PG_OK) return rc;
    derep_finish_kernel<Nearest><<<(unsigned)std::min<uint64_t>((n + 255) / 256, (uint64_t)sm_count() * 16), 256, 0, st>>>(d_rep, d_key, n, base, d_n_reps);
    PG_LAUNCH_CHECK("derep_finish_kernel");
    return PG_OK;
}

}  // namespace

int mash_derep_check(uint64_t n, int s, uint32_t min_same, uint32_t flags) {
    if (flags & ~PG_DEREP_NEAREST) { set_error("unknown dereplication flags 0x%x", flags); return PG_ERR_ARG; }
    return mash_cluster_check(n, s, min_same);
}

int launch_mash_derep(const uint32_t *d_sk, uint64_t n, int s, uint32_t min_same, uint32_t flags, uint32_t *d_rep,
                      unsigned long long *d_n_reps, cudaStream_t st) {
    if (d_n_reps) PG_CUDA(cudaMemsetAsync(d_n_reps, 0, 8, st));
    int rc = mash_derep_check(n, s, min_same, flags);
    if (rc != PG_OK || n == 0) return rc;
    StreamScratch tmp(st);  // keys (nearest), the sub-block's link bits and list: freed on every way out
    if (!(flags & PG_DEREP_NEAREST)) {
        PG_CUDA(cudaMemsetAsync(d_rep, 0xff, n * 4, st));  // kNone: the assignment is built in place
        return derep_tiles<false>(d_sk, n, s, min_same, 0, d_rep, nullptr, d_n_reps, tmp, st);
    }
    unsigned long long *d_key = nullptr;
    if (tmp.alloc(&d_key, n) != cudaSuccess) {
        cudaGetLastError();
        set_error("cudaMallocAsync(%llu) for the dereplication keys failed", (unsigned long long)(n * 8));
        return PG_ERR_NOMEM;
    }
    PG_CUDA(cudaMemsetAsync(d_key, 0, n * 8, st));
    return derep_tiles<true>(d_sk, n, s, min_same, 0, d_rep, d_key, d_n_reps, tmp, st);
}

int launch_mash_derep_add(const DistancePlan &plan, const uint32_t *d_ids, const uint32_t *d_b, uint64_t m, int s, uint32_t min_same,
                          uint32_t flags, uint32_t base, uint32_t *d_rep, unsigned long long *d_n_new, cudaStream_t st) {
    PG_CUDA(cudaMemsetAsync(d_n_new, 0, 8, st));
    StreamScratch tmp(st);
    const bool nearest = flags & PG_DEREP_NEAREST;
    unsigned long long *d_key = nullptr;
    if (!nearest) {
        PG_CUDA(cudaMemsetAsync(d_rep, 0xff, m * 4, st));  // kNone, then the seeds
    } else {
        if (tmp.alloc(&d_key, m) != cudaSuccess) {
            cudaGetLastError();
            set_error("cudaMallocAsync(%llu) for the dereplication keys failed", (unsigned long long)(m * 8));
            return PG_ERR_NOMEM;
        }
        PG_CUDA(cudaMemsetAsync(d_key, 0, m * 8, st));
    }
    int rc = launch_index_link(plan, d_b, m, s, min_same, d_ids, nearest, d_rep, d_key, st);
    if (rc != PG_OK) return rc;
    return nearest ? derep_tiles<true>(d_b, m, s, min_same, base, d_rep, d_key, d_n_new, tmp, st)
                   : derep_tiles<false>(d_b, m, s, min_same, base, d_rep, nullptr, d_n_new, tmp, st);
}

namespace {

// Batch row i is a new representative iff its slot holds its own id
struct IsNewRep {
    const uint32_t *rep;
    uint32_t base;
    __device__ bool operator()(uint32_t i) const { return rep[i] == base + i; }
};

// Row p of the list: sel[p]'s sketch to rows[p], its id to ids[p].  One warp per row.
__global__ void __launch_bounds__(256)
derep_gather_kernel(const uint32_t *__restrict__ b, uint32_t s, const uint32_t *__restrict__ sel, uint64_t n_sel, uint32_t base,
                    uint32_t *__restrict__ rows, uint32_t *__restrict__ ids) {
    const uint32_t lane = threadIdx.x & 31u;
    for (uint64_t p = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; p < n_sel; p += ((uint64_t)gridDim.x * blockDim.x) >> 5) {
        const uint32_t i = sel[p];
        const uint32_t *src = b + (uint64_t)i * s;
        uint32_t *dst = rows + p * s;
        for (uint32_t w = lane; w < s; w += 32) dst[w] = src[w];
        if (lane == 0) ids[p] = base + i;
    }
}

}  // namespace

int launch_derep_gather(const uint32_t *d_b, uint64_t m, int s, uint32_t base, const uint32_t *d_rep, uint64_t n_new, uint32_t *d_rows,
                        uint32_t *d_ids, cudaStream_t st) {
    if (n_new == 0) return PG_OK;
    StreamScratch tmp(st);
    uint32_t *d_sel = nullptr;
    unsigned long long *d_n_sel = nullptr;
    if (tmp.alloc(&d_sel, n_new) != cudaSuccess || tmp.alloc(&d_n_sel, 1) != cudaSuccess) {
        cudaGetLastError();
        set_error("cudaMallocAsync for the new representatives failed");
        return PG_ERR_NOMEM;
    }
    // an order-preserving compaction of the batch rows: no atomic decides a position
    const thrust::counting_iterator<uint32_t> rows(0);
    const IsNewRep pred{d_rep, base};
    size_t bytes = 0;
    PG_CUDA(cub::DeviceSelect::If(nullptr, bytes, rows, d_sel, d_n_sel, (int64_t)m, pred, st));
    uint8_t *d_tmp = nullptr;
    if (tmp.alloc(&d_tmp, bytes) != cudaSuccess) {
        cudaGetLastError();
        set_error("cudaMallocAsync(%zu) for the selection failed", bytes);
        return PG_ERR_NOMEM;
    }
    PG_CUDA(cub::DeviceSelect::If(d_tmp, bytes, rows, d_sel, d_n_sel, (int64_t)m, pred, st));
    const unsigned grid = (unsigned)std::min<uint64_t>((n_new + 7) / 8, (uint64_t)sm_count() * 16);
    derep_gather_kernel<<<grid, 256, 0, st>>>(d_b, (uint32_t)s, d_sel, n_new, base, d_rows, d_ids);
    PG_LAUNCH_CHECK("derep_gather_kernel");
    return PG_OK;
}

}  // namespace pg
