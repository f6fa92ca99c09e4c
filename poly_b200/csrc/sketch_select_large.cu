// sketch_select_large.cu -- K2x: mash.Sketch in the select regime (L-k >= s) beyond the shared-memory
// kernels of sketch_select.cu: sketch sizes above 16384 words or k above 1024 bytes.
//
// /root/reference/search/mash/mash.go:68-104 has no such limits (a `mash sketch -s 100000` of a genome
// is an ordinary call), so they must not surface as errors.  Nothing here is tuned like K2t -- the
// row's hashes simply go through global memory:
//   1. large_hash_kernel: every k-mer hash of every select-regime row of the group -> tmp (one thread
//      per k-mer, byte-wise murmur3: any k)
//   2. large_select_kernel, one CTA per row: exact radix select of the s-th smallest value (4 passes
//      over the row's hashes with a 256-bin histogram), warp-aggregated compaction of the s smallest
//      (ties counted) into a power-of-two sort buffer, bitonic sort of that buffer (strides below the
//      tile size in shared memory, the rest in L2-resident global memory), copy to every destination.
// Rows are processed in groups whose temporaries stay below ~2 GiB.
#include <algorithm>
#include <vector>

#include "common.cuh"
#include "murmur3.cuh"

namespace pg {

namespace {

constexpr int LG_HASH_THREADS = 256;
constexpr uint32_t LG_CHUNK = 8192;   // k-mer positions per hashing work item
constexpr int LG_THREADS = 1024;
constexpr uint32_t LG_TILE = 8192;    // words of the sort buffer one shared-memory tile holds

__global__ void __launch_bounds__(LG_HASH_THREADS)
large_hash_kernel(const uint8_t *__restrict__ bases, const uint64_t *__restrict__ offsets, uint32_t uniform_len, uint64_t row0,
                  uint64_t n_items, uint32_t chunks_per_row, uint32_t k, uint32_t s, uint64_t base_off, uint32_t *__restrict__ tmp) {
    for (uint64_t item = blockIdx.x; item < n_items; item += gridDim.x) {
        const uint64_t row = row0 + item / chunks_per_row;
        const uint64_t i0 = (item % chunks_per_row) * (uint64_t)LG_CHUNK;
        const RowSpan sp = row_span(offsets, uniform_len, row, k);
        const uint64_t n = sp.n;
        if (!select_regime(n, s) || i0 >= n) continue;  // fill regime rows belong to the other kernel
        const uint8_t *seq = bases + sp.beg;
        uint32_t *dst = tmp + (sp.beg - base_off);
        const uint64_t i1 = min(n, i0 + (uint64_t)LG_CHUNK);
        for (uint64_t i = i0 + threadIdx.x; i < i1; i += LG_HASH_THREADS) {
            const uint8_t *p = seq + i;
            dst[i] = mm3_bytes([&](uint32_t j) { return __ldg(p + j); }, k);
        }
    }
}

// compare-exchange network of one bitonic merge step set {j = j_hi, j_hi / 2, ..., 1} of phase kk on a tile that
// lives in shared memory; `g0` is the global index of the tile's first word (the direction depends on it)
__device__ __forceinline__ void bitonic_tile(uint32_t *tile, uint32_t words, uint64_t g0, uint64_t kk, uint32_t j_hi) {
    for (uint32_t j = j_hi; j > 0; j >>= 1) {
        for (uint32_t t = threadIdx.x; t < words / 2; t += LG_THREADS) {
            const uint32_t i = 2 * t - (t & (j - 1));
            const uint32_t l = i + j;
            const bool up = ((g0 + i) & kk) == 0;
            const uint32_t a = tile[i], b = tile[l];
            if ((a > b) == up) { tile[i] = b; tile[l] = a; }
        }
        __syncthreads();
    }
}

// Two CTAs per SM, as the launcher's grid assumes (left to itself ptxas takes 56 registers: one CTA per SM).
__global__ void __launch_bounds__(LG_THREADS, 2)
large_select_kernel(const uint64_t *__restrict__ offsets, uint32_t uniform_len, uint64_t row0, uint64_t n_rows, uint32_t k, uint32_t s,
                    uint64_t P, uint64_t base_off, const uint32_t *__restrict__ tmp, uint32_t *__restrict__ sortbuf,
                    uint32_t *__restrict__ out, uint64_t row_stride, uint32_t *__restrict__ count, int32_t *__restrict__ status,
                    const SketchDst extra) {
    __shared__ uint32_t s_hist[256];
    __shared__ uint32_t s_sel[4];  // 0 prefix, 1 mask, 2 want, 3 unused
    __shared__ unsigned long long s_cnt[2];  // 0 values below v*, 1 copies of v* seen
    __shared__ uint32_t s_tile[LG_TILE];
    const uint32_t tid = threadIdx.x, lane = tid & 31u;
    for (uint64_t lrow = blockIdx.x; lrow < n_rows; lrow += gridDim.x) {
        const uint64_t row = row0 + lrow;
        const RowSpan sp = row_span(offsets, uniform_len, row, k);
        const uint64_t n = sp.n;
        if (!select_regime(n, s)) continue;
        if (empty_sketch_panics(s, status, count, row)) continue;
        const uint32_t *src = tmp + (sp.beg - base_off);
        uint32_t *sb = sortbuf + lrow * P;
        uint32_t *dst = out + row * row_stride;
        // ---- exact radix select: v* = the s-th smallest hash, need_eq = copies of v* among the s smallest ----
        if (tid == 0) { s_sel[0] = 0; s_sel[1] = 0; s_sel[2] = s; }
        for (int shift = 24; shift >= 0; shift -= 8) {
            for (uint32_t i = tid; i < 256; i += LG_THREADS) s_hist[i] = 0;
            __syncthreads();
            const uint32_t prefix = s_sel[0], mask = s_sel[1];
            for (uint64_t i = tid; i < n; i += LG_THREADS) {
                const uint32_t v = src[i];
                if ((v & mask) == prefix) atomicAdd(&s_hist[(v >> shift) & 255u], 1u);
            }
            __syncthreads();
            if (tid == 0) {
                uint32_t want = s_sel[2], b = 0;
                while (b < 255 && s_hist[b] < want) { want -= s_hist[b]; ++b; }
                s_sel[0] = prefix | (b << shift);
                s_sel[1] = mask | (255u << shift);
                s_sel[2] = want;
            }
            __syncthreads();
        }
        const uint32_t vstar = s_sel[0], need_eq = s_sel[2], n_lt = s - need_eq;
        // ---- compaction: values below v* to the front, need_eq copies of v* behind them, padding up to P ----
        if (tid == 0) { s_cnt[0] = 0; s_cnt[1] = 0; }
        __syncthreads();
        for (uint64_t i0 = 0; i0 < n; i0 += LG_THREADS) {
            const uint64_t i = i0 + tid;
            const uint32_t v = i < n ? src[i] : 0xffffffffu;
            const bool lt = i < n && v < vstar, eq = i < n && v == vstar;
            const uint32_t b_lt = __ballot_sync(0xffffffffu, lt), b_eq = __ballot_sync(0xffffffffu, eq);
            unsigned long long o_lt = 0, o_eq = 0;
            if (lane == 0) {
                if (b_lt) o_lt = atomicAdd(&s_cnt[0], (unsigned long long)__popc(b_lt));
                if (b_eq) o_eq = atomicAdd(&s_cnt[1], (unsigned long long)__popc(b_eq));
            }
            o_lt = __shfl_sync(0xffffffffu, o_lt, 0);
            o_eq = __shfl_sync(0xffffffffu, o_eq, 0);
            const uint32_t below = (1u << lane) - 1u;
            if (lt) sb[o_lt + __popc(b_lt & below)] = v;
            if (eq) {
                const unsigned long long e = o_eq + __popc(b_eq & below);
                if (e < need_eq) sb[n_lt + e] = v;
            }
        }
        for (uint64_t i = (uint64_t)s + tid; i < P; i += LG_THREADS) sb[i] = 0xffffffffu;
        __syncthreads();
        // ---- bitonic sort of sb[0, P) ----
        if (P <= LG_TILE) {
            for (uint32_t i = tid; i < P; i += LG_THREADS) s_tile[i] = sb[i];
            __syncthreads();
            for (uint64_t kk = 2; kk <= P; kk <<= 1) bitonic_tile(s_tile, (uint32_t)P, 0, kk, (uint32_t)(kk >> 1));
            for (uint32_t i = tid; i < P; i += LG_THREADS) sb[i] = s_tile[i];
            __syncthreads();
        } else {
            // phases kk <= LG_TILE: whole phases inside a tile
            for (uint64_t g0 = 0; g0 < P; g0 += LG_TILE) {
                for (uint32_t i = tid; i < LG_TILE; i += LG_THREADS) s_tile[i] = sb[g0 + i];
                __syncthreads();
                for (uint64_t kk = 2; kk <= LG_TILE; kk <<= 1) bitonic_tile(s_tile, LG_TILE, g0, kk, (uint32_t)(kk >> 1));
                for (uint32_t i = tid; i < LG_TILE; i += LG_THREADS) sb[g0 + i] = s_tile[i];
                __syncthreads();
            }
            for (uint64_t kk = 2ull * LG_TILE; kk <= P; kk <<= 1) {
                // strides >= tile size through global memory (L2), then the rest of the phase tile by tile in shared memory
                for (uint64_t j = kk >> 1; j >= LG_TILE; j >>= 1) {
                    for (uint64_t t = tid; t < P / 2; t += LG_THREADS) {
                        const uint64_t i = 2 * t - (t & (j - 1));
                        const uint64_t l = i + j;
                        const bool up = (i & kk) == 0;
                        const uint32_t a = sb[i], b = sb[l];
                        if ((a > b) == up) { sb[i] = b; sb[l] = a; }
                    }
                    __syncthreads();
                }
                for (uint64_t g0 = 0; g0 < P; g0 += LG_TILE) {
                    for (uint32_t i = tid; i < LG_TILE; i += LG_THREADS) s_tile[i] = sb[g0 + i];
                    __syncthreads();
                    bitonic_tile(s_tile, LG_TILE, g0, kk, LG_TILE / 2);
                    for (uint32_t i = tid; i < LG_TILE; i += LG_THREADS) sb[g0 + i] = s_tile[i];
                    __syncthreads();
                }
            }
        }
        // ---- output: ascending bottom-s to every destination ----
        for (uint32_t i = tid; i < s; i += LG_THREADS) dst[i] = sb[i];
        replicate_row<LG_THREADS>(extra, row, row_stride, sb, dst, s);
        // s == 1: mash.go:96-98 indexes Sketches[-1] as soon as a later hash is strictly below Sketches[0]
        put_row_status(status, count, row, s, s == 1 && sb[0] < src[0]);
        __syncthreads();
    }
}

}  // namespace

int launch_sketch_select_large(const uint8_t *d_bases, const uint64_t *d_offsets, uint32_t read_len, uint64_t n_reads, int k, int s,
                               uint32_t *d_out, uint64_t row_stride, uint32_t *d_count, int32_t *d_status, cudaStream_t st,
                               const SketchDst &ex) {
    // row starts on the host: groups are cut where the temporaries reach the budget
    std::vector<uint64_t> off;
    if (d_offsets) {
        const int rc = host_row_starts(d_offsets, n_reads, st, off);
        if (rc != PG_OK) return rc;
    }
    auto row_beg = [&](uint64_t r) -> uint64_t { return d_offsets ? off[r] : r * (uint64_t)read_len; };
    uint64_t P = 2;
    while (P < (uint64_t)std::max(s, 1)) P <<= 1;
    const uint64_t budget_words = 1ull << 29;  // 2 GiB of temporaries per group (one row is always taken)
    uint64_t r0 = 0;
    while (r0 < n_reads) {
        uint64_t r1 = r0 + 1, max_len = row_beg(r0 + 1) - row_beg(r0);
        while (r1 < n_reads && (row_beg(r1 + 1) - row_beg(r0)) + (r1 + 1 - r0) * P <= budget_words) {
            max_len = std::max(max_len, row_beg(r1 + 1) - row_beg(r1));
            ++r1;
        }
        const uint64_t rows = r1 - r0, base_off = row_beg(r0), words = row_beg(r1) - base_off;
        if (max_len > (uint64_t)k && max_len - (uint64_t)k >= (uint64_t)std::max(s, 0)) {  // the group holds a select-regime row
            StreamScratch tmp(st);
            uint32_t *d_tmp = nullptr, *d_sort = nullptr;
            PG_CUDA(tmp.alloc(&d_tmp, words));
            PG_CUDA(tmp.alloc(&d_sort, rows * P));
            const uint64_t cpr = (max_len - (uint64_t)k + LG_CHUNK - 1) / LG_CHUNK;
            if (cpr > 0xffffffffull) {
                set_error("sequence of %llu bases is too long for the large-sketch path", (unsigned long long)max_len);
                return PG_ERR_UNSUPPORTED;
            }
            const uint64_t n_items = rows * cpr;
            const unsigned hash_blocks = (unsigned)std::min<uint64_t>(n_items, (uint64_t)sm_count() * 32);
            large_hash_kernel<<<hash_blocks, LG_HASH_THREADS, 0, st>>>(d_bases, d_offsets, read_len, r0, n_items, (uint32_t)cpr, (uint32_t)k,
                                                                      (uint32_t)s, base_off, d_tmp);
            PG_LAUNCH_CHECK("large_hash_kernel");
            const unsigned sel_blocks = (unsigned)std::min<uint64_t>(rows, (uint64_t)sm_count() * 2);
            large_select_kernel<<<sel_blocks, LG_THREADS, 0, st>>>(d_offsets, read_len, r0, rows, (uint32_t)k, (uint32_t)s, P, base_off, d_tmp,
                                                                  d_sort, d_out, row_stride, d_count, d_status, ex);
            PG_LAUNCH_CHECK("large_select_kernel");
        }
        r0 = r1;
    }
    return PG_OK;
}

}  // namespace pg
