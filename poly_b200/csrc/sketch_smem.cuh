// sketch_smem.cuh -- the dynamic shared memory of the sketch kernels (sketch_fill.cu, sketch_select.cu): one
// __host__ __device__ description per kernel, built from its launch parameters.  The launcher sizes the launch with
// it and the kernel carves with it, so the two cannot drift apart.  Offsets are in 32-bit words from the start of
// the dynamic shared memory unless they say bytes.  tests/test_sketch_smem.py checks the totals, the alignment of
// the TMA stage buffers and that no regions overlap.
#pragma once
#include <stddef.h>
#include <stdint.h>

namespace pg {
// ---- K1 (sketch_fill_uniform_kernel): 2 input stages | out tile [32][nk] ------------------------------------
// an input stage: 32 reads of L bytes + 16 B over-read pad, 16-byte rounded (+ 1 KB static table when k % 4 == 1)
__host__ __device__ inline uint32_t k1_in_bytes(uint32_t L) { return (32u * L + 16u + 15u) & ~15u; }
__host__ __device__ inline size_t k1_smem_bytes(uint32_t L, uint32_t nk) { return 2 * (size_t)k1_in_bytes(L) + (size_t)32 * nk * 4; }
// ---- K1r (sketch_fill_ragged_kernel): input stage [in_cap bytes] | out tile [32][stride] -------------------
// in_cap: 32 reads of at most max_len bytes, the < 16 B head before the first 16-byte boundary and 32 B over-read
// pad, 16-byte rounded (so also the out tile, the source of a bulk store, starts on a 16-byte boundary)
__host__ __device__ inline uint64_t k1r_in_bytes(uint64_t max_len) { return (32 * max_len + 48 + 15) & ~15ull; }
__host__ __device__ inline size_t k1r_smem_bytes(uint32_t in_cap, uint32_t stride) { return (size_t)in_cap + (size_t)32 * stride * 4; }
// ---- select-regime geometry --------------------------------------------------------------------------------
constexpr int SEL_CHUNK = 2048;     // k-mer positions per chunk of sketch_select_kernel
constexpr int SEL_LOOKAHEAD = 1024; // max k supported by the staged path (bytes beyond chunk)
constexpr int SEL_NBK = 2048;       // value buckets of the final sort-select (v >> 21)
constexpr uint32_t STAGE_PAD = 32;  // zero bytes behind a staged chunk: the walks read up to a word step beyond it
constexpr int SEL_STAGE_WORDS = (15 + SEL_CHUNK + SEL_LOOKAHEAD + STAGE_PAD + 15) / 16 * 4;  // head + chunk + k + pad, 16-B multiple
constexpr int SELW_THREADS = 256;
constexpr int SELW_SEG = 20;  // bytes between the segments of adjacent lanes = 5 words: conflict-free smem reads
constexpr int SELW_CHUNK = SELW_THREADS * SELW_SEG;                          // 5120 k-mer positions
constexpr int SELW_STAGE_WORDS = (15 + SELW_CHUNK + 32 + 48 + 15) / 16 * 4;  // head + chunk + k + over-read pad
// misc words: 0 cnt, 1 prefix, 2 want, 3 kept_lt, 4 kept_eq, 5 hmin_later, 6 bt, 7 need; K2w adds 3 per-chunk
// counters from SELW_CHUNK_CTR on
constexpr uint32_t SEL_MISC_WORDS = 8, SELW_MISC_WORDS = 16, SELW_CHUNK_CTR = 8;
static_assert(SELW_CHUNK_CTR >= SEL_MISC_WORDS && SELW_CHUNK_CTR + 3 <= SELW_MISC_WORDS, "misc holds K2w's chunk counters");
static_assert(SEL_STAGE_WORDS % 4 == 0 && SELW_STAGE_WORDS % 4 == 0 && (SEL_CHUNK + SEL_LOOKAHEAD) % 4 == 0, "16-byte granules");
// The shared memory of one select CTA as its device code sees it.
struct SelSmem {
    uint32_t *cand;   // [cap]
    uint32_t *keep;   // [s]
    uint32_t *kv;     // [SEL_CHUNK + SEL_LOOKAHEAD] (sketch_select_kernel only)
    uint32_t *bytes;  // 2 x stage words of staged read bytes (word view), double-buffered
    uint32_t *hist;   // [SEL_NBK + 1] (radix select uses the first 256 words)
    uint32_t *misc;   // see SEL_MISC_WORDS
    uint32_t tmpcap;  // words available at keep[] for the final scatter (keep+kv+bytes are contiguous)
};
// ---- the SelSmem kernels (sketch_select_kernel, K2w sketch_select_walk_kernel, select_merge_kernel) --------
//   cand [cap] | keep [keep_w] | kv [kv_w] | stage 2 x [stage_w] | hist [SEL_NBK + 1] | misc [misc_w]
// keep is keep_w + keep_pad words, keep_pad a constant of the kernel.  The stage buffers start on 16-byte
// boundaries when cap is a multiple of 4 (the launchers check).  carve() adds the regions up pointer by pointer,
// which is the address arithmetic the kernels were tuned with.
struct SelLayout {
    uint32_t cap, keep_w, keep_pad, kv_w, stage_w, misc_w;  // region sizes in words
    __host__ __device__ size_t kv() const { return (size_t)cap + keep_w + keep_pad; }
    __host__ __device__ size_t stage() const { return kv() + kv_w; }
    __host__ __device__ size_t hist() const { return stage() + 2 * (size_t)stage_w; }
    __host__ __device__ size_t bytes() const { return (hist() + SEL_NBK + 1 + misc_w) * 4; }  // misc: the last misc_w words
    __host__ __device__ SelSmem carve(uint32_t *smem_w) const {
        SelSmem m;
        m.cand = smem_w;
        m.keep = m.cand + cap;
        m.kv = m.keep + keep_w + keep_pad;
        m.bytes = m.kv + kv_w;
        m.hist = m.bytes + 2 * stage_w;
        m.misc = m.hist + SEL_NBK + 1;
        m.tmpcap = (uint32_t)(m.hist - m.keep);
        return m;
    }
};
// the hashing kernels' keep: s words in 16-byte granules, + one granule
__host__ __device__ inline SelLayout sel_generic_layout(uint32_t cap, uint32_t s) { return {cap, (s + 3u) & ~3u, 4u, SEL_CHUNK + SEL_LOOKAHEAD, SEL_STAGE_WORDS, SEL_MISC_WORDS}; }
__host__ __device__ inline SelLayout sel_walk_layout(uint32_t cap, uint32_t s) { return {cap, (s + 3u) & ~3u, 4u, 0, SELW_STAGE_WORDS, SELW_MISC_WORDS}; }
// the merge stages nothing; keep is the scratch of the final stage: s + ties + one cursor per bucket
__host__ __device__ inline SelLayout sel_merge_layout(uint32_t cap, uint32_t s) { return {cap, s, SEL_NBK + 64, 0, 0, SEL_MISC_WORDS}; }
// ---- K2t stage A (sketch_thresh_walk_kernel<K>): 2 stage buffers [STAGE bytes] | strip [SEG][32] -----------
// Positions per lane per chunk: 4 x an ODD number of word steps (lanes read their staged words an odd number
// of words apart: bank-conflict free) that is a multiple of NB = K / 4 where NB is odd, so that a full
// segment is whole groups of the NB-step loop body and never enters the bounds-checked tail; for even NB one
// checked step remains.
template <int K>
struct SeltGeom {
    static constexpr int NB = K / 4;
    static constexpr int STEPS = NB == 2 ? 17 : NB == 3 ? 21 : NB == 4 ? 17 : NB == 5 ? 15 : 21;  // NB >= 6: whole groups of 3 steps
    static constexpr int SEG = 4 * STEPS;      // 60 .. 84 k-mer positions
    static constexpr int CHUNK = 32 * SEG;     // per warp chunk
    static constexpr int STAGE = (15 + CHUNK + 32 + 48 + 15 + 255) / 256 * 256;  // head + chunk + k + over-read pad; also the dense flush buffer
    static constexpr uint32_t STRIP = 2 * STAGE / 4;                // word offset of the strip
    static constexpr uint32_t SMEM_BYTES = (STRIP + SEG * 32) * 4;
    static_assert(STEPS % 2 == 1 && (NB % 2 == 0 || STEPS % NB == 0), "segment geometry");
    static_assert(STAGE % 16 == 0, "stage buffers start on 16-byte boundaries");
};
// ---- K2t stage B (sketch_thresh_select_kernel): tmp [cap] in 16-byte granules | cur [SEL_NBK] | flag [16] ------
struct SeltSelLayout {
    uint32_t tmp = 0, cur, flag, words;
    __host__ __device__ explicit SeltSelLayout(uint32_t cap) : cur((cap + 3u) & ~3u), flag(cur + SEL_NBK), words(flag + 16) {}
    __host__ __device__ size_t bytes() const { return (size_t)words * 4; }
};

}  // namespace pg
