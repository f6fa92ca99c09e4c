// kmer_walk.cuh -- the register-ring k-mer walk shared by K1 (sketch_fill.cu) and K2
// (sketch_select.cu): one thread walks consecutive k-mer positions of a byte string staged in
// shared memory, 4 bytes (= 4 k-mers) per step.  The murmur3 block pre-mix K(p) of the 4 bytes at
// position p is computed once and kept in a register ring shared by the k/4 k-mers that use it.
//
// A walk kernel is a template on K that opens with PG_WALK_CONSTANTS (K, NB = K/4, TAIL = K%4,
// TAILMASK, LUT = (TAIL == 1), all compile-time), loads the tail table with load_kmix_table when LUT,
// and starts each walk with PG_WALK_PROLOGUE.  PG_KMER_STEP(U, CHECKED, EMIT) is then one word step
// (ring slot U); PG_K1_STEP is the same with the positional store.  They use these locals of the
// enclosing scope:
//   sw, sh                 staged words of the walk (the first at or before its first byte), funnel-shift amount
//   w_cur, w_nxt          the realigned words at the current / next word position      (PG_WALK_PROLOGUE)
//   raw_a, raw_b, swp      raw staged words one step ahead of their use                 (PG_WALK_PROLOGUE)
//   ring[4][NB]            pre-mixes of the last NB word steps                          (PG_WALK_PROLOGUE)
//   sb                     byte pointer: the tail byte of k-mer i is sb[i]      (LUT only)
//   lut_stride, lut_base   shared-memory tail table (256 x kmix(byte)); the stride (4) is a
//                          runtime value so byte*4 + base stays an IMAD on the FMA pipe
//   my_out, i, nk          hashes of k-mers i .. i+3 go to my_out[i ..]; CHECKED guards i+r < nk
#pragma once
#include <stdint.h>
#include <utility>

#include "murmur3.cuh"
#include "tma.cuh"

namespace pg {

// Shared-space load from a 32-bit shared address.  volatile: the rank loop of sketch_thresh_select_kernel
// reads what other threads scattered before a barrier, and the load must stay behind that barrier.
__device__ __forceinline__ uint32_t lds_u32(uint32_t saddr) {
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(saddr));
    return v;
}

// kmix(b) for a single tail byte b, built at compile time
struct KmixTable {
    uint32_t v[256];
};
constexpr uint32_t c_rotl(uint32_t x, int r) { return (x << r) | (x >> (32 - r)); }
constexpr KmixTable make_kmix_table() {
    KmixTable t{};
    for (uint32_t b = 0; b < 256; ++b) t.v[b] = c_rotl(b * MM3_C1, 15) * MM3_C2;
    return t;
}
static __device__ __align__(16) const KmixTable g_kmix_byte = make_kmix_table();

// The tail table into shared memory by one bulk copy that completes on `bar`; called by the thread that
// initialised the barrier.
__device__ __forceinline__ void load_kmix_table(uint32_t *s_lut, uint64_t *bar) {
    mbar_expect_tx(bar, sizeof(KmixTable));
    bulk_g2s(s_lut, &g_kmix_byte, sizeof(KmixTable), bar);
}

#define PG_WALK_CONSTANTS                                                                      \
    constexpr int NB = K / 4;    /* 4-byte body blocks per k-mer */                            \
    constexpr int TAIL = K % 4;  /* tail bytes per k-mer */                                    \
    constexpr uint32_t TAILMASK = TAIL == 1 ? 0xffu : TAIL == 2 ? 0xffffu : 0xffffffu;         \
    constexpr bool LUT = TAIL == 1;                                                            \
    static_assert(NB >= 1 && K <= 32, "walk path: 4 <= k <= 32")

// The k for which the walk kernels (K1, K1r, K2w, K2t) are instantiated.  with_walk_k(k, f) calls
// f(std::integral_constant<int, K>{}) when k is one of them and returns whether it did.
using WalkKs = std::integer_sequence<int, 11, 13, 15, 16, 17, 19, 21, 23, 24, 25, 27, 29, 31, 32>;
template <class F, int... Ks>
bool with_k_in(std::integer_sequence<int, Ks...>, int k, F &f) { return ((k == Ks && (f(std::integral_constant<int, Ks>{}), true)) || ...); }
template <class F>
bool with_walk_k(int k, F &&f) { return with_k_in(WalkKs{}, k, f); }

// The first two realigned words, the raw words one step ahead of them, and word steps 0 .. NB-1,
// which only fill the ring.
#define PG_WALK_PROLOGUE                                                                       \
    uint32_t raw_a = sw[0], raw_b = sw[1];                                                     \
    uint32_t w_cur = __funnelshift_r(raw_a, raw_b, sh); /* bytes 4Q .. 4Q+3 of the walk */     \
    raw_a = raw_b; raw_b = sw[2];                                                              \
    uint32_t w_nxt = __funnelshift_r(raw_a, raw_b, sh); /* bytes 4Q+4 .. 4Q+7 */               \
    raw_a = raw_b; raw_b = sw[3];                                                              \
    const uint32_t *swp = sw + 4;                                                              \
    uint32_t ring[4][NB]; /* ring[r][*]: pre-mixes K(4q+r) of the last NB word steps */        \
    _Pragma("unroll") for (int q = 0; q < NB; ++q) {                                           \
        ring[0][q] = mm3_kmix(w_cur);                                                          \
        ring[1][q] = mm3_kmix(__funnelshift_r(w_cur, w_nxt, 8));                               \
        ring[2][q] = mm3_kmix(__funnelshift_r(w_cur, w_nxt, 16));                              \
        ring[3][q] = mm3_kmix(__funnelshift_r(w_cur, w_nxt, 24));                              \
        w_cur = w_nxt;                                                                         \
        w_nxt = __funnelshift_r(raw_a, raw_b, sh);                                             \
        raw_a = raw_b;                                                                         \
        raw_b = *swp++;                                                                        \
    }

// One word step = 4 k-mers (ring slot U).  EMIT(r, value) consumes the hash of k-mer i + r.
#define PG_KMER_STEP(U, CHECKED, EMIT)                                                         \
    {                                                                                          \
        uint32_t w[4];                                                                         \
        w[0] = w_cur;                                                                          \
        w[1] = __funnelshift_r(w_cur, w_nxt, 8);                                               \
        w[2] = __funnelshift_r(w_cur, w_nxt, 16);                                              \
        w[3] = __funnelshift_r(w_cur, w_nxt, 24);                                              \
        uint32_t h[4];                                                                         \
        _Pragma("unroll") for (int r = 0; r < 4; ++r) {                                        \
            uint32_t x = mm3_round0(ring[r][U]);                                               \
            _Pragma("unroll") for (int j = 1; j < NB; ++j)                                     \
                x = mm3_round(x, ring[r][((U) + j) % NB]);                                     \
            if (LUT) x ^= lds_u32(sb[i + r] * lut_stride + lut_base);                          \
            else if (TAIL) x ^= mm3_kmix(w[r] & TAILMASK);                                     \
            x ^= (uint32_t)K;                                                                  \
            h[r] = mm3_fmix(x);                                                                \
            ring[r][U] = mm3_kmix(w[r]);                                                       \
        }                                                                                      \
        EMIT(0, h[0]);                                                                         \
        if (!(CHECKED) || i + 1 < nk) EMIT(1, h[1]);                                           \
        if (!(CHECKED) || i + 2 < nk) EMIT(2, h[2]);                                           \
        if (!(CHECKED) || i + 3 < nk) EMIT(3, h[3]);                                           \
        w_cur = w_nxt;                                                                         \
        w_nxt = __funnelshift_r(raw_a, raw_b, sh);                                             \
        raw_a = raw_b;                                                                         \
        raw_b = *swp++;                                                                        \
        i += 4;                                                                                \
    }
// The same word step with a ROLLED ring: slot 0 is always the oldest pre-mix and the ring is shifted by one
// after the step ((NB - 1) x 4 register moves), so a loop over steps needs ONE step of code instead of NB
// (k = 31: 15 KB of SASS -> 2.5 KB).  For kernels whose unrolled body no longer fits the instruction caches.
#define PG_KMER_STEP_ROLLED(CHECKED, EMIT)                                                     \
    {                                                                                          \
        uint32_t w[4];                                                                         \
        w[0] = w_cur;                                                                          \
        w[1] = __funnelshift_r(w_cur, w_nxt, 8);                                               \
        w[2] = __funnelshift_r(w_cur, w_nxt, 16);                                              \
        w[3] = __funnelshift_r(w_cur, w_nxt, 24);                                              \
        uint32_t h[4];                                                                         \
        _Pragma("unroll") for (int r = 0; r < 4; ++r) {                                        \
            uint32_t x = mm3_round0(ring[r][0]);                                               \
            _Pragma("unroll") for (int j = 1; j < NB; ++j) x = mm3_round(x, ring[r][j]);       \
            if (LUT) x ^= lds_u32(sb[i + r] * lut_stride + lut_base);                          \
            else if (TAIL) x ^= mm3_kmix(w[r] & TAILMASK);                                     \
            x ^= (uint32_t)K;                                                                  \
            h[r] = mm3_fmix(x);                                                                \
            _Pragma("unroll") for (int j = 0; j + 1 < NB; ++j) ring[r][j] = ring[r][j + 1];    \
            ring[r][NB - 1] = mm3_kmix(w[r]);                                                  \
        }                                                                                      \
        EMIT(0, h[0]);                                                                         \
        if (!(CHECKED) || i + 1 < nk) EMIT(1, h[1]);                                           \
        if (!(CHECKED) || i + 2 < nk) EMIT(2, h[2]);                                           \
        if (!(CHECKED) || i + 3 < nk) EMIT(3, h[3]);                                           \
        w_cur = w_nxt;                                                                         \
        w_nxt = __funnelshift_r(raw_a, raw_b, sh);                                             \
        raw_a = raw_b;                                                                         \
        raw_b = *swp++;                                                                        \
        i += 4;                                                                                \
    }
// Rotate the ring by G slots (slot G becomes slot 0).  A loop body of G unrolled PG_KMER_STEP(0..G-1) followed by
// this rotation is the middle ground between the fully unrolled NB-step body (no moves, NB steps of code) and the
// rolled one ((NB - 1) x 4 moves per step): about (NB + 1) x 4 / G moves per step.
#define PG_RING_ROTATE(G)                                                                      \
    {                                                                                          \
        _Pragma("unroll") for (int r = 0; r < 4; ++r) {                                        \
            uint32_t t_[NB];                                                                   \
            _Pragma("unroll") for (int q = 0; q < NB; ++q) t_[q] = ring[r][(q + (G)) % NB];    \
            _Pragma("unroll") for (int q = 0; q < NB; ++q) ring[r][q] = t_[q];                 \
        }                                                                                      \
    }
// ---- the canonical walk (PG_KMER_CANONICAL): each window hashes the smaller of itself and its reverse complement.
// Beside s_in the chunk is staged complemented (c[q] = complement(byte q)).  The reverse strand's block j of the
// window at p is the byte-reversed complemented word at p + k - 4 - 4j, so its pre-mix R(q) = kmix(bswap(cword(q)))
// is shared between windows like the forward K(q): a second ring, rring[r][*], holds R(4q + r + TAIL) of the last NB
// word steps, fed by a complemented stream that runs TAIL bytes ahead of the forward one (cw, csh).  Its tail is the
// complemented bytes p .. p + TAIL - 1 in reverse.  The strand is decided before hashing: w's first 4 bytes as a
// big-endian word (from a third stream, l_*, the forward bytes at the window itself) against rc(w)'s, which are
// cword(p + k - 4) read little-endian, the previous step's complemented word (cprev); only a tie compares further
// bytes.  The NB rounds and the fmix then run once, each block selected from the chosen ring.  Extra locals:
//   cw, csh                complemented staged words from byte b0 + TAIL, funnel-shift amount
//   sbf, sbc               s_in + b0 and s_rc + b0: forward and complemented byte of window i is sbf[i], sbc[i]

// Whether rc(w) < w, given that their first 4 bytes are equal: bytes 4 .. K - 1 of w (f) against those of rc(w)
// (complemented bytes of w read backwards, c).
template <int K>
__device__ __forceinline__ bool canon_tie(const uint8_t *f, const uint8_t *c) {
    for (int t = 4; t < K; ++t) {
        const uint8_t a = f[t], b = c[K - 1 - t];
        if (a != b) return b < a;
    }
    return false;
}

// rc(w)'s tail: complemented bytes p + TAIL - 1 .. p of the window at p, little-endian
template <int TAIL>
__device__ __forceinline__ uint32_t canon_tail(const uint8_t *c) {
    uint32_t t = 0;
#pragma unroll
    for (int x = 0; x < TAIL; ++x) t |= (uint32_t)c[x] << (8 * (TAIL - 1 - x));
    return t;
}

// After PG_WALK_PROLOGUE: the complemented stream, its ring and cprev, and the lagging forward stream.
#define PG_CANON_PROLOGUE                                                                      \
    uint32_t craw_a = cw[0], craw_b = cw[1];                                                   \
    uint32_t c_cur = __funnelshift_r(craw_a, craw_b, csh);                                     \
    craw_a = craw_b; craw_b = cw[2];                                                           \
    uint32_t c_nxt = __funnelshift_r(craw_a, craw_b, csh);                                     \
    craw_a = craw_b; craw_b = cw[3];                                                           \
    const uint32_t *cwp = cw + 4;                                                              \
    uint32_t rring[4][NB], cprev[4];                                                           \
    _Pragma("unroll") for (int q = 0; q < NB; ++q) {                                           \
        _Pragma("unroll") for (int r = 0; r < 4; ++r) {                                        \
            cprev[r] = __funnelshift_r(c_cur, c_nxt, 8 * r);                                   \
            rring[r][q] = mm3_kmix(__byte_perm(cprev[r], 0, 0x0123));                          \
        }                                                                                      \
        c_cur = c_nxt;                                                                         \
        c_nxt = __funnelshift_r(craw_a, craw_b, csh);                                          \
        craw_a = craw_b;                                                                       \
        craw_b = *cwp++;                                                                       \
    }                                                                                          \
    uint32_t lraw_a = sw[0], lraw_b = sw[1];                                                   \
    uint32_t l_cur = __funnelshift_r(lraw_a, lraw_b, sh);                                      \
    lraw_a = lraw_b; lraw_b = sw[2];                                                           \
    uint32_t l_nxt = __funnelshift_r(lraw_a, lraw_b, sh);                                      \
    lraw_a = lraw_b; lraw_b = sw[3];                                                           \
    const uint32_t *lwp = sw + 4;

// One canonical word step = 4 windows (ring slot U of both rings), unchecked.  EMIT(r, value) as PG_KMER_STEP.
#define PG_KMER_STEP_CANON(U, EMIT)                                                            \
    {                                                                                          \
        uint32_t w[4], c[4];                                                                   \
        uint32_t h[4];                                                                         \
        _Pragma("unroll") for (int r = 0; r < 4; ++r) {                                        \
            w[r] = __funnelshift_r(w_cur, w_nxt, 8 * r);                                       \
            c[r] = __funnelshift_r(c_cur, c_nxt, 8 * r);                                       \
            const uint32_t a_ = __byte_perm(__funnelshift_r(l_cur, l_nxt, 8 * r), 0, 0x0123);  \
            bool rc_ = a_ > cprev[r];                                                          \
            if (a_ == cprev[r]) rc_ = canon_tie<K>(sbf + i + r, sbc + i + r);                  \
            uint32_t x = mm3_round0(rc_ ? rring[r][((U) + NB - 1) % NB] : ring[r][U]);         \
            _Pragma("unroll") for (int j = 1; j < NB; ++j)                                     \
                x = mm3_round(x, rc_ ? rring[r][((U) + NB - 1 - j) % NB] : ring[r][((U) + j) % NB]); \
            if (LUT) x ^= lds_u32((rc_ ? sbc[i + r] : sb[i + r]) * lut_stride + lut_base);     \
            else if (TAIL) x ^= mm3_kmix(rc_ ? canon_tail<TAIL>(sbc + i + r) : w[r] & TAILMASK); \
            x ^= (uint32_t)K;                                                                  \
            h[r] = mm3_fmix(x);                                                                \
            ring[r][U] = mm3_kmix(w[r]);                                                       \
            rring[r][U] = mm3_kmix(__byte_perm(c[r], 0, 0x0123));                              \
            cprev[r] = c[r];                                                                   \
        }                                                                                      \
        EMIT(0, h[0]);                                                                         \
        EMIT(1, h[1]);                                                                         \
        EMIT(2, h[2]);                                                                         \
        EMIT(3, h[3]);                                                                         \
        w_cur = w_nxt;                                                                         \
        w_nxt = __funnelshift_r(raw_a, raw_b, sh);                                             \
        raw_a = raw_b;                                                                         \
        raw_b = *swp++;                                                                        \
        c_cur = c_nxt;                                                                         \
        c_nxt = __funnelshift_r(craw_a, craw_b, csh);                                          \
        craw_a = craw_b;                                                                       \
        craw_b = *cwp++;                                                                       \
        l_cur = l_nxt;                                                                         \
        l_nxt = __funnelshift_r(lraw_a, lraw_b, sh);                                           \
        lraw_a = lraw_b;                                                                       \
        lraw_b = *lwp++;                                                                       \
        i += 4;                                                                                \
    }

// positional store: hash of k-mer i + r -> my_out[i + r]
#define PG_EMIT_POSITIONAL(R_, H_) my_out[i + (R_)] = (H_)
#define PG_K1_STEP(U, CHECKED) PG_KMER_STEP(U, CHECKED, PG_EMIT_POSITIONAL)

}  // namespace pg
