// seqhash.cu -- seqhash.Hash and seqhash.RotateSequence (/root/reference/seqhash/seqhash.go:78-223)
// for a ragged batch: one sequence type and one circular / double-stranded choice per call.
//
// Stages, each a kernel (DESIGN.md §4 "Seqhash"):
//   1. orientation and rotation (circular or double-stranded input only): per sequence, the start of
//      the least rotation of s and of rc(s) and the strand whose deterministic string is smaller.
//      rc(s) is never materialised: it is s read backwards through transform's complement table.
//   2. canonical copy + alphabet check: the deterministic bytes are written once, at the input's
//      offsets, into a scratch buffer; the first byte outside the alphabet (or >= 0x80) is recorded.
//   3. BLAKE3 chunks: one thread per 1 KiB chunk, 16 block compressions.
//   4. BLAKE3 parents (sequences of more than one chunk): one CTA per sequence, level by level.
//   5. finish: error codes, and the root chaining value (or zeros) as the digest.
// Sequence bytes are folded on every read (ASCII upper-case, then U -> T for RNA), so the raw input is
// never rewritten; hashing reads only the canonical copy.
#include <algorithm>

#include "common.cuh"

namespace pg {

namespace {

// ---- sequence access ---------------------------------------------------------------------------
enum Fold : int { FOLD_NONE = 0, FOLD_UPPER = 1, FOLD_RNA = 2 };

__device__ __forceinline__ uint8_t fold(uint8_t c, int mode) {
    if (mode == FOLD_NONE) return c;
    if (c >= 'a' && c <= 'z') c -= 32;  // strings.ToUpper on ASCII
    if (mode == FOLD_RNA && c == 'U') c = 'T';
    return c;
}

// Byte maps of one call in shared memory: map[0][c] = fold(c), map[1][c] = complement(fold(c)).  Every CTA
// fills them once; a lookup replaces the compare chains on every read.
__device__ __forceinline__ void fill_maps(uint8_t (*map)[256], int mode) {
    for (int c = threadIdx.x; c < 256; c += blockDim.x) {
        map[0][c] = fold((uint8_t)c, mode);
        map[1][c] = complement(fold((uint8_t)c, mode));
    }
    __syncthreads();
}

// One strand of one sequence: s, or rc(s) read backwards through the complement table.
struct Strand {
    const uint8_t *p;
    uint64_t n;
    const uint8_t *map;  // map[0] (s) or map[1] (rc(s)) of fill_maps
    bool rc;
    __device__ __forceinline__ uint8_t at(uint64_t q) const {  // q in [0, n)
        return map[__ldg(p + (rc ? n - 1 - q : q))];
    }
    __device__ __forceinline__ uint8_t rot(uint64_t start, uint64_t t) const {  // start, t < n
        uint64_t q = start + t;
        return at(q >= n ? q - n : q);
    }
};

// First t in [0, lim) where rotation a of A and rotation b of B differ, or lim; 128 bytes per step, and the
// same value in every lane.  lim <= n of both strands.
__device__ uint64_t first_mismatch(const Strand &A, uint64_t a, const Strand &B, uint64_t b, uint64_t lim, int lane) {
    for (uint64_t t0 = 0; t0 < lim; t0 += 128) {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const uint64_t t = t0 + 32 * k + lane;
            const bool diff = t < lim && A.rot(a, t) != B.rot(b, t);
            const unsigned m = __ballot_sync(0xffffffffu, diff);
            if (m) return t0 + 32 * k + (__ffs(m) - 1);
        }
    }
    return lim;
}

// Smallest start of the least rotation by the two-pointer algorithm (i, j, k): every mismatch moves i or j
// past the k + 1 starts it rules out, so at most 2n starts are discarded and the cost is O(n) for any input.
__device__ uint64_t least_rotation_two_pointer(const Strand &S, int lane) {
    const uint64_t n = S.n;
    uint64_t i = 0, j = 1;
    while (i < n && j < n) {
        const uint64_t t = first_mismatch(S, i, S, j, n, lane);
        if (t == n) break;  // rotations i and j are equal: the string is periodic, min(i, j) is the answer
        if (S.rot(i, t) > S.rot(j, t)) i += t + 1;
        else j += t + 1;
        if (i == j) ++j;
    }
    return i < j ? i : j;
}

// 16-byte prefixes of rotations, big-endian in (hi, lo): ordered as the rotations' first 16 bytes of the
// infinite repetition of the string, so the least rotation always has the least key.
struct Key {
    uint64_t hi, lo;
};
__device__ __forceinline__ bool key_less(Key a, Key b) { return a.hi < b.hi || (a.hi == b.hi && a.lo < b.lo); }
__device__ __forceinline__ void key_push(Key &k, uint8_t c) {
    k.hi = (k.hi << 8) | (k.lo >> 56);
    k.lo = (k.lo << 8) | c;
}

constexpr int ROT_MAX_CANDIDATES = 64;  // starts kept for the tournament; more fall back to the two-pointer walk
constexpr uint64_t ROT_MIN_SEGMENT = 64;  // starts per thread at least, so the 16-byte window warm-up stays small

// Least rotation of strand S by the whole CTA.  Pass 1: every thread slides a 16-byte window over its own
// segment of starts and keeps the least key; the CTA reduces it.  Pass 2: the starts holding that key are
// collected.  Warp 0 then either compares the (<= ROT_MAX_CANDIDATES) candidates against each other, or,
// when the key does not separate them (low-entropy or periodic input), runs the two-pointer walk.
template <int NT>
__device__ uint64_t least_rotation_cta(const Strand &S, Key *red, uint64_t *cand, uint32_t *n_cand, uint32_t *again) {
    const uint64_t n = S.n;
    if (n <= 1) return 0;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint64_t seg = std::max<uint64_t>(uint64_t(ROT_MIN_SEGMENT), (n + NT - 1) / NT);
    const uint64_t b = (uint64_t)tid * seg, e = std::min<uint64_t>(n, b + seg);
    Key best = {~0ull, ~0ull}, mine;
    uint64_t first = 0;  // the thread's first start holding its least key, and how many do
    uint32_t count = 0;
    if (b < e) {
        Key k = {0, 0};
        uint64_t q = b % n;
        for (int r = 0; r < 16; ++r) {
            key_push(k, S.at(q));
            if (++q == n) q = 0;
        }
        for (uint64_t p = b;;) {
            if (key_less(k, best)) {
                best = k;
                first = p;
                count = 1;
            } else if (k.hi == best.hi && k.lo == best.lo) {
                ++count;
            }
            if (++p == e) break;
            key_push(k, S.at(q));
            if (++q == n) q = 0;
        }
    }
    mine = best;
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        Key other = {__shfl_xor_sync(0xffffffffu, best.hi, o), __shfl_xor_sync(0xffffffffu, best.lo, o)};
        if (key_less(other, best)) best = other;
    }
    if (lane == 0) red[warp] = best;
    if (tid == 0) *n_cand = *again = 0;
    __syncthreads();
    best = red[0];
    for (int w = 1; w < NT / 32; ++w)
        if (key_less(red[w], best)) best = red[w];
    const bool holds = count && mine.hi == best.hi && mine.lo == best.lo;
    if (holds && count == 1) {
        const uint32_t slot = atomicAdd(n_cand, 1u);
        if (slot < ROT_MAX_CANDIDATES) cand[slot] = first;
    } else if (holds) {
        *again = 1;
    }
    __syncthreads();
    if (*again) {  // some thread holds the least key more than once: collect every start in a second pass
        __syncthreads();  // every thread has read *again
        if (tid == 0) *n_cand = 0;
        __syncthreads();
    }
    if (*again && b < e) {
        Key k = {0, 0};
        uint64_t q = b % n;
        for (int r = 0; r < 16; ++r) {
            key_push(k, S.at(q));
            if (++q == n) q = 0;
        }
        for (uint64_t p = b;;) {
            if (k.hi == best.hi && k.lo == best.lo) {
                const uint32_t slot = atomicAdd(n_cand, 1u);
                if (slot < ROT_MAX_CANDIDATES) cand[slot] = p;
            }
            if (++p == e) break;
            key_push(k, S.at(q));
            if (++q == n) q = 0;
        }
    }
    __syncthreads();
    uint64_t r = 0;
    if (warp == 0) {
        const uint32_t nc = *n_cand;
        if (nc <= ROT_MAX_CANDIDATES) {
            r = cand[0];
            for (uint32_t c = 1; c < nc; ++c) {
                const uint64_t x = cand[c];
                const uint64_t t = first_mismatch(S, r, S, x, n, lane);
                if (t < n ? S.rot(x, t) < S.rot(r, t) : x < r) r = x;
            }
        } else {
            r = least_rotation_two_pointer(S, lane);
        }
    }
    __syncthreads();  // red / cand / n_cand are reused by the next call
    return r;
}

// ---- stage 1: orientation and rotation ----------------------------------------------------------
// Circular input, one CTA per sequence: start[i] = start of the deterministic rotation, rc[i] = 1 when it
// is a rotation of rc(s).  Without double-stranded only s is rotated (rc may be NULL): this is also
// pg_least_rotation_batch (mode FOLD_NONE).
template <int NT>
__global__ void __launch_bounds__(NT) seqhash_rotate_kernel(const uint8_t *__restrict__ in, const uint64_t *__restrict__ off,
                                                            uint64_t n_seq, int mode, int ds, uint64_t *__restrict__ start,
                                                            uint8_t *__restrict__ rc) {
    __shared__ Key red[NT / 32];
    __shared__ uint64_t cand[ROT_MAX_CANDIDATES];
    __shared__ uint32_t n_cand, again;
    __shared__ uint8_t map[2][256];
    fill_maps(map, mode);
    for (uint64_t i = blockIdx.x; i < n_seq; i += gridDim.x) {
        const uint64_t b = off[i], n = off[i + 1] - b;
        const Strand f = {in + b, n, map[0], false};
        const uint64_t rf = least_rotation_cta<NT>(f, red, cand, &n_cand, &again);
        uint64_t r = rf;
        bool use_rc = false;
        if (ds) {
            const Strand v = {in + b, n, map[1], true};
            const uint64_t rr = least_rotation_cta<NT>(v, red, cand, &n_cand, &again);
            if (threadIdx.x < 32) {  // sort.Strings of the two rotations (seqhash.go:181-183)
                const uint64_t t = first_mismatch(f, rf, v, rr, n, threadIdx.x);
                use_rc = t < n && v.rot(rr, t) < f.rot(rf, t);
                r = use_rc ? rr : rf;
            }
        }
        if (threadIdx.x == 0) {
            start[i] = r;
            if (rc) rc[i] = use_rc;
        }
    }
}

// Linear double-stranded input, one warp per sequence: rc[i] = 1 when rc(s) < s (seqhash.go:186-189).
__global__ void __launch_bounds__(256) seqhash_strand_kernel(const uint8_t *__restrict__ in, const uint64_t *__restrict__ off,
                                                             uint64_t n_seq, int mode, uint64_t *__restrict__ start,
                                                             uint8_t *__restrict__ rc) {
    __shared__ uint8_t map[2][256];
    fill_maps(map, mode);
    const int lane = threadIdx.x & 31;
    const uint64_t warps = (uint64_t)gridDim.x * (blockDim.x >> 5);
    for (uint64_t i = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); i < n_seq; i += warps) {
        const uint64_t b = off[i], n = off[i + 1] - b;
        const Strand f = {in + b, n, map[0], false}, v = {in + b, n, map[1], true};
        const uint64_t t = first_mismatch(f, 0, v, 0, n, lane);
        if (lane == 0) {
            start[i] = 0;
            rc[i] = t < n && v.at(t) < f.at(t);
        }
    }
}

// ---- stage 2: canonical copy and alphabet check --------------------------------------------------
// Seqhash alphabets (seqhash.go:155,168): bit c set when upper-case letter c is allowed
struct Alphabet {
    uint32_t w[4];
};
__host__ Alphabet make_alphabet(const char *letters) {
    Alphabet a = {{0, 0, 0, 0}};
    for (const char *p = letters; *p; ++p) a.w[(uint8_t)*p >> 5] |= 1u << ((uint8_t)*p & 31);
    return a;
}

// index of the sequence holding byte g (relative to off[0]) among sequences [lo, hi]: the last i with
// off[i] - off[0] <= g
__device__ __forceinline__ uint64_t seq_of_byte(const uint64_t *off, uint64_t lo, uint64_t hi, uint64_t g) {
    const uint64_t b0 = off[0];
    while (lo < hi) {
        const uint64_t mid = (lo + hi + 1) >> 1;
        if (off[mid] - b0 <= g) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// One thread per 16 bytes of the canonical buffer (16-byte aligned, indexed like the input relative to
// off[0]).  start / rc NULL: the canonical bytes are the folded input (linear single-stranded).
// first_bad[i] = the least byte index (relative to off[0]) of sequence i holding a byte >= 0x80 or a folded
// letter outside the alphabet; the caller set it to ~0.
__global__ void __launch_bounds__(256) seqhash_canon_kernel(const uint8_t *__restrict__ in, const uint64_t *__restrict__ off,
                                                            uint64_t n_seq, uint64_t total, int mode, Alphabet alpha,
                                                            const uint64_t *__restrict__ start, const uint8_t *__restrict__ rc,
                                                            uint8_t *__restrict__ canon, unsigned long long *__restrict__ first_bad) {
    __shared__ uint8_t map[2][256];
    __shared__ uint64_t tile_seq[2];
    fill_maps(map, mode);
    const uint64_t b0 = off[0], tile = 16ull * blockDim.x;
    for (uint64_t t0 = blockIdx.x * tile; t0 < total; t0 += gridDim.x * tile) {
        __syncthreads();  // tile_seq of the previous tile is no longer read
        if (threadIdx.x < 2) tile_seq[threadIdx.x] = seq_of_byte(off, 0, n_seq - 1, threadIdx.x ? std::min(total, t0 + tile) - 1 : t0);
        __syncthreads();
        const uint64_t g0 = t0 + 16ull * threadIdx.x, s_lo = tile_seq[0], s_hi = tile_seq[1];
        if (g0 >= total) continue;
        uint64_t i = seq_of_byte(off, s_lo, s_hi, g0);
        uint64_t sb = off[i] - b0, se = off[i + 1] - b0;
        const bool rci = rc ? rc[i] != 0 : false;
        Strand S = {in + b0 + sb, se - sb, map[rci], rci};
        uint64_t r = start ? start[i] : 0;
        uint64_t bad = ~0ull;
        uint32_t w[4] = {0, 0, 0, 0};
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            const uint64_t g = g0 + k;
            if (g >= total) break;
            if (g >= se) {  // next sequence (empty ones skipped)
                if (bad != ~0ull) atomicMin(first_bad + i, (unsigned long long)bad);
                bad = ~0ull;
                i = seq_of_byte(off, i + 1, s_hi, g);
                sb = off[i] - b0;
                se = off[i + 1] - b0;
                const bool rcn = rc ? rc[i] != 0 : false;
                S = {in + b0 + sb, se - sb, map[rcn], rcn};
                r = start ? start[i] : 0;
            }
            const uint8_t raw = __ldg(in + b0 + g), c = map[0][raw];
            if (bad == ~0ull && (raw >= 0x80 || !((alpha.w[c >> 5] >> (c & 31)) & 1u))) bad = g;
            const uint8_t out = (start || rc) ? S.rot(r, g - sb) : c;
            w[k >> 2] |= (uint32_t)out << (8 * (k & 3));
        }
        if (bad != ~0ull) atomicMin(first_bad + i, (unsigned long long)bad);
        *reinterpret_cast<uint4 *>(canon + g0) = make_uint4(w[0], w[1], w[2], w[3]);
    }
}

// ---- stage 3-4: BLAKE3 (hash mode, 32-byte output), from the specification --------------------------
__constant__ uint32_t c_iv[8] = {0x6A09E667u, 0xBB67AE85u, 0x3C6EF372u, 0xA54FF53Au,
                                 0x510E527Fu, 0x9B05688Cu, 0x1F83D9ABu, 0x5BE0CD19u};
constexpr uint32_t IV0 = 0x6A09E667u, IV1 = 0xBB67AE85u, IV2 = 0x3C6EF372u, IV3 = 0xA54FF53Au;
constexpr uint32_t CHUNK_START = 1, CHUNK_END = 2, PARENT = 4, ROOT = 8;
constexpr uint64_t CHUNK = 1024;

__device__ __forceinline__ uint32_t rotr(uint32_t x, int r) { return __funnelshift_r(x, x, r); }
__device__ __forceinline__ void gmix(uint32_t &a, uint32_t &b, uint32_t &c, uint32_t &d, uint32_t x, uint32_t y) {
    a = a + b + x; d = rotr(d ^ a, 16); c = c + d; b = rotr(b ^ c, 12);
    a = a + b + y; d = rotr(d ^ a, 8);  c = c + d; b = rotr(b ^ c, 7);
}

// the message word order of rounds 0..6 (round r+1 permutes round r by 2,6,3,10,7,0,4,13,1,11,12,5,9,14,15,8)
#define SH_ROUND(m, s0, s1, s2, s3, s4, s5, s6, s7, s8, s9, s10, s11, s12, s13, s14, s15) \
    gmix(v[0], v[4], v[8], v[12], m[s0], m[s1]);                                            \
    gmix(v[1], v[5], v[9], v[13], m[s2], m[s3]);                                            \
    gmix(v[2], v[6], v[10], v[14], m[s4], m[s5]);                                           \
    gmix(v[3], v[7], v[11], v[15], m[s6], m[s7]);                                           \
    gmix(v[0], v[5], v[10], v[15], m[s8], m[s9]);                                           \
    gmix(v[1], v[6], v[11], v[12], m[s10], m[s11]);                                         \
    gmix(v[2], v[7], v[8], v[13], m[s12], m[s13]);                                          \
    gmix(v[3], v[4], v[9], v[14], m[s14], m[s15]);

// h <- the chaining value (first 8 output words) of compressing block m under h
__device__ __forceinline__ void compress(uint32_t h[8], const uint32_t m[16], uint64_t counter, uint32_t blen, uint32_t flags) {
    uint32_t v[16] = {h[0], h[1], h[2], h[3], h[4], h[5], h[6], h[7],
                      IV0, IV1, IV2, IV3, (uint32_t)counter, (uint32_t)(counter >> 32), blen, flags};
    SH_ROUND(m, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15)
    SH_ROUND(m, 2, 6, 3, 10, 7, 0, 4, 13, 1, 11, 12, 5, 9, 14, 15, 8)
    SH_ROUND(m, 3, 4, 10, 12, 13, 2, 7, 14, 6, 5, 9, 0, 11, 15, 8, 1)
    SH_ROUND(m, 10, 7, 12, 9, 14, 3, 13, 15, 4, 0, 11, 2, 5, 8, 1, 6)
    SH_ROUND(m, 12, 13, 9, 11, 15, 10, 14, 8, 7, 2, 5, 3, 0, 1, 6, 4)
    SH_ROUND(m, 9, 14, 11, 5, 8, 12, 15, 1, 13, 3, 0, 10, 2, 6, 4, 7)
    SH_ROUND(m, 11, 15, 5, 0, 1, 9, 8, 6, 14, 10, 2, 12, 3, 4, 7, 13)
#pragma unroll
    for (int k = 0; k < 8; ++k) h[k] = v[k] ^ v[k + 8];
}
#undef SH_ROUND

__device__ __forceinline__ uint64_t chunks_of(uint64_t len) { return len ? (len + CHUNK - 1) / CHUNK : 1; }
// Chaining-value slot of the first chunk of sequence i: (off[i] - off[0]) / 1024 + i.  Consecutive slots
// differ by at least the chunk count of the earlier sequence, so no prefix sum is needed and the slots
// stay below total / 1024 + n.
__device__ __forceinline__ uint64_t slot_of(const uint64_t *off, uint64_t i) { return (off[i] - off[0]) / CHUNK + i; }

// One thread per chaining-value slot (ONE_CHUNK: every sequence <= 1 KiB and slot = sequence).  The thread
// hashes chunk t of its sequence: 16 compressions of 64-byte blocks, counter t, ROOT on the last block of a
// single-chunk sequence.  The canonical buffer has 64 bytes of slack, so the aligned word loads may run
// past the end of the data.
template <bool ONE_CHUNK>
__global__ void __launch_bounds__(128) blake3_chunk_kernel(const uint8_t *__restrict__ canon, const uint64_t *__restrict__ off,
                                                           uint64_t n_seq, uint64_t n_slots, uint32_t *__restrict__ cv) {
    __shared__ uint64_t tile_seq[2];
    const uint64_t b0 = off[0];
    for (uint64_t g_first = (uint64_t)blockIdx.x * blockDim.x; g_first < n_slots; g_first += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t g = g_first + threadIdx.x;
        uint64_t i = g, t = 0;
        if (!ONE_CHUNK) {
            __syncthreads();  // tile_seq of the previous tile is no longer read
            if (threadIdx.x < 2) {  // the sequences of the tile's first and last slot
                const uint64_t x = threadIdx.x ? std::min(n_slots, g_first + blockDim.x) - 1 : g_first;
                uint64_t lo = 0, hi = n_seq - 1;
                while (lo < hi) {
                    const uint64_t mid = (lo + hi + 1) >> 1;
                    if (slot_of(off, mid) <= x) lo = mid;
                    else hi = mid - 1;
                }
                tile_seq[threadIdx.x] = lo;
            }
            __syncthreads();
            if (g >= n_slots) continue;
            uint64_t lo = tile_seq[0], hi = tile_seq[1];  // the last sequence whose first slot is <= g
            while (lo < hi) {
                const uint64_t mid = (lo + hi + 1) >> 1;
                if (slot_of(off, mid) <= g) lo = mid;
                else hi = mid - 1;
            }
            i = lo;
            t = g - slot_of(off, i);
        } else if (g >= n_slots) {
            continue;
        }
        const uint64_t len = off[i + 1] - off[i], nc = chunks_of(len);
        if (t >= nc) continue;  // a slot between two sequences
        const uint64_t cb = off[i] - b0 + t * CHUNK;
        const uint32_t cl = (uint32_t)std::min<uint64_t>(uint64_t(CHUNK), len - t * CHUNK);
        const uint32_t nb = cl ? (cl + 63) / 64 : 1;
        uint32_t h[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) h[k] = c_iv[k];
        for (uint32_t blk = 0; blk < nb; ++blk) {
            const uint64_t a = cb + 64ull * blk;
            const uint32_t *w = reinterpret_cast<const uint32_t *>(canon + (a & ~3ull));
            const int sh = (int)(a & 3) * 8;
            const int blen = (int)std::min<uint32_t>(64, cl - 64 * blk);
            uint32_t m[16];
            uint32_t prev = __ldg(w);
#pragma unroll
            for (int k = 0; k < 16; ++k) {
                const uint32_t next = __ldg(w + k + 1);
                const uint32_t x = __funnelshift_r(prev, next, sh);
                const int vb = blen - 4 * k;
                m[k] = vb >= 4 ? x : vb <= 0 ? 0u : x & ((1u << (8 * vb)) - 1u);
                prev = next;
            }
            const uint32_t flags = (blk == 0 ? CHUNK_START : 0) | (blk + 1 == nb ? CHUNK_END : 0) | (blk + 1 == nb && nc == 1 ? ROOT : 0);
            compress(h, m, t, (uint32_t)blen, flags);
        }
        uint4 *dst = reinterpret_cast<uint4 *>(cv + 8 * g);
        dst[0] = make_uint4(h[0], h[1], h[2], h[3]);
        dst[1] = make_uint4(h[4], h[5], h[6], h[7]);
    }
}

// One CTA per sequence of more than one chunk.  Level by level, in place: node j of a level with m nodes is
// at slot first + j * step; nodes 2j and 2j+1 become node j of the next level (at node 2j's slot), an odd
// last node is carried up unchanged.  This is BLAKE3's left-balanced tree.  ROOT goes on the one parent of
// the level with two nodes.  The root chaining value ends at the sequence's first slot.
__global__ void __launch_bounds__(256) blake3_tree_kernel(const uint64_t *__restrict__ off, uint64_t n_seq, uint32_t *cv) {
    for (uint64_t i = blockIdx.x; i < n_seq; i += gridDim.x) {
        const uint64_t nc = chunks_of(off[i + 1] - off[i]);
        if (nc <= 1) continue;
        uint32_t *base = cv + 8 * slot_of(off, i);
        for (uint64_t step = 1, m = nc; m > 1; step *= 2, m = (m + 1) / 2) {
            for (uint64_t j = threadIdx.x; j < m / 2; j += blockDim.x) {
                uint32_t *left = base + 8 * (2 * j * step);
                const uint32_t *right = left + 8 * step;
                uint32_t msg[16], h[8];
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    msg[k] = left[k];
                    msg[k + 8] = right[k];
                    h[k] = c_iv[k];
                }
                compress(h, msg, 0, 64, PARENT | (m == 2 ? ROOT : 0));
#pragma unroll
                for (int k = 0; k < 8; ++k) left[k] = h[k];
            }
            __syncthreads();  // the next level reads this level's nodes
        }
    }
}

// ---- stage 5 ----------------------------------------------------------------------------------
// err 0 ok, 1 letter outside the alphabet, 2 double-stranded protein, 3 byte >= 0x80 first; pos = byte index
// in the sequence (0 unless 1 or 3).  Failed sequences get a zero digest.
template <bool ONE_CHUNK>
__global__ void __launch_bounds__(256) seqhash_finish_kernel(const uint8_t *__restrict__ in, const uint64_t *__restrict__ off,
                                                             uint64_t n_seq, int protein_ds, const unsigned long long *__restrict__ first_bad,
                                                             const uint32_t *__restrict__ cv, uint8_t *__restrict__ digest,
                                                             int32_t *__restrict__ err_code, uint64_t *__restrict__ err_pos) {
    const uint64_t b0 = off[0];
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_seq; i += stride) {
        const uint64_t fb = first_bad[i];
        int32_t code = 0;
        uint64_t pos = 0;
        if (fb != ~0ull) {
            code = in[b0 + fb] >= 0x80 ? 3 : 1;
            pos = fb - (off[i] - b0);
        } else if (protein_ds) {
            code = 2;
        }
        const uint32_t *h = cv + 8 * (ONE_CHUNK ? i : slot_of(off, i));
        uint32_t *d = reinterpret_cast<uint32_t *>(digest + 32 * i);  // the digest array is 4-byte aligned
#pragma unroll
        for (int k = 0; k < 8; ++k) d[k] = code ? 0u : h[k];
        if (err_code) err_code[i] = code;
        if (err_pos) err_pos[i] = pos;
    }
}

constexpr int ROT_NT_SHORT = 128, ROT_NT_LONG = 512;
constexpr uint64_t ROT_LONG = 1ull << 16;  // sequences this long get the wider CTA

int launch_rotate(const uint8_t *d_in, const uint64_t *d_off, uint64_t n, uint64_t max_len, int mode, bool ds,
                  uint64_t *d_start, uint8_t *d_rc, cudaStream_t st) {
    const unsigned grid = (unsigned)std::min<uint64_t>(n, 0x7fffffffull);
    if (max_len >= ROT_LONG) {
        seqhash_rotate_kernel<ROT_NT_LONG><<<grid, ROT_NT_LONG, 0, st>>>(d_in, d_off, n, mode, ds, d_start, d_rc);
        PG_LAUNCH_CHECK("seqhash_rotate_kernel<512>");
    } else {
        seqhash_rotate_kernel<ROT_NT_SHORT><<<grid, ROT_NT_SHORT, 0, st>>>(d_in, d_off, n, mode, ds, d_start, d_rc);
        PG_LAUNCH_CHECK("seqhash_rotate_kernel<128>");
    }
    return PG_OK;
}

unsigned flat_grid(uint64_t work, int threads) {
    return (unsigned)std::max<uint64_t>(1, std::min<uint64_t>((work + threads - 1) / threads, (uint64_t)sm_count() * 64));
}

}  // namespace

int launch_least_rotation(const uint8_t *d_in, const uint64_t *d_off, uint64_t n, uint64_t max_len, uint64_t *d_rotation,
                           cudaStream_t st) {
    if (n == 0) return PG_OK;
    return launch_rotate(d_in, d_off, n, max_len, FOLD_NONE, false, d_rotation, nullptr, st);
}

int launch_seqhash(const uint8_t *d_in, const uint64_t *d_off, uint64_t n, uint64_t max_len, uint64_t total, int seq_type,
                   uint32_t flags, uint8_t *d_digest, int32_t *d_err, uint64_t *d_pos, cudaStream_t st) {
    if (n == 0) return PG_OK;
    const bool circular = flags & PG_SEQHASH_CIRCULAR, ds = flags & PG_SEQHASH_DOUBLE_STRANDED;
    const int mode = seq_type == PG_SEQHASH_RNA ? FOLD_RNA : FOLD_UPPER;
    static const Alphabet nucleic = make_alphabet("ATUGCYRSWKMBDHVNZ"), protein = make_alphabet("ACDEFGHIKLMNPQRSTVWYUO*BXZ");
    const bool one_chunk = max_len <= CHUNK;
    const uint64_t n_slots = one_chunk ? n : total / CHUNK + n;
    StreamScratch sc(st);
    uint8_t *canon = nullptr, *rc = nullptr;
    uint64_t *start = nullptr;
    unsigned long long *first_bad = nullptr;
    uint32_t *cv = nullptr;
    auto fail = [](uint64_t bytes) {
        cudaGetLastError();
        set_error("seqhash scratch of %llu bytes does not fit in device memory", (unsigned long long)bytes);
        return PG_ERR_NOMEM;
    };
    if (sc.alloc(&canon, total + 64) != cudaSuccess) return fail(total + 64);  // slack for the chunk kernel's word loads
    if (sc.alloc(&cv, 8 * n_slots) != cudaSuccess) return fail(32 * n_slots);
    if (sc.alloc(&first_bad, n) != cudaSuccess) return fail(8 * n);
    PG_CUDA(cudaMemsetAsync(first_bad, 0xff, n * 8, st));
    if (circular || ds) {
        if (sc.alloc(&start, n) != cudaSuccess || sc.alloc(&rc, n) != cudaSuccess) return fail(9 * n);
        if (circular) {
            const int rc_ = launch_rotate(d_in, d_off, n, max_len, mode, ds, start, rc, st);
            if (rc_ != PG_OK) return rc_;
        } else {
            seqhash_strand_kernel<<<flat_grid(n * 32, 256), 256, 0, st>>>(d_in, d_off, n, mode, start, rc);
            PG_LAUNCH_CHECK("seqhash_strand_kernel");
        }
    }
    if (total) {
        seqhash_canon_kernel<<<flat_grid((total + 15) / 16, 256), 256, 0, st>>>(d_in, d_off, n, total, mode,
                                                                                seq_type == PG_SEQHASH_PROTEIN ? protein : nucleic,
                                                                                start, rc, canon, first_bad);
        PG_LAUNCH_CHECK("seqhash_canon_kernel");
    }
    if (one_chunk) {
        blake3_chunk_kernel<true><<<flat_grid(n_slots, 128), 128, 0, st>>>(canon, d_off, n, n_slots, cv);
        PG_LAUNCH_CHECK("blake3_chunk_kernel<1>");
    } else {
        blake3_chunk_kernel<false><<<flat_grid(n_slots, 128), 128, 0, st>>>(canon, d_off, n, n_slots, cv);
        PG_LAUNCH_CHECK("blake3_chunk_kernel<0>");
        blake3_tree_kernel<<<(unsigned)std::min<uint64_t>(n, 0x7fffffffull), 256, 0, st>>>(d_off, n, cv);
        PG_LAUNCH_CHECK("blake3_tree_kernel");
    }
    const int protein_ds = seq_type == PG_SEQHASH_PROTEIN && ds;
    if (one_chunk) seqhash_finish_kernel<true><<<flat_grid(n, 256), 256, 0, st>>>(d_in, d_off, n, protein_ds, first_bad, cv, d_digest, d_err, d_pos);
    else seqhash_finish_kernel<false><<<flat_grid(n, 256), 256, 0, st>>>(d_in, d_off, n, protein_ds, first_bad, cv, d_digest, d_err, d_pos);
    PG_LAUNCH_CHECK("seqhash_finish_kernel");
    return PG_OK;
}

}  // namespace pg
