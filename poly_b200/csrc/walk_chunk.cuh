// walk_chunk.cuh -- the byte-chunked window walk over a ragged set of records that the screen's add
// (mash_screen.cu) and the grouped sketch (sketch_groups.cu) share: a CTA stages a fixed chunk of the records'
// bytes in shared memory, whatever the record lengths, and each thread walks consecutive windows of it with the
// register ring of kmer_walk.cuh; window_in_read then tells a window that ends inside its record from one that
// crosses a record end.  Each kernel brings its own EMIT.
//
// Canonical mode (PG_KMER_CANONICAL, CANON = true): a record of length L has the windows 0 .. L - k (Mash's k-mer set,
// one more than the forward mode's 0 .. L - k - 1), and each window hashes the smaller of itself and its reverse
// complement in byte order.  The walk then also stages a complemented copy of its chunk (stage_chunk<.., true>) and
// runs the reverse strand's ring of kmer_walk.cuh beside the forward one.
#pragma once
#include <stdint.h>

#include "common.cuh"
#include "murmur3.cuh"

namespace pg {

// Whether the window at byte p is one of its read's: p + k < the end of the read that holds p, the first offset
// above p (p + k <= that end in canonical mode).  j caches the index of that offset (~0 = not searched yet); a
// thread's windows only move forward.
template <bool CANON = false>
__device__ __forceinline__ bool window_in_read(const uint64_t *off, uint64_t n_reads, uint64_t p, uint32_t k, uint64_t &j) {
    if (j == ~0ull) {
        uint64_t lo = 0, hi = n_reads + 1;
        while (lo < hi) {
            const uint64_t mid = (lo + hi) >> 1;
            if (off[mid] > p) hi = mid;
            else lo = mid + 1;
        }
        j = lo;
    }
    while (j <= n_reads && off[j] <= p) ++j;
    return j <= n_reads && (CANON ? p + k <= off[j] : p + k < off[j]);
}

// Whether a window of k bytes that starts `room` bytes before the end of its span can be one of its read's.
template <bool CANON>
__device__ __forceinline__ bool window_fits(uint64_t room, uint32_t k) { return CANON ? room >= k : room > k; }

// The hash of the k-byte window at w, read from global memory: murmur3 over its raw bytes, or in canonical mode over
// the smaller of w and rc(w) (rc(w)[x] = complement(w[k - 1 - x])), compared byte by byte as memcmp does.
template <bool CANON>
__device__ __forceinline__ uint32_t window_hash(const uint8_t *w, uint32_t k) {
    bool rc = false;
    if constexpr (CANON)
        for (uint32_t x = 0; x < k; ++x) {
            const uint8_t a = __ldg(w + x), b = complement(__ldg(w + k - 1 - x));
            if (a != b) {
                rc = b < a;
                break;
            }
        }
    if (rc) return mm3_bytes([w, k](uint32_t x) { return complement(__ldg(w + k - 1 - x)); }, k);
    return mm3_bytes([w](uint32_t x) { return __ldg(w + x); }, k);
}

// the 16-byte alignment head of a chunk that starts at byte P0: chunk byte 0 is staged at s_in[head]
__device__ __forceinline__ uint32_t chunk_head(const uint8_t *bases, uint64_t P0) { return (uint32_t)((uintptr_t)(bases + P0) & 15u); }

// Stages the STAGE bytes of a chunk that starts at byte P0, after its alignment head, into s_in with 16-byte
// loads, by the NT threads of the CTA; bytes outside [lo, hi) are zeros and are never read from global memory.
// With RC, s_rc[x] = s_comp[s_in[x]] as well: the complemented copy (s_comp: complement() of every byte).
// The caller puts a CTA barrier before (the previous chunk's walk is done with s_in) and after (the stage is
// complete).
template <uint32_t STAGE, uint32_t NT, bool RC = false>
__device__ __forceinline__ void stage_chunk(uint8_t *s_in, const uint8_t *bases, uint64_t P0, uint32_t head, uint64_t lo, uint64_t hi,
                                            uint8_t *s_rc = nullptr, const uint8_t *s_comp = nullptr) {
    const int64_t q_base = (int64_t)P0 - (int64_t)head;  // position of staged byte 0
    const uint8_t *g = bases + P0 - head;
    for (uint32_t x = threadIdx.x; x < STAGE / 16; x += NT) {
        const int64_t q = q_base + 16 * (int64_t)x;
        uint4 v;
        if (q >= (int64_t)lo && q + 16 <= (int64_t)hi) {
            v = __ldg(reinterpret_cast<const uint4 *>(g) + x);
        } else {
            uint8_t b[16];
#pragma unroll
            for (int t = 0; t < 16; ++t) b[t] = (q + t >= (int64_t)lo && q + t < (int64_t)hi) ? __ldg(g + 16 * x + t) : (uint8_t)0;
            v = make_uint4(b[0] | b[1] << 8 | b[2] << 16 | (uint32_t)b[3] << 24, b[4] | b[5] << 8 | b[6] << 16 | (uint32_t)b[7] << 24,
                           b[8] | b[9] << 8 | b[10] << 16 | (uint32_t)b[11] << 24, b[12] | b[13] << 8 | b[14] << 16 | (uint32_t)b[15] << 24);
        }
        reinterpret_cast<uint4 *>(s_in)[x] = v;
        if constexpr (RC) {
            uint32_t c[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int t = 0; t < 4; ++t)
                c[t] = (uint32_t)s_comp[c[t] & 0xff] | (uint32_t)s_comp[c[t] >> 8 & 0xff] << 8 | (uint32_t)s_comp[c[t] >> 16 & 0xff] << 16 |
                       (uint32_t)s_comp[c[t] >> 24] << 24;
            reinterpret_cast<uint4 *>(s_rc)[x] = make_uint4(c[0], c[1], c[2], c[3]);
        }
    }
}

// windows per thread of a walk kernel: whole groups of NB word steps, about 64
__host__ __device__ constexpr uint32_t walk_span(int nb) { return 4u * nb * (16 / nb > 0 ? 16 / nb : 1); }

}  // namespace pg
