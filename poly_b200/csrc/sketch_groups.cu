// sketch_groups.cu -- one bottom-s sketch per group of records (a draft assembly's contigs, a sample's reads), with
// Mash's minimum-copies filter: row g is the smallest s distinct window hashes v of group g's records whose count
// c_g(v) is at least m, ascending.
//
// Passes over disjoint hash ranges.  Pass t admits the windows of group g whose hash lies in [lo_g, lo_g + w_g) and
// counts every one of them into g's open-addressing table, so after the pass c_g(v) is final for each v of the range.
// The table entries with count >= m are sorted (one radix sort of (slot << 32 | v) keys) and appended to the row:
// ranges only move up, so the row stays ascending.  A group is done when its row holds s values or its range has
// reached 2^32.  The first range is K2t's admission rule, mu = s + 6 sqrt(s) + 48 windows on average; the next one
// is scaled from the qualifying values found per unit of range so far, at most 64 times the last width, and its
// table from the distinct values seen per unit of range.  A table that fills past half of its slots drops its pass,
// and the group retries with half the width and twice the table; its row and its earlier ranges are untouched.
// Later passes walk only the byte spans of the groups they admit.
//
// The walk (k in WalkKs) is the screen's: persistent CTAs take fixed byte chunks of the spans, stage them in
// shared memory (walk_chunk.cuh) and each thread walks W consecutive windows with the register ring of
// kmer_walk.cuh.  One thread per CTA finds the chunk's first and last group while the chunk is staged.  A thread whose
// W windows lie in one group keeps that group's range in registers; a thread whose windows cross a group end (rare)
// admits every window and sorts them out with a forward cursor over the group byte offsets.  Per window: one range
// compare and a warp vote, as in the screen; the rare admitted windows then take window_in_read and one table add per
// distinct (group, value) of the warp.
//
// Canonical mode (PG_KMER_CANONICAL) is the template parameter CANON of the walk, generic and window-count kernels:
// windows 0 .. L - k of each record, each hashing the smaller of itself and its reverse complement (walk_chunk.cuh,
// kmer_walk.cuh).  Everything after the walk is the same.
#include <algorithm>
#include <cmath>
#include <vector>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <thrust/iterator/transform_iterator.h>

#include "common.cuh"
#include "kmer_walk.cuh"
#include "murmur3.cuh"
#include "walk_chunk.cuh"

namespace pg {

namespace {

constexpr int GS_THREADS = 256;
constexpr unsigned long long GS_EMPTY = ~0ull;
// table slots of one pass (16 bytes each, plus 16 of sorted output): 1 GiB of tables at most
constexpr uint64_t GS_PASS_SLOTS = 1ull << 26;
constexpr uint64_t GS_MAX_TABLE = 1ull << 25;
constexpr uint64_t GS_RANGE = 1ull << 32;

// a group's place in a pass: its range [lo, lo + width) (width 0: not in this pass) and its table
struct GroupPass {
    uint64_t width;
    uint64_t tab;   // first slot
    uint32_t lo;
    uint32_t mask;  // slots - 1
    uint32_t slot;  // its index among the pass's groups
    uint32_t pad;
};

// one byte span of the pass: records [.., ..) of consecutive admitted groups, bytes [beg, end); chunk0: its first chunk
struct Span {
    uint64_t beg, end, chunk0;
};

struct PassArgs {
    const uint64_t *off;     // [n_records + 1] record offsets
    uint64_t n_records;
    const uint64_t *gbyte;   // [n_groups + 1] byte offset of each group's first record
    uint64_t n_groups;
    const GroupPass *gp;     // [n_groups]
    const Span *spans;
    uint32_t n_spans;
    unsigned long long *keys, *cnt;  // table slots
    unsigned int *claims, *ovf;     // per pass slot
};

// the span of chunk c: the last span whose chunk0 <= c
__device__ __forceinline__ uint32_t span_of(const Span *sp, uint32_t n, uint64_t c) {
    uint32_t lo = 0, hi = n;
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (sp[mid].chunk0 <= c) lo = mid;
        else hi = mid;
    }
    return lo;
}

// the group that holds byte p of the records: the last g with gbyte[g] <= p (empty groups share their byte offset with
// the next group, which is the one found)
__device__ __forceinline__ uint64_t group_of(const uint64_t *gbyte, uint64_t G, uint64_t p) {
    uint64_t lo = 0, hi = G;
    while (hi - lo > 1) {
        const uint64_t mid = (lo + hi) >> 1;
        if (gbyte[mid] <= p) lo = mid;
        else hi = mid;
    }
    return lo;
}

// Adds n windows of hash h to the table of group g's pass.  The claim that takes the table past half of its slots marks
// the group's pass as overflowed, and an overflowed pass stops adding: the host drops it.
__device__ __forceinline__ void table_add(const PassArgs &A, const GroupPass &g, uint32_t h, unsigned n) {
    if (*(volatile unsigned int *)&A.ovf[g.slot]) return;
    uint32_t i = h & g.mask;
    for (uint32_t probe = 0; probe <= g.mask; ++probe, i = (i + 1) & g.mask) {
        unsigned long long *key = A.keys + g.tab + i;
        unsigned long long cur = *(volatile unsigned long long *)key;
        if (cur == GS_EMPTY) {
            cur = atomicCAS(key, GS_EMPTY, (unsigned long long)h);
            if (cur == GS_EMPTY) {
                if (atomicAdd(&A.claims[g.slot], 1u) + 1 > (g.mask + 1) / 2) atomicExch(&A.ovf[g.slot], 1u);
                cur = h;
            }
        }
        if (cur == h) {
            atomicAdd(&A.cnt[g.tab + i], (unsigned long long)n);
            return;
        }
    }
    atomicExch(&A.ovf[g.slot], 1u);  // full: only reached once the claims have marked it already
}

// One window of every lane of a converged warp; cand: the lane's hash passed its admission compare.  For a thread whose
// windows all lie in group g that compare was exact; a mixed thread (its windows cross a group end or the span end)
// admits every window, and here finds the group of window p with its forward cursor g and applies that group's range.
// Lanes with the same (group, hash) add once, with their number.
template <bool CANON>
__device__ __forceinline__ void group_hit(const PassArgs &A, bool cand, bool mixed, uint64_t &g, uint64_t send, uint64_t p, uint32_t k, uint32_t h,
                                          uint64_t &j) {
    if (cand && mixed) {
        if (p >= send) {
            cand = false;
        } else {
            while (A.gbyte[g + 1] <= p) ++g;
            cand = (uint64_t)(h - A.gp[g].lo) < A.gp[g].width;
        }
    }
    const bool hit = cand && window_in_read<CANON>(A.off, A.n_records, p, k, j);
    const unsigned long long key = hit ? (g << 32 | h) : ~0ull;
    const unsigned peers = __match_any_sync(0xffffffffu, key);
    if (hit && (int)(threadIdx.x & 31) == __ffs(peers) - 1) table_add(A, A.gp[g], h, (unsigned)__popc(peers));
}

// EMIT of the walk: window p0 + i + R_, admitted when (h - lo) <= wm1, a compare as cheap as the screen's.
#define PG_GROUPS_EMIT(R_, H_)                                                                                              \
    {                                                                                                                       \
        const bool cand_ = (uint32_t)((H_) - lo) <= wm1;                                                                    \
        if (__any_sync(0xffffffffu, cand_)) group_hit<CANON>(A, cand_, mixed, g, send, p0 + i + (R_), (uint32_t)K, (H_), j);\
    }

template <int K, bool CANON>
__global__ void __launch_bounds__(GS_THREADS, 2) groups_walk_kernel(const uint8_t *__restrict__ bases, const PassArgs A, uint64_t chunks,
                                                                    uint32_t lut_stride) {
    PG_WALK_CONSTANTS;
    constexpr uint32_t W = walk_span(NB);
    constexpr uint32_t CHUNK = GS_THREADS * W;
    constexpr uint32_t STAGE = CHUNK + 128;  // + head (< 16) + the walk's look-ahead (< 4 NB + 20 bytes)
    constexpr uint32_t nk = W;
    // CANON: the complemented copy s_rc and the complement table s_comp follow the chunk
    __shared__ __align__(16) uint8_t s_in[CANON ? 2 * STAGE + 256 : STAGE];
    __shared__ __align__(16) uint32_t s_lut[LUT ? 256 : 4];
    __shared__ uint64_t s_g[2];  // the groups of the chunk's first and last window
    uint8_t *s_rc = nullptr, *s_comp = nullptr;
    const uint32_t tid = threadIdx.x;
    if (LUT)
        for (uint32_t x = tid; x < 256; x += GS_THREADS) s_lut[x] = g_kmix_byte.v[x];
    if constexpr (CANON) {
        s_rc = s_in + STAGE;
        s_comp = s_in + 2 * STAGE;
        for (uint32_t x = tid; x < 256; x += GS_THREADS) s_comp[x] = complement((uint8_t)x);
    }
    const uint32_t lut_base = smem_u32(s_lut);

    for (uint64_t c = blockIdx.x; c < chunks; c += gridDim.x) {
        const Span sp = A.spans[span_of(A.spans, A.n_spans, c)];
        const uint64_t P0 = sp.beg + (c - sp.chunk0) * CHUNK, send = sp.end;
        const uint32_t head = chunk_head(bases, P0);
        __syncthreads();  // the previous chunk's walk is done with s_in and s_g (and, the first time, s_lut is written)
        if (tid == 0) {  // while the other threads stage: one search for the chunk, not one per thread
            s_g[0] = group_of(A.gbyte, A.n_groups, P0);
            s_g[1] = group_of(A.gbyte, A.n_groups, min(P0 + CHUNK, send) - 1);
        }
        if constexpr (CANON) stage_chunk<STAGE, GS_THREADS, true>(s_in, bases, P0, head, sp.beg, sp.end, s_rc, s_comp);
        else stage_chunk<STAGE, GS_THREADS>(s_in, bases, P0, head, sp.beg, sp.end);
        __syncthreads();

        const uint32_t b0 = head + tid * W;
        const uint32_t *sw = reinterpret_cast<const uint32_t *>(s_in) + (b0 >> 2);
        const uint32_t sh = (b0 & 3u) * 8u;
        const uint8_t *sb = s_in + b0 + 4 * NB;
        const uint64_t p0 = P0 + tid * W;
        uint64_t j = ~0ull, g = 0;
        uint32_t lo = 1, wm1 = 0;  // past the span: admit only h == 1, which group_hit rejects there
        bool mixed = true;
        if (p0 < send) {  // the last group in [s_g[0], s_g[1]] that starts at or before p0
            g = s_g[0];
            for (uint64_t hi = s_g[1] + 1; hi - g > 1;) {
                const uint64_t mid = (g + hi) >> 1;
                if (A.gbyte[mid] <= p0) g = mid;
                else hi = mid;
            }
            mixed = p0 + W > min(A.gbyte[g + 1], send);
            lo = mixed ? 0u : A.gp[g].lo;
            wm1 = mixed ? 0xFFFFFFFFu : (uint32_t)(A.gp[g].width - 1);  // a group of the pass has width >= 1
        }

        if constexpr (CANON) {
            const uint8_t *sbf = s_in + b0, *sbc = s_rc + b0;
            const uint32_t *cw = reinterpret_cast<const uint32_t *>(s_rc) + ((b0 + TAIL) >> 2);
            const uint32_t csh = ((b0 + TAIL) & 3u) * 8u;
            PG_WALK_PROLOGUE
            PG_CANON_PROLOGUE
            uint32_t i = 0;
            while (i < W) {
#pragma unroll
                for (int u = 0; u < NB; ++u) PG_KMER_STEP_CANON(u, PG_GROUPS_EMIT)
            }
        } else {
            PG_WALK_PROLOGUE
            uint32_t i = 0;
            while (i < W) {
#pragma unroll
                for (int u = 0; u < NB; ++u) PG_KMER_STEP(u, false, PG_GROUPS_EMIT)
            }
        }
    }
}

// Any other k (0 included, but not in canonical mode): one window per thread from global memory, over chunks of
// GS_THREADS bytes of the spans.
template <bool CANON>
__global__ void __launch_bounds__(GS_THREADS) groups_generic_kernel(const uint8_t *__restrict__ bases, const PassArgs A, uint64_t chunks, uint32_t k) {
    for (uint64_t c = blockIdx.x; c < chunks; c += gridDim.x) {
        const Span sp = A.spans[span_of(A.spans, A.n_spans, c)];
        const uint64_t p = sp.beg + (c - sp.chunk0) * GS_THREADS + threadIdx.x;
        uint32_t h = 0;
        bool cand = false;
        uint64_t g = 0;
        if (p < sp.end && window_fits<CANON>(sp.end - p, k)) {
            h = window_hash<CANON>(bases + p, k);
            g = group_of(A.gbyte, A.n_groups, p);
            cand = (uint64_t)(h - A.gp[g].lo) < A.gp[g].width;
        }
        if (__any_sync(0xffffffffu, cand)) {
            uint64_t j = ~0ull;
            group_hit<CANON>(A, cand, false, g, sp.end, p, k, h, j);
        }
    }
}

// windows of each record, max(len - k, 0) (canonical: max(len - k + 1, 0))
template <bool CANON>
__global__ void groups_windows_kernel(const uint64_t *__restrict__ off, uint64_t n, uint32_t k, uint64_t *__restrict__ win) {
    for (uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t len = off[r + 1] - off[r];
        win[r] = CANON ? (len >= k ? len - k + 1 : 0) : (len > k ? len - k : 0);
    }
}

// per group: its windows (from the exclusive prefix pre[] of the records' windows) and its first byte
__global__ void groups_sizes_kernel(const uint64_t *__restrict__ goff, uint64_t G, const uint64_t *__restrict__ pre, const uint64_t *__restrict__ off,
                                    uint64_t *__restrict__ wg, uint64_t *__restrict__ gbyte) {
    for (uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; g <= G; g += (uint64_t)gridDim.x * blockDim.x) {
        gbyte[g] = off[goff[g]];
        if (g < G) wg[g] = pre[goff[g + 1]] - pre[goff[g]];
    }
}

// every table entry with count >= m, as (pass slot << 32 | value), and the number per pass slot
__global__ void groups_collect_kernel(const unsigned long long *__restrict__ keys, const unsigned long long *__restrict__ cnt,
                                      const uint32_t *__restrict__ slot_of, uint64_t slots, uint32_t m, unsigned long long *__restrict__ out,
                                      unsigned long long *__restrict__ n_out, unsigned int *__restrict__ qual) {
    for (uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; e < slots; e += (uint64_t)gridDim.x * blockDim.x) {
        if (keys[e] != GS_EMPTY && cnt[e] >= m) {
            const uint32_t a = slot_of[e >> 6];  // tables are whole multiples of 64 slots
            out[atomicAdd(n_out, 1ull)] = (unsigned long long)a << 32 | keys[e];
            atomicAdd(&qual[a], 1u);
        }
    }
}

// what a pass appends for pass slot a: its group's row, where it starts in the sorted keys, how many and where in the row
struct Append {
    uint64_t row, first;
    uint32_t take, base;
};

__global__ void groups_append_kernel(const unsigned long long *__restrict__ sorted, uint64_t n, const Append *__restrict__ ap, uint32_t *__restrict__ out,
                                     uint64_t row_stride) {
    for (uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (uint64_t)gridDim.x * blockDim.x) {
        const unsigned long long key = sorted[e];
        const Append a = ap[key >> 32];
        const uint64_t r = e - a.first;
        if (r < a.take) out[a.row * row_stride + a.base + r] = (uint32_t)key;
    }
}

// ---- the grown grouped sketch (pg_mash_sketcher): an add is a run of passes over the batch with three changes.
// Each group's ranges stop at its cap; each table is seeded with the group's state entries of the range; and a pass
// appends every entry up to the group's cut (the s-th qualifying value or the B-th value), with its saturated count,
// to the add's list, which becomes the group's new state.

// The state entries [seg[0], seg[nb]) of the batch's groups whose value lies in their group's range of the pass, into
// its table with their saturated counts: a seeded value is a claim like any other, so the overflow rule covers it.
__global__ void sketcher_seed_kernel(const uint32_t *__restrict__ val, const uint32_t *__restrict__ cnt, const uint64_t *__restrict__ seg, uint64_t nb,
                                     const PassArgs A) {
    const uint64_t e0 = seg[0], n = seg[nb] - e0;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t e = e0 + i;
        const GroupPass g = A.gp[group_of(seg, nb, e)];
        const uint32_t v = val[e];
        if ((uint64_t)(v - g.lo) < g.width) table_add(A, g, v, cnt[e]);
    }
}

// every table entry as (pass slot << 32 | value) with its count saturated at m, and the entries per pass slot
__global__ void sketcher_collect_kernel(const unsigned long long *__restrict__ keys, const unsigned long long *__restrict__ cnt,
                                        const uint32_t *__restrict__ slot_of, uint64_t slots, uint32_t m, unsigned long long *__restrict__ out,
                                        uint32_t *__restrict__ out_cnt, unsigned long long *__restrict__ n_out, unsigned int *__restrict__ per_slot) {
    for (uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; e < slots; e += (uint64_t)gridDim.x * blockDim.x) {
        if (keys[e] != GS_EMPTY) {
            const uint32_t a = slot_of[e >> 6];
            const unsigned long long o = atomicAdd(n_out, 1ull);
            out[o] = (unsigned long long)a << 32 | keys[e];
            out_cnt[o] = (uint32_t)min(cnt[e], (unsigned long long)m);
            atomicAdd(&per_slot[a], 1u);
        }
    }
}

struct QualFlag {
    uint32_t m;
    __host__ __device__ uint32_t operator()(uint32_t c) const { return c >= m ? 1u : 0u; }
};

// a pass slot's place in the cut: its entries [first, first + n) of the sorted list, what earlier passes of this add
// kept for its group (held values, qual of them qualifying), and its positions [out, out + room) of the add's list,
// room = min(n, B - held).  live == 0: the pass overflowed for this slot and is dropped.
struct Cut {
    uint64_t first, n, held, out, room;
    uint32_t qual, group, live, pad;
};

// what the cut found for a pass slot: the values it kept, the qualifying ones among them, and the caps the s-th
// qualifying value (its value + 1) and the (B + 1)-th value give, 2^32 where not found
struct CutOut {
    unsigned long long cap_s, cap_b;
    uint32_t kept, qkept;
};

// Entry e of slot a is the (held + r)-th value of its group in this add (r: its rank in the slot) and has qb qualifying
// values before it.  It is kept while held + r < B and qb < s; kept entries go to the add's list as
// (batch group << 32 | value), the rest of the slot's room gets the sentinel nb << 32, which sorts after every group.
__global__ void sketcher_cut_kernel(const unsigned long long *__restrict__ sorted, const uint32_t *__restrict__ scnt, const uint32_t *__restrict__ qscan,
                                    uint64_t n, const Cut *__restrict__ cut, uint32_t m, uint32_t s, uint64_t B, unsigned long long sentinel,
                                    unsigned long long *__restrict__ akey, uint32_t *__restrict__ acnt, CutOut *__restrict__ res) {
    for (uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (uint64_t)gridDim.x * blockDim.x) {
        const unsigned long long key = sorted[e];
        const uint32_t a = (uint32_t)(key >> 32);
        const Cut c = cut[a];
        if (!c.live) continue;
        const uint32_t v = (uint32_t)key;
        const uint64_t r = e - c.first, i = c.held + r;
        const uint64_t qb = c.qual + (qscan[e] - qscan[c.first]);
        const uint32_t q = scnt[e] >= m ? 1u : 0u;
        const bool keep = i < B && qb < s;
        if (i == B) res[a].cap_b = v;
        if (keep && q && qb + 1 == s) res[a].cap_s = (unsigned long long)v + 1;
        if (keep && !(r + 1 < c.n && i + 1 < B && qb + q < s)) {  // the slot's last kept entry
            res[a].kept = (uint32_t)(r + 1);
            res[a].qkept = (uint32_t)(qb + q - c.qual);
        }
        if (r < c.room) {
            akey[c.out + r] = keep ? ((unsigned long long)c.group << 32 | v) : sentinel;
            acnt[c.out + r] = scnt[e];
        }
    }
}

constexpr uint64_t SK_FROM_ADD = 1ull << 63;

// The new state of the batch's groups, segment g = [nseg[g], nseg[g + 1]): from the add's sorted list at from[g] when
// the add walked g (SK_FROM_ADD set), else the old state's segment, which starts at from[g].
__global__ void sketcher_merge_kernel(const uint64_t *__restrict__ nseg, uint64_t nb, const uint64_t *__restrict__ from,
                                      const unsigned long long *__restrict__ akey, const uint32_t *__restrict__ acnt, const uint32_t *__restrict__ oval,
                                      const uint32_t *__restrict__ ocnt, uint32_t *__restrict__ val, uint32_t *__restrict__ cnt) {
    const uint64_t n = nseg[nb];
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t g = group_of(nseg, nb, i), f = from[g], j = (f & ~SK_FROM_ADD) + (i - nseg[g]);
        val[i] = (f & SK_FROM_ADD) ? (uint32_t)akey[j] : oval[j];
        cnt[i] = (f & SK_FROM_ADD) ? acnt[j] : ocnt[j];
    }
}

// One warp per group of [first, first + count): the first s values of its state segment with count >= m (a segment
// holds at most s of them), zeros to row_stride, their number, complete and held.
__global__ void sketcher_rows_kernel(const uint32_t *__restrict__ val, const uint32_t *__restrict__ cnt, const uint64_t *__restrict__ seg,
                                     const uint64_t *__restrict__ cap, uint64_t first, uint64_t count, uint32_t s, uint32_t m, uint32_t *__restrict__ out,
                                     uint64_t row_stride, uint32_t *__restrict__ n_out, uint8_t *__restrict__ complete, uint64_t *__restrict__ held) {
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t warps = (uint64_t)gridDim.x * (blockDim.x >> 5);
    for (uint64_t w = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < count; w += warps) {
        const uint64_t g = first + w, b = seg[g], e = seg[g + 1];
        uint32_t *row = out + w * row_stride;
        uint32_t taken = 0;
        for (uint64_t p = b; p < e && taken < s; p += 32) {
            const uint64_t x = p + lane;
            const bool ok = x < e && cnt[x] >= m;
            const unsigned bal = __ballot_sync(0xffffffffu, ok);
            const uint32_t pos = taken + __popc(bal & ((1u << lane) - 1u));
            if (ok && pos < s) row[pos] = val[x];
            taken = min(s, taken + (uint32_t)__popc(bal));
        }
        for (uint64_t j = taken + lane; j < row_stride; j += 32) row[j] = 0;
        if (lane == 0) {
            n_out[w] = taken;
            if (complete) complete[w] = taken == s || cap[g] == GS_RANGE;
            if (held) held[w] = e - b;
        }
    }
}

unsigned grid_for(uint64_t work) { return (unsigned)std::max<uint64_t>(1, std::min<uint64_t>((work + 255) / 256, (uint64_t)sm_count() * 16)); }

uint64_t pow2_at_least(uint64_t x) {
    uint64_t p = 64;
    while (p < x) p <<= 1;
    return p;
}

double admit_target(double need) { return need + 6.0 * std::sqrt(need) + 48.0; }

// the host's view of one group across passes
struct GroupState {
    uint64_t windows = 0;
    uint64_t covered = 0;   // the range [0, covered) is final
    uint64_t width = 0;     // the next pass's width
    uint64_t slots = 0;     // the next pass's table
    uint64_t distinct = 0;  // distinct values seen in [0, covered)
    uint64_t qualified = 0; // values with count >= m in [0, covered)
    uint32_t rows = 0;
    bool done = false;
};

// the table for a width: twice the expected distinct values plus six deviations, from the distinct values seen per
// unit of range (or, before any, the windows per unit of range, which bounds them)
uint64_t table_for(const GroupState &st, uint64_t width) {
    const double per = st.covered ? (double)std::max<uint64_t>(st.distinct, 1) / (double)st.covered : (double)st.windows / (double)GS_RANGE;
    const double est = std::min((double)st.windows, per * (double)width);
    return std::min(GS_MAX_TABLE, pow2_at_least((uint64_t)(2.0 * (est + 6.0 * std::sqrt(est) + 16.0))));
}

int gs_nomem(cudaError_t e) {
    set_error("cudaMallocAsync for the grouped sketch failed: %s", cudaGetErrorString(e));
    cudaGetLastError();
    return PG_ERR_NOMEM;
}

// per group of a batch: its windows wg[g] and the byte offset of its first record gbyte[g] (G + 1 of them), on the
// host and in *d_gbyte (from tmp)
int group_sizes(const uint64_t *d_off, uint64_t n_records, const uint64_t *d_goff, uint64_t G, int k, bool canon, StreamScratch &tmp, std::vector<uint64_t> &wg,
                std::vector<uint64_t> &gbyte, uint64_t **d_gbyte, cudaStream_t st) {
    cudaError_t e;
    uint64_t *d_win = nullptr, *d_pre = nullptr, *d_wg = nullptr;
    if ((e = tmp.alloc(&d_win, n_records + 1)) != cudaSuccess || (e = tmp.alloc(&d_pre, n_records + 1)) != cudaSuccess ||
        (e = tmp.alloc(&d_wg, G)) != cudaSuccess || (e = tmp.alloc(d_gbyte, G + 1)) != cudaSuccess)
        return gs_nomem(e);
    PG_CUDA(cudaMemsetAsync(d_win + n_records, 0, 8, st));
    if (canon) groups_windows_kernel<true><<<grid_for(n_records), 256, 0, st>>>(d_off, n_records, (uint32_t)k, d_win);
    else groups_windows_kernel<false><<<grid_for(n_records), 256, 0, st>>>(d_off, n_records, (uint32_t)k, d_win);
    PG_LAUNCH_CHECK("groups_windows_kernel");
    {
        size_t bytes = 0;
        uint8_t *d_cub = nullptr;
        PG_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, bytes, d_win, d_pre, n_records + 1, st));
        if ((e = tmp.alloc(&d_cub, bytes)) != cudaSuccess) return gs_nomem(e);
        PG_CUDA(cub::DeviceScan::ExclusiveSum(d_cub, bytes, d_win, d_pre, n_records + 1, st));
    }
    groups_sizes_kernel<<<grid_for(G + 1), 256, 0, st>>>(d_goff, G, d_pre, d_off, d_wg, *d_gbyte);
    PG_LAUNCH_CHECK("groups_sizes_kernel");
    wg.resize(G);
    gbyte.resize(G + 1);
    PG_CUDA(cudaMemcpyAsync(wg.data(), d_wg, G * 8, cudaMemcpyDeviceToHost, st));
    PG_CUDA(cudaMemcpyAsync(gbyte.data(), *d_gbyte, (G + 1) * 8, cudaMemcpyDeviceToHost, st));
    PG_CUDA(cudaStreamSynchronize(st));
    return PG_OK;
}

// The next pass's groups into act, by pass slot (ascending): open groups in order, from where the last pass stopped so
// that none waits forever, while their tables fit.  Returns the pass's table slots.
uint64_t pick_pass(const std::vector<GroupState> &gs, uint64_t &next, std::vector<uint64_t> &act) {
    const uint64_t G = gs.size();
    act.clear();
    uint64_t slots = 0;
    for (uint64_t t = 0; t < G && act.size() < (1u << 24); ++t) {
        const uint64_t g = (next + t) % G;
        if (gs[g].done) continue;
        if (!act.empty() && slots + gs[g].slots > GS_PASS_SLOTS) break;
        act.push_back(g);
        slots += gs[g].slots;
    }
    if (act.empty()) return 0;
    next = (act.back() + 1) % G;
    std::sort(act.begin(), act.end());
    return slots;
}

// A pass over the groups act: their ranges [covered, covered + width) and tables in gp, the pass slot of every 64
// table slots, and the byte spans of their records.  Returns the walk's chunks.
uint64_t lay_out_pass(const std::vector<uint64_t> &act, const std::vector<GroupState> &gs, const std::vector<uint64_t> &gbyte, uint64_t slots,
                      uint64_t chunk_bytes, std::vector<GroupPass> &gp, std::vector<uint32_t> &slot_of, std::vector<Span> &spans) {
    for (GroupPass &x : gp) x = GroupPass{0, 0, 0, 0, 0, 0};
    slot_of.assign(slots / 64, 0);
    spans.clear();
    uint64_t tab = 0;
    uint64_t chunks = 0;
    for (uint32_t a = 0; a < act.size(); ++a) {
        const uint64_t g = act[a];
        const GroupState &x = gs[g];
        gp[g] = GroupPass{x.width, tab, (uint32_t)x.covered, (uint32_t)(x.slots - 1), a, 0};
        for (uint64_t q = tab / 64; q < (tab + x.slots) / 64; ++q) slot_of[q] = a;
        tab += x.slots;
        if (gbyte[g + 1] == gbyte[g]) continue;
        if (!spans.empty() && spans.back().end == gbyte[g]) {
            spans.back().end = gbyte[g + 1];
        } else {
            if (!spans.empty()) chunks += (spans.back().end - spans.back().beg + chunk_bytes - 1) / chunk_bytes;
            spans.push_back(Span{gbyte[g], gbyte[g + 1], chunks});
        }
    }
    if (!spans.empty()) chunks += (spans.back().end - spans.back().beg + chunk_bytes - 1) / chunk_bytes;
    return chunks;
}

// bytes per chunk of the walk for k
uint64_t walk_chunk_bytes(int k) {
    int walk_k = 0;
    const bool walk = with_walk_k(k, [&](auto kk) { walk_k = decltype(kk)::value; });
    return walk ? (uint64_t)GS_THREADS * walk_span(walk_k / 4) : (uint64_t)GS_THREADS;
}

// a pass's walk over its spans: groups_walk_kernel<k> for k in WalkKs, groups_generic_kernel for any other k
template <bool CANON>
int launch_walk_mode(const uint8_t *d_bases, const PassArgs &args, uint64_t chunks, int k, cudaStream_t st) {
    uint64_t grid = 0;
    int rc = PG_OK;
    const bool walk = with_walk_k(k, [&](auto kk) {
        constexpr int K = decltype(kk)::value;
        if ((rc = resident_blocks((const void *)groups_walk_kernel<K, CANON>, GS_THREADS, 0, chunks, &grid)) != PG_OK) return;
        groups_walk_kernel<K, CANON><<<(unsigned)grid, GS_THREADS, 0, st>>>(d_bases, args, chunks, 4u);
    });
    if (!walk) {
        if ((rc = resident_blocks((const void *)groups_generic_kernel<CANON>, GS_THREADS, 0, chunks, &grid)) != PG_OK) return rc;
        groups_generic_kernel<CANON><<<(unsigned)grid, GS_THREADS, 0, st>>>(d_bases, args, chunks, (uint32_t)k);
    }
    if (rc != PG_OK) return rc;
    PG_LAUNCH_CHECK(walk ? "groups_walk_kernel" : "groups_generic_kernel");
    return PG_OK;
}

int launch_walk(const uint8_t *d_bases, const PassArgs &args, uint64_t chunks, int k, bool canon, cudaStream_t st) {
    if (!chunks) return PG_OK;
    return canon ? launch_walk_mode<true>(d_bases, args, chunks, k, st) : launch_walk_mode<false>(d_bases, args, chunks, k, st);
}

}  // namespace

int sketch_groups(const uint8_t *d_bases, const uint64_t *d_off, uint64_t n_records, const uint64_t *d_goff, uint64_t G, int k, int s,
                  uint32_t m, bool canon, uint32_t *d_out, uint64_t row_stride, uint32_t *d_count, cudaStream_t st) {
    if (G == 0) return PG_OK;
    StreamScratch tmp(st);
    cudaError_t e;
    PG_CUDA(cudaMemsetAsync(d_out, 0, G * row_stride * 4, st));
    std::vector<uint64_t> wg, gbyte;
    uint64_t *d_gbyte = nullptr;
    int rc = group_sizes(d_off, n_records, d_goff, G, k, canon, tmp, wg, gbyte, &d_gbyte, st);
    if (rc != PG_OK) return rc;

    const double mu = admit_target((double)s);
    std::vector<GroupState> gs(G);
    for (uint64_t g = 0; g < G; ++g) {
        GroupState &x = gs[g];
        x.windows = wg[g];
        x.done = x.windows == 0;
        if (x.done) continue;
        x.width = std::min<uint64_t>(GS_RANGE, (uint64_t)std::ceil(mu / (double)x.windows * (double)GS_RANGE));
        x.width = std::max<uint64_t>(x.width, 1);
        x.slots = table_for(x, x.width);
    }

    GroupPass *d_gp = nullptr;
    unsigned long long *d_n = nullptr;
    if ((e = tmp.alloc(&d_gp, G)) != cudaSuccess || (e = tmp.alloc(&d_n, 1)) != cudaSuccess) return gs_nomem(e);
    std::vector<GroupPass> gp(G);
    std::vector<uint64_t> act;  // the pass's groups, by pass slot
    std::vector<Span> spans;
    std::vector<uint32_t> slot_of;
    std::vector<unsigned int> h_claims, h_ovf, h_qual;
    std::vector<Append> ap;
    const uint64_t chunk_bytes = walk_chunk_bytes(k);
    uint64_t next = 0;

    for (;;) {
        const uint64_t slots = pick_pass(gs, next, act);
        if (act.empty()) break;
        const uint64_t chunks = lay_out_pass(act, gs, gbyte, slots, chunk_bytes, gp, slot_of, spans);
        const uint64_t A = act.size();
        StreamScratch pass(st);  // this pass's tables and lists, released behind its work on the stream
        unsigned long long *d_keys = nullptr, *d_cnt = nullptr, *d_col = nullptr, *d_sorted = nullptr;
        unsigned int *d_claims = nullptr, *d_ovf = nullptr, *d_qual = nullptr;
        uint32_t *d_slot_of = nullptr;
        Span *d_spans = nullptr;
        Append *d_ap = nullptr;
        uint8_t *d_cub = nullptr;
        if ((e = pass.alloc(&d_keys, slots)) != cudaSuccess || (e = pass.alloc(&d_cnt, slots)) != cudaSuccess ||
            (e = pass.alloc(&d_col, slots)) != cudaSuccess || (e = pass.alloc(&d_sorted, slots)) != cudaSuccess ||
            (e = pass.alloc(&d_slot_of, slots / 64)) != cudaSuccess || (e = pass.alloc(&d_claims, A)) != cudaSuccess ||
            (e = pass.alloc(&d_ovf, A)) != cudaSuccess || (e = pass.alloc(&d_qual, A)) != cudaSuccess || (e = pass.alloc(&d_ap, A)) != cudaSuccess ||
            (e = pass.alloc(&d_spans, spans.size())) != cudaSuccess)
            return gs_nomem(e);
        PG_CUDA(cudaMemcpyAsync(d_gp, gp.data(), G * sizeof(GroupPass), cudaMemcpyHostToDevice, st));
        PG_CUDA(cudaMemcpyAsync(d_slot_of, slot_of.data(), slot_of.size() * 4, cudaMemcpyHostToDevice, st));
        if (!spans.empty()) PG_CUDA(cudaMemcpyAsync(d_spans, spans.data(), spans.size() * sizeof(Span), cudaMemcpyHostToDevice, st));
        PG_CUDA(cudaMemsetAsync(d_keys, 0xff, slots * 8, st));
        PG_CUDA(cudaMemsetAsync(d_cnt, 0, slots * 8, st));
        PG_CUDA(cudaMemsetAsync(d_claims, 0, A * 4, st));
        PG_CUDA(cudaMemsetAsync(d_ovf, 0, A * 4, st));
        PG_CUDA(cudaMemsetAsync(d_qual, 0, A * 4, st));
        PG_CUDA(cudaMemsetAsync(d_n, 0, 8, st));

        const PassArgs args{d_off, n_records, d_gbyte, G, d_gp, d_spans, (uint32_t)spans.size(), d_keys, d_cnt, d_claims, d_ovf};
        if ((rc = launch_walk(d_bases, args, chunks, k, canon, st)) != PG_OK) return rc;
        groups_collect_kernel<<<grid_for(slots), 256, 0, st>>>(d_keys, d_cnt, d_slot_of, slots, m, d_col, d_n, d_qual);
        PG_LAUNCH_CHECK("groups_collect_kernel");
        unsigned long long n_col = 0;
        h_claims.resize(A);
        h_ovf.resize(A);
        h_qual.resize(A);
        PG_CUDA(cudaMemcpyAsync(&n_col, d_n, 8, cudaMemcpyDeviceToHost, st));
        PG_CUDA(cudaMemcpyAsync(h_claims.data(), d_claims, A * 4, cudaMemcpyDeviceToHost, st));
        PG_CUDA(cudaMemcpyAsync(h_ovf.data(), d_ovf, A * 4, cudaMemcpyDeviceToHost, st));
        PG_CUDA(cudaMemcpyAsync(h_qual.data(), d_qual, A * 4, cudaMemcpyDeviceToHost, st));
        PG_CUDA(cudaStreamSynchronize(st));

        // what each group takes from its pass, and its next range
        ap.assign(A, Append{0, 0, 0, 0});
        uint64_t first = 0;
        bool any = false;
        for (uint32_t a = 0; a < A; ++a) {
            GroupState &x = gs[act[a]];
            ap[a].first = first;
            first += h_qual[a];
            if (h_ovf[a]) {  // drop the pass: half the width, twice the table
                x.width = std::max<uint64_t>(1, x.width / 2);
                x.slots = std::min(GS_MAX_TABLE, x.slots * 2);
                continue;
            }
            const uint32_t take = (uint32_t)std::min<uint64_t>(h_qual[a], (uint64_t)s - x.rows);
            ap[a] = Append{act[a], ap[a].first, take, x.rows};
            any = any || take;
            x.rows += take;
            x.covered += x.width;
            x.distinct += h_claims[a];
            x.qualified += h_qual[a];
            if (x.rows == (uint32_t)s || x.covered == GS_RANGE) {
                x.done = true;
                continue;
            }
            const double need = (double)s - (double)x.rows;
            double w = 64.0 * (double)x.width;
            if (x.qualified) w = std::min(w, admit_target(need) * (double)x.covered / (double)x.qualified);
            x.width = std::min<uint64_t>(GS_RANGE - x.covered, std::max<uint64_t>(1, (uint64_t)std::ceil(w)));
            x.slots = table_for(x, x.width);
            // a table past its largest size takes a narrower range instead
            while (x.slots == GS_MAX_TABLE && x.width > 1 && table_for(x, x.width / 2) == GS_MAX_TABLE) x.width /= 2;
        }
        if (any && n_col) {
            int bits = 32;
            while (bits < 64 && (A - 1) >> (bits - 32)) ++bits;
            size_t bytes = 0;
            PG_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, bytes, d_col, d_sorted, (int64_t)n_col, 0, bits, st));
            if ((e = pass.alloc(&d_cub, bytes)) != cudaSuccess) return gs_nomem(e);
            PG_CUDA(cub::DeviceRadixSort::SortKeys(d_cub, bytes, d_col, d_sorted, (int64_t)n_col, 0, bits, st));
            PG_CUDA(cudaMemcpyAsync(d_ap, ap.data(), A * sizeof(Append), cudaMemcpyHostToDevice, st));
            groups_append_kernel<<<grid_for(n_col), 256, 0, st>>>(d_sorted, n_col, d_ap, d_out, row_stride);
            PG_LAUNCH_CHECK("groups_append_kernel");
        }
        PG_CUDA(cudaStreamSynchronize(st));  // the host arrays of this pass are reused by the next
    }
    std::vector<uint32_t> cnt(G);
    for (uint64_t g = 0; g < G; ++g) cnt[g] = gs[g].rows;
    PG_CUDA(cudaMemcpyAsync(d_count, cnt.data(), G * 4, cudaMemcpyHostToDevice, st));
    PG_CUDA(cudaStreamSynchronize(st));
    return PG_OK;
}

void sketcher_free(SketcherState &S, cudaStream_t st) {
    for (void *p : {(void *)S.d_val, (void *)S.d_cnt, (void *)S.d_seg, (void *)S.d_cap})
        if (p) cudaFreeAsync(p, st);
    S.d_val = S.d_cnt = nullptr;
    S.d_seg = S.d_cap = nullptr;
}

int sketcher_init(SketcherState &S, cudaStream_t st) {
    S.seg.assign(S.G + 1, 0);
    S.cap.assign(S.G, GS_RANGE);
    cudaError_t e;
    if ((e = cudaMallocAsync(&S.d_seg, (S.G + 1) * 8, st)) != cudaSuccess || (e = cudaMallocAsync(&S.d_cap, S.G * 8, st)) != cudaSuccess) {
        sketcher_free(S, st);
        return gs_nomem(e);
    }
    PG_CUDA(cudaMemcpyAsync(S.d_seg, S.seg.data(), (S.G + 1) * 8, cudaMemcpyHostToDevice, st));
    PG_CUDA(cudaMemcpyAsync(S.d_cap, S.cap.data(), S.G * 8, cudaMemcpyHostToDevice, st));
    PG_CUDA(cudaStreamSynchronize(st));
    return PG_OK;
}

int sketcher_add(SketcherState &S, const uint8_t *d_bases, const uint64_t *d_off, uint64_t n_records, const uint64_t *d_goff, uint64_t first,
                 uint64_t nb, cudaStream_t st) {
    if (nb == 0 || n_records == 0) return PG_OK;
    StreamScratch tmp(st), keep(st);  // keep: the new state, released unless the add succeeds
    cudaError_t e;
    std::vector<uint64_t> wg, gbyte;
    uint64_t *d_gbyte = nullptr;
    int rc = group_sizes(d_off, n_records, d_goff, nb, S.k, S.canon, tmp, wg, gbyte, &d_gbyte, st);
    if (rc != PG_OK) return rc;
    const uint64_t B = S.B;
    const uint32_t s = (uint32_t)S.s, m = S.m;
    const uint64_t *seg = S.seg.data() + first;  // the batch's old segments
    const uint64_t old0 = seg[0], old_n = seg[nb] - seg[0];

    // a group walks ranges from 0 up to its old cap; the first admits mu of its windows and state entries on average
    const double mu = admit_target((double)s);
    std::vector<GroupState> gs(nb);
    std::vector<uint64_t> end(nb), cap(nb), held(nb, 0);  // old cap, new cap, values this add keeps
    std::vector<bool> walked(nb);
    for (uint64_t g = 0; g < nb; ++g) {
        GroupState &x = gs[g];
        end[g] = cap[g] = S.cap[first + g];
        walked[g] = wg[g] > 0;  // a group without windows keeps its state as it is
        x.done = !walked[g];
        if (x.done) continue;
        x.windows = wg[g] + (seg[g + 1] - seg[g]);
        x.width = std::min<uint64_t>(end[g], (uint64_t)std::ceil(mu / (double)x.windows * (double)GS_RANGE));
        x.width = std::max<uint64_t>(x.width, 1);
        x.slots = table_for(x, x.width);
    }
    if (std::none_of(walked.begin(), walked.end(), [](bool w) { return w; })) return PG_OK;

    GroupPass *d_gp = nullptr;
    unsigned long long *d_n = nullptr;
    if ((e = tmp.alloc(&d_gp, nb)) != cudaSuccess || (e = tmp.alloc(&d_n, 1)) != cudaSuccess) return gs_nomem(e);
    // the add's list: every kept entry as (batch group << 32 | value) and its count, in pass order, and sentinels
    unsigned long long *d_akey = nullptr;
    uint32_t *d_acnt = nullptr;
    uint64_t acc_n = 0, acc_cap = 0;
    const unsigned long long sentinel = (unsigned long long)nb << 32;
    std::vector<GroupPass> gp(nb);
    std::vector<uint64_t> act;
    std::vector<Span> spans;
    std::vector<uint32_t> slot_of;
    std::vector<unsigned int> h_ovf, h_per;
    std::vector<Cut> cut;
    std::vector<CutOut> res;
    const uint64_t chunk_bytes = walk_chunk_bytes(S.k);
    uint64_t next = 0;

    for (;;) {
        const uint64_t slots = pick_pass(gs, next, act);
        if (act.empty()) break;
        const uint64_t chunks = lay_out_pass(act, gs, gbyte, slots, chunk_bytes, gp, slot_of, spans);
        const uint64_t A = act.size();
        StreamScratch pass(st);
        unsigned long long *d_keys = nullptr, *d_cnt = nullptr, *d_col = nullptr, *d_sorted = nullptr;
        uint32_t *d_ccnt = nullptr, *d_scnt = nullptr, *d_qscan = nullptr, *d_slot_of = nullptr;
        unsigned int *d_claims = nullptr, *d_ovf = nullptr, *d_per = nullptr;
        Span *d_spans = nullptr;
        Cut *d_cut = nullptr;
        CutOut *d_res = nullptr;
        uint8_t *d_cub = nullptr;
        if ((e = pass.alloc(&d_keys, slots)) != cudaSuccess || (e = pass.alloc(&d_cnt, slots)) != cudaSuccess ||
            (e = pass.alloc(&d_col, slots)) != cudaSuccess || (e = pass.alloc(&d_sorted, slots)) != cudaSuccess ||
            (e = pass.alloc(&d_ccnt, slots)) != cudaSuccess || (e = pass.alloc(&d_scnt, slots)) != cudaSuccess ||
            (e = pass.alloc(&d_qscan, slots)) != cudaSuccess || (e = pass.alloc(&d_slot_of, slots / 64)) != cudaSuccess ||
            (e = pass.alloc(&d_claims, A)) != cudaSuccess || (e = pass.alloc(&d_ovf, A)) != cudaSuccess || (e = pass.alloc(&d_per, A)) != cudaSuccess ||
            (e = pass.alloc(&d_cut, A)) != cudaSuccess || (e = pass.alloc(&d_res, A)) != cudaSuccess ||
            (e = pass.alloc(&d_spans, spans.size())) != cudaSuccess)
            return gs_nomem(e);
        PG_CUDA(cudaMemcpyAsync(d_gp, gp.data(), nb * sizeof(GroupPass), cudaMemcpyHostToDevice, st));
        PG_CUDA(cudaMemcpyAsync(d_slot_of, slot_of.data(), slot_of.size() * 4, cudaMemcpyHostToDevice, st));
        if (!spans.empty()) PG_CUDA(cudaMemcpyAsync(d_spans, spans.data(), spans.size() * sizeof(Span), cudaMemcpyHostToDevice, st));
        PG_CUDA(cudaMemsetAsync(d_keys, 0xff, slots * 8, st));
        PG_CUDA(cudaMemsetAsync(d_cnt, 0, slots * 8, st));
        PG_CUDA(cudaMemsetAsync(d_claims, 0, A * 4, st));
        PG_CUDA(cudaMemsetAsync(d_ovf, 0, A * 4, st));
        PG_CUDA(cudaMemsetAsync(d_per, 0, A * 4, st));
        PG_CUDA(cudaMemsetAsync(d_n, 0, 8, st));

        const PassArgs args{d_off, n_records, d_gbyte, nb, d_gp, d_spans, (uint32_t)spans.size(), d_keys, d_cnt, d_claims, d_ovf};
        // a pass is always 4 launches (seed, walk, collect, cut), so that a caller can count passes
        sketcher_seed_kernel<<<grid_for(old_n), 256, 0, st>>>(S.d_val, S.d_cnt, S.d_seg + first, nb, args);
        PG_LAUNCH_CHECK("sketcher_seed_kernel");
        if ((rc = launch_walk(d_bases, args, chunks, S.k, S.canon, st)) != PG_OK) return rc;
        sketcher_collect_kernel<<<grid_for(slots), 256, 0, st>>>(d_keys, d_cnt, d_slot_of, slots, m, d_col, d_ccnt, d_n, d_per);
        PG_LAUNCH_CHECK("sketcher_collect_kernel");
        unsigned long long n_col = 0;
        h_ovf.resize(A);
        h_per.resize(A);
        PG_CUDA(cudaMemcpyAsync(&n_col, d_n, 8, cudaMemcpyDeviceToHost, st));
        PG_CUDA(cudaMemcpyAsync(h_ovf.data(), d_ovf, A * 4, cudaMemcpyDeviceToHost, st));
        PG_CUDA(cudaMemcpyAsync(h_per.data(), d_per, A * 4, cudaMemcpyDeviceToHost, st));
        PG_CUDA(cudaStreamSynchronize(st));

        // each slot's entries in the sorted list and its room in the add's list
        cut.assign(A, Cut{0, 0, 0, 0, 0, 0, 0, 0, 0});
        res.assign(A, CutOut{GS_RANGE, GS_RANGE, 0, 0});
        uint64_t at = 0, room = 0;
        for (uint32_t a = 0; a < A; ++a) {
            const uint64_t g = act[a];
            GroupState &x = gs[g];
            Cut &c = cut[a];
            c.first = at;
            c.n = h_per[a];
            at += h_per[a];
            if (h_ovf[a]) {  // drop the pass: half the width, twice the table
                x.width = std::max<uint64_t>(1, x.width / 2);
                x.slots = std::min(GS_MAX_TABLE, x.slots * 2);
                continue;
            }
            c.held = held[g];
            c.qual = x.rows;
            c.group = (uint32_t)g;
            c.live = 1;
            c.out = acc_n + room;
            c.room = std::min<uint64_t>(c.n, B - held[g]);
            room += c.room;
        }
        if (acc_n + room > acc_cap) {  // grow the add's list; the old one is released with tmp
            const uint64_t want = std::max(acc_n + room, 2 * acc_cap);
            unsigned long long *k2 = nullptr;
            uint32_t *c2 = nullptr;
            if ((e = tmp.alloc(&k2, want)) != cudaSuccess || (e = tmp.alloc(&c2, want)) != cudaSuccess) return gs_nomem(e);
            if (acc_n) {
                PG_CUDA(cudaMemcpyAsync(k2, d_akey, acc_n * 8, cudaMemcpyDeviceToDevice, st));
                PG_CUDA(cudaMemcpyAsync(c2, d_acnt, acc_n * 4, cudaMemcpyDeviceToDevice, st));
            }
            d_akey = k2;
            d_acnt = c2;
            acc_cap = want;
        }
        if (n_col) {
            int bits = 32;
            while (bits < 64 && (A - 1) >> (bits - 32)) ++bits;
            const auto flags = thrust::make_transform_iterator(d_scnt, QualFlag{m});
            size_t sort_bytes = 0, scan_bytes = 0;
            PG_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, d_col, d_sorted, d_ccnt, d_scnt, (int64_t)n_col, 0, bits, st));
            PG_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, flags, d_qscan, (int64_t)n_col, st));
            if ((e = pass.alloc(&d_cub, std::max(sort_bytes, scan_bytes))) != cudaSuccess) return gs_nomem(e);
            PG_CUDA(cub::DeviceRadixSort::SortPairs(d_cub, sort_bytes, d_col, d_sorted, d_ccnt, d_scnt, (int64_t)n_col, 0, bits, st));
            PG_CUDA(cub::DeviceScan::ExclusiveSum(d_cub, scan_bytes, flags, d_qscan, (int64_t)n_col, st));
        }
        PG_CUDA(cudaMemcpyAsync(d_cut, cut.data(), A * sizeof(Cut), cudaMemcpyHostToDevice, st));
        PG_CUDA(cudaMemcpyAsync(d_res, res.data(), A * sizeof(CutOut), cudaMemcpyHostToDevice, st));
        sketcher_cut_kernel<<<grid_for(n_col), 256, 0, st>>>(d_sorted, d_scnt, d_qscan, n_col, d_cut, m, s, B, sentinel, d_akey, d_acnt, d_res);
        PG_LAUNCH_CHECK("sketcher_cut_kernel");
        PG_CUDA(cudaMemcpyAsync(res.data(), d_res, A * sizeof(CutOut), cudaMemcpyDeviceToHost, st));
        PG_CUDA(cudaStreamSynchronize(st));  // the host arrays of this pass are reused by the next
        acc_n += room;

        // what each group kept, its cap, and its next range
        for (uint32_t a = 0; a < A; ++a) {
            if (!cut[a].live) continue;
            const uint64_t g = act[a];
            GroupState &x = gs[g];
            held[g] += res[a].kept;
            x.rows += res[a].qkept;
            x.distinct += h_per[a];
            x.qualified += res[a].qkept;
            x.covered += x.width;
            cap[g] = std::min<uint64_t>(cap[g], std::min<uint64_t>(res[a].cap_s, res[a].cap_b));
            if (cap[g] < end[g] || x.covered >= end[g]) {  // cut inside the range, or every range below the old cap done
                x.done = true;
                continue;
            }
            const double need = (double)s - (double)x.rows;
            double w = 64.0 * (double)x.width;
            if (x.qualified) w = std::min(w, admit_target(need) * (double)x.covered / (double)x.qualified);
            if (x.distinct) w = std::min(w, admit_target((double)(B - held[g]) + 1.0) * (double)x.covered / (double)x.distinct);
            x.width = std::min<uint64_t>(end[g] - x.covered, std::max<uint64_t>(1, (uint64_t)std::ceil(w)));
            x.slots = table_for(x, x.width);
            while (x.slots == GS_MAX_TABLE && x.width > 1 && table_for(x, x.width / 2) == GS_MAX_TABLE) x.width /= 2;
        }
    }

    // the add's list sorted by (group, value): the sentinels go last, each walked group's entries form one run
    unsigned long long *d_skey = nullptr;
    uint32_t *d_sacnt = nullptr;
    if (acc_n) {
        int bits = 32;
        while (bits < 64 && nb >> (bits - 32)) ++bits;
        size_t bytes = 0;
        uint8_t *d_cub = nullptr;
        if ((e = tmp.alloc(&d_skey, acc_n)) != cudaSuccess || (e = tmp.alloc(&d_sacnt, acc_n)) != cudaSuccess) return gs_nomem(e);
        PG_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, bytes, d_akey, d_skey, d_acnt, d_sacnt, (int64_t)acc_n, 0, bits, st));
        if ((e = tmp.alloc(&d_cub, bytes)) != cudaSuccess) return gs_nomem(e);
        PG_CUDA(cub::DeviceRadixSort::SortPairs(d_cub, bytes, d_akey, d_skey, d_acnt, d_sacnt, (int64_t)acc_n, 0, bits, st));
    }

    // the new state: the old one before and after the batch's groups, and their new segments between
    std::vector<uint64_t> nseg(nb + 1), from(nb), new_seg(S.seg), new_cap(S.cap);
    uint64_t run = 0;  // where the next walked group's run starts in the sorted list
    for (uint64_t g = 0; g < nb; ++g) {
        const uint64_t h = walked[g] ? held[g] : seg[g + 1] - seg[g];
        from[g] = walked[g] ? (SK_FROM_ADD | run) : seg[g];
        if (walked[g]) run += held[g];
        nseg[g + 1] = nseg[g] + h;
        new_cap[first + g] = cap[g];
    }
    const uint64_t mid = nseg[nb], total = S.seg[S.G] - old_n + mid;
    for (uint64_t g = 0; g <= S.G - first; ++g)
        new_seg[first + g] = g <= nb ? old0 + nseg[g] : S.seg[first + g] - old_n + mid;
    uint32_t *d_val = nullptr, *d_vcnt = nullptr;
    uint64_t *d_seg = nullptr, *d_cap = nullptr, *d_nseg = nullptr, *d_from = nullptr;
    if ((e = keep.alloc(&d_val, total)) != cudaSuccess || (e = keep.alloc(&d_vcnt, total)) != cudaSuccess ||
        (e = keep.alloc(&d_seg, S.G + 1)) != cudaSuccess || (e = keep.alloc(&d_cap, S.G)) != cudaSuccess ||
        (e = tmp.alloc(&d_nseg, nb + 1)) != cudaSuccess || (e = tmp.alloc(&d_from, nb)) != cudaSuccess)
        return gs_nomem(e);
    if (old0) {
        PG_CUDA(cudaMemcpyAsync(d_val, S.d_val, old0 * 4, cudaMemcpyDeviceToDevice, st));
        PG_CUDA(cudaMemcpyAsync(d_vcnt, S.d_cnt, old0 * 4, cudaMemcpyDeviceToDevice, st));
    }
    const uint64_t tail = S.seg[S.G] - seg[nb];
    if (tail) {
        PG_CUDA(cudaMemcpyAsync(d_val + old0 + mid, S.d_val + seg[nb], tail * 4, cudaMemcpyDeviceToDevice, st));
        PG_CUDA(cudaMemcpyAsync(d_vcnt + old0 + mid, S.d_cnt + seg[nb], tail * 4, cudaMemcpyDeviceToDevice, st));
    }
    PG_CUDA(cudaMemcpyAsync(d_nseg, nseg.data(), (nb + 1) * 8, cudaMemcpyHostToDevice, st));
    PG_CUDA(cudaMemcpyAsync(d_from, from.data(), nb * 8, cudaMemcpyHostToDevice, st));
    PG_CUDA(cudaMemcpyAsync(d_seg, new_seg.data(), (S.G + 1) * 8, cudaMemcpyHostToDevice, st));
    PG_CUDA(cudaMemcpyAsync(d_cap, new_cap.data(), S.G * 8, cudaMemcpyHostToDevice, st));
    sketcher_merge_kernel<<<grid_for(mid), 256, 0, st>>>(d_nseg, nb, d_from, d_skey, d_sacnt, S.d_val, S.d_cnt, d_val + old0, d_vcnt + old0);
    PG_LAUNCH_CHECK("sketcher_merge_kernel");
    PG_CUDA(cudaStreamSynchronize(st));

    keep.ptr.clear();
    sketcher_free(S, st);
    S.d_val = d_val;
    S.d_cnt = d_vcnt;
    S.d_seg = d_seg;
    S.d_cap = d_cap;
    S.seg.swap(new_seg);
    S.cap.swap(new_cap);
    return PG_OK;
}

int sketcher_rows(const SketcherState &S, uint64_t first, uint64_t count, uint32_t *d_out, uint64_t row_stride, uint32_t *d_n, uint8_t *d_complete,
                  uint64_t *d_held, cudaStream_t st) {
    if (count == 0) return PG_OK;
    sketcher_rows_kernel<<<grid_for(count * 32), 256, 0, st>>>(S.d_val, S.d_cnt, S.d_seg, S.d_cap, first, count, (uint32_t)S.s, S.m, d_out, row_stride,
                                                               d_n, d_complete, d_held);
    PG_LAUNCH_CHECK("sketcher_rows_kernel");
    return PG_OK;
}

}  // namespace pg
