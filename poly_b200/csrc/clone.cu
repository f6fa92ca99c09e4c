// clone.cu -- clone.CutWithEnzyme (clone/clone.go:138-268) for every (part, enzyme) item of a batch, and the
// byte copy that materialises ligation constructs from their recipes (DESIGN.md "Clone").
//
// Digest, count -> scan -> write (as fastq_ingest.cu):
//   1. clone_sites_kernel<false>: one warp per item walks the part (twice its length when circular, read as
//      index mod L and upper-cased on the fly -- the doubled string is never built) 32 positions at a time,
//      tests both literal sites at every position, and keeps the leftmost non-overlapping matches of each
//      (regexp.FindAllStringIndex) in position order.  It counts them and flags bytes >= 0x80.
//   2. the same kernel with WRITE: items with matches walk again and store the match starts.
//   3. clone_fragments_kernel: one thread per item turns its matches into overhangs (drop, stable merge)
//      and fragments (the four branches), checking every slice bound as Go does; a slice out of range
//      makes the item PG_ITEM_PANIC.  A fragment is spans of the virtual sequence.
//   4. scans of the per-item fragment and byte counts; clone_offsets_kernel writes the output offsets.
//   5. clone_copy_kernel: one warp per fragment copies its spans, upper-cased.
// Ligation: clone_pieces_kernel, one warp per piece, copies a span of the source buffer forwards or
// reverse-complemented (read backwards through complement()) to its place in the construct buffer.
#include <cub/device/device_scan.cuh>

#include "clone.cuh"

namespace pg {

namespace {

constexpr unsigned FULL = 0xffffffffu;

__device__ __forceinline__ uint8_t upper(uint8_t c) { return (c >= 'a' && c <= 'z') ? c - 32 : c; }

// byte x of strings.ToUpper(part) or of strings.ToUpper(part + part); 0 past the end (sites hold no 0 byte)
__device__ __forceinline__ uint8_t vbyte(const uint8_t *part, uint64_t L, uint64_t N, uint64_t x) {
    if (x >= N) return 0;
    return upper(__ldg(part + (x < L ? x : x - L)));
}

// Go's s[lo:hi] on a string of length n is in range iff 0 <= lo <= hi <= n
__device__ __forceinline__ bool in_range(int64_t lo, int64_t hi, int64_t n) { return 0 <= lo && lo <= hi && hi <= n; }

// One warp per (part, enzyme) item.  Per item: n_fwd / n_rev leftmost non-overlapping matches of the two sites
// (no reverse matches for a palindromic recognition site), and PG_ITEM_UNSUPPORTED for a byte >= 0x80.
// WRITE: the match starts go to starts[base[item] ..) -- forward first, then reverse.
template <bool WRITE>
__global__ void __launch_bounds__(256) clone_sites_kernel(const uint8_t *__restrict__ parts, const uint64_t *__restrict__ off,
                                                          const uint8_t *__restrict__ circular, uint64_t n_items, uint32_t n_enz,
                                                          const CloneEnzyme *__restrict__ enz, uint32_t *n_fwd, uint32_t *n_rev,
                                                          int32_t *status, const uint64_t *__restrict__ base, int64_t *starts) {
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t warps = (uint64_t)gridDim.x * (blockDim.x / 32);
    for (uint64_t item = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32; item < n_items; item += warps) {
        if (WRITE && n_fwd[item] + n_rev[item] == 0) continue;
        const uint64_t p = item / n_enz;
        const CloneEnzyme &e = enz[item % n_enz];
        const uint8_t *part = parts + off[p];
        const uint64_t L = off[p + 1] - off[p], N = circular[p] ? 2 * L : L;
        const uint32_t fl = e.fl, rl = e.palindromic ? 0 : e.rl;
        uint64_t f_next = 0, r_next = 0;  // a match may start here or later (non-overlap)
        uint32_t nf = 0, nr = 0;
        bool wide = false;
        int64_t *fs = WRITE ? starts + base[item] : nullptr, *rs = WRITE ? fs + n_fwd[item] : nullptr;
        uint8_t b1 = vbyte(part, L, N, lane);
        for (uint64_t q = 0; q < N; q += 32) {
            const uint8_t b0 = b1;
            b1 = vbyte(part, L, N, q + 32 + lane);
            if (!WRITE) wide |= __any_sync(FULL, q + lane < L && __ldg(part + q + lane) >= 0x80);
            bool fm = fl > 0, rm = rl > 0;
            const uint32_t m = max(fl, rl);
            for (uint32_t j = 0; j < m; ++j) {  // byte q + lane + j of the window, from the lane that holds it
                const uint32_t src = (lane + j) & 31;
                const uint8_t lo = __shfl_sync(FULL, b0, src), hi = __shfl_sync(FULL, b1, src);
                const uint8_t c = lane + j < 32 ? lo : hi;
                if (j < fl) fm &= c == e.fsite[j];
                if (j < rl) rm &= c == e.rsite[j];
            }
            // greedy non-overlap in position order, the same on every lane
            for (uint32_t bits = __ballot_sync(FULL, fm); bits; bits &= bits - 1) {
                const uint64_t pos = q + __ffs(bits) - 1;
                if (pos < f_next) continue;
                if (WRITE && lane == 0) fs[nf] = (int64_t)pos;
                ++nf;
                f_next = pos + fl;
            }
            for (uint32_t bits = __ballot_sync(FULL, rm); bits; bits &= bits - 1) {
                const uint64_t pos = q + __ffs(bits) - 1;
                if (pos < r_next) continue;
                if (WRITE && lane == 0) rs[nr] = (int64_t)pos;
                ++nr;
                r_next = pos + rl;
            }
        }
        if (!WRITE && lane == 0) {
            n_fwd[item] = wide ? 0 : nf;
            n_rev[item] = wide ? 0 : nr;
            status[item] = wide ? PG_ITEM_UNSUPPORTED : PG_ITEM_OK;
        }
    }
}

// Overhang k of an item in sort.SliceStable order of forward ++ reverse: both sets are ascending, so the
// stable sort is a merge that takes the forward overhang on ties.
struct Overhangs {
    const int64_t *fs, *rs;
    int64_t kf, kr, fshift, rshift;  // kept counts; position = start + shift
    int64_t a = 0, b = 0;
    __device__ bool next(int64_t *pos, bool *fwd) {
        if (a >= kf && b >= kr) return false;
        *fwd = b >= kr || (a < kf && fs[a] + fshift <= rs[b] + rshift);
        *pos = *fwd ? fs[a++] + fshift : rs[b++] + rshift;
        return true;
    }
};

// One thread per item (grid-stride): the fragments of CutWithEnzyme (clone.go:139-267) as span records, at most
// n_fwd + n_rev + 1 of them, at rec[base[item] + item ..).
__global__ void __launch_bounds__(128) clone_fragments_kernel(const uint64_t *__restrict__ off, const uint8_t *__restrict__ circular,
                                                              uint64_t n_items, uint32_t n_enz, const CloneEnzyme *__restrict__ enz,
                                                              int directional, const uint32_t *__restrict__ n_fwd,
                                                              const uint32_t *__restrict__ n_rev, const uint64_t *__restrict__ base,
                                                              const int64_t *__restrict__ starts, int32_t *status, FragRec *rec,
                                                              uint64_t *n_frag, uint64_t *seq_bytes, uint64_t *oh_bytes) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t item = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; item < n_items; item += stride) {
        const uint64_t p = item / n_enz;
        const CloneEnzyme &e = enz[item % n_enz];
        const bool circ = circular[p];
        const int64_t L = (int64_t)(off[p + 1] - off[p]), N = circ ? 2 * L : L;
        const int64_t skip = e.skip, OH = e.ohl, nf = n_fwd[item], nr = n_rev[item];
        Overhangs ov{starts + base[item], starts + base[item] + nf, nf, nr, (int64_t)e.fl + skip, -skip};
        // on a linear part, drop the last overhang of a set past the end (Skip counted twice, clone.go:166-174)
        if (!circ && ov.kf > 0 && ov.fs[ov.kf - 1] + ov.fshift + skip + OH > N) --ov.kf;
        if (!circ && ov.kr > 0 && ov.rs[ov.kr - 1] + ov.rshift + skip + OH > N) --ov.kr;
        const int64_t n = ov.kf + ov.kr;
        FragRec *out = rec + base[item] + item;
        uint64_t cnt = 0, sb = 0, ob = 0;
        bool panic = false;
        auto put = [&](int64_t a0, int64_t a1, int64_t b0, int64_t b1, int64_t f0, int64_t f1, int64_t r0, int64_t r1) {
            out[cnt++] = FragRec{a0, a1, b0, b1, f0, f1, r0, r1, p};
            sb += (a1 - a0) + (b1 - b0);
            ob += (f1 - f0) + (r1 - r0);
        };
        int64_t P;
        bool fwd;
        if (status[item] != PG_ITEM_OK) {
            // a byte >= 0x80: not cut
        } else if (n == 1 && !directional && !circ) {  // a single cut on a linear part (clone.go:187-209)
            ov.next(&P, &fwd);
            if (nf > 0) {  // len(forwardOverhangs): the set before the drop
                panic = !in_range(P + OH, N, N) || !in_range(0, P, N) || !in_range(P, P + OH, N);
                if (!panic) {
                    put(P + OH, N, 0, 0, P, P + OH, 0, 0);
                    put(0, P, 0, 0, 0, 0, P, P + OH);
                }
            } else {
                panic = !in_range(P, N, N) || !in_range(0, P - OH, N) || !in_range(P - OH, P, N);
                if (!panic) {
                    put(0, P - OH, 0, 0, 0, 0, P - OH, P);
                    put(P, N, 0, 0, P - OH, P, 0, 0);
                }
            }
        } else if (n == 2 && !directional && circ) {  // one fragment across the origin (clone.go:214-222)
            ov.next(&P, &fwd);
            panic = !in_range(P + OH, L, N) || !in_range(0, P, N) || !in_range(P, P + OH, N);
            if (!panic) put(P + OH, L, 0, P, P, P + OH, P, P + OH);
        } else if (n > 1) {  // the pairwise loop (clone.go:232-253) and the length filter (:255-264)
            const int64_t rssl = (int64_t)e.recl + skip;
            const bool pairwise_all = !(directional && !e.palindromic);
            int64_t cur, nxt;
            bool cur_fwd, nxt_fwd;
            ov.next(&cur, &cur_fwd);
            for (int64_t i = 0; i < n - 1 && !panic; ++i) {
                ov.next(&nxt, &nxt_fwd);
                if (pairwise_all || (cur_fwd && !nxt_fwd)) {
                    const int64_t len = nxt - cur;
                    if (!in_range(cur, nxt, N)) {
                        panic = true;
                    } else if (len > 8) {
                        panic = !in_range(OH, len - OH, len) || !in_range(0, OH, len) || !in_range(len - OH, len, len);
                        if (!panic) put(cur + OH, nxt - OH, 0, 0, cur, cur + OH, nxt - OH, nxt);
                    }
                }
                if (nxt - rssl > L) break;
                cur = nxt;
                cur_fwd = nxt_fwd;
            }
        }
        if (panic) {
            status[item] = PG_ITEM_PANIC;
            cnt = sb = ob = 0;
        }
        n_frag[item] = cnt;
        seq_bytes[item] = sb;
        oh_bytes[item] = ob;
    }
}

// One thread per item (grid-stride): output offsets of its fragments from the scanned counts; the last item also writes
// the closing offsets.  frag_rec[f] = the record of output fragment f.
__global__ void __launch_bounds__(128) clone_offsets_kernel(uint64_t n_items, const uint32_t *__restrict__ n_fwd,
                                                            const uint32_t *__restrict__ n_rev, const uint64_t *__restrict__ base,
                                                            const FragRec *__restrict__ rec, const uint64_t *__restrict__ n_frag,
                                                            const uint64_t *__restrict__ f_scan, const uint64_t *__restrict__ s_scan,
                                                            const uint64_t *__restrict__ o_scan, uint64_t *seq_off, uint64_t *oh_off,
                                                            uint64_t *frag_rec) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t item = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; item < n_items; item += stride) {
        const uint64_t r0 = base[item] + item;
        uint64_t f = f_scan[item], s = s_scan[item], o = o_scan[item];
        for (uint64_t k = 0; k < n_frag[item]; ++k, ++f) {
            const FragRec &r = rec[r0 + k];
            frag_rec[f] = r0 + k;
            seq_off[f] = s;
            oh_off[2 * f] = o;
            oh_off[2 * f + 1] = o + (r.f1 - r.f0);
            s += (r.a1 - r.a0) + (r.b1 - r.b0);
            o += (r.f1 - r.f0) + (r.r1 - r.r0);
        }
        if (item == n_items - 1) {
            seq_off[f] = s;
            oh_off[2 * f] = o;
        }
    }
}

__device__ __forceinline__ void copy_span(const uint8_t *part, uint64_t L, int64_t a, int64_t b, uint8_t *dst, uint32_t lane) {
    for (int64_t x = a + lane; x < b; x += 32) dst[x - a] = upper(__ldg(part + (x < (int64_t)L ? x : x - (int64_t)L)));
}

// One warp per output fragment: Sequence (one or two spans), ForwardOverhang and ReverseOverhang, upper-cased
__global__ void __launch_bounds__(256) clone_copy_kernel(const uint8_t *__restrict__ parts, const uint64_t *__restrict__ off,
                                                         uint64_t n_frags, const FragRec *__restrict__ rec,
                                                         const uint64_t *__restrict__ frag_rec, const uint64_t *__restrict__ seq_off,
                                                         const uint64_t *__restrict__ oh_off, uint8_t *seq, uint8_t *oh) {
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t warps = (uint64_t)gridDim.x * (blockDim.x / 32);
    for (uint64_t f = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32; f < n_frags; f += warps) {
        const FragRec r = rec[frag_rec[f]];
        const uint8_t *part = parts + off[r.part];
        const uint64_t L = off[r.part + 1] - off[r.part];
        copy_span(part, L, r.a0, r.a1, seq + seq_off[f], lane);
        copy_span(part, L, r.b0, r.b1, seq + seq_off[f] + (r.a1 - r.a0), lane);
        copy_span(part, L, r.f0, r.f1, oh + oh_off[2 * f], lane);
        copy_span(part, L, r.r0, r.r1, oh + oh_off[2 * f + 1], lane);
    }
}

// One warp per piece: src[s, s + len) forwards, or its reverse complement, to dst
__global__ void __launch_bounds__(256) clone_pieces_kernel(const uint8_t *__restrict__ src, const Piece *__restrict__ pieces,
                                                           uint64_t n_pieces, uint8_t *dst) {
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t warps = (uint64_t)gridDim.x * (blockDim.x / 32);
    for (uint64_t k = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32; k < n_pieces; k += warps) {
        const Piece pc = pieces[k];
        const uint8_t *s = src + pc.src;
        uint8_t *d = dst + pc.dst;
        if (pc.rc)
            for (uint64_t i = lane; i < pc.len; i += 32) d[i] = complement(__ldg(s + pc.len - 1 - i));
        else
            for (uint64_t i = lane; i < pc.len; i += 32) d[i] = __ldg(s + i);
    }
}

// cnt[i] = matches of item i, cnt[n] = 0 (the scan's total)
__global__ void clone_sum_kernel(const uint32_t *__restrict__ n_fwd, const uint32_t *__restrict__ n_rev, uint64_t n, uint64_t *cnt) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= n; i += stride) cnt[i] = i < n ? (uint64_t)n_fwd[i] + n_rev[i] : 0;
}

unsigned grid_for(uint64_t work, unsigned per_block, unsigned cap) {
    return (unsigned)std::max<uint64_t>(1, std::min<uint64_t>((work + per_block - 1) / per_block, cap));
}

int exclusive_sum(const uint64_t *in, uint64_t *out, uint64_t n, StreamScratch &tmp, cudaStream_t st) {
    size_t bytes = 0;
    PG_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, bytes, in, out, (int64_t)n, st));
    uint8_t *t = nullptr;
    PG_CUDA(tmp.alloc(&t, bytes));
    PG_CUDA(cub::DeviceScan::ExclusiveSum(t, bytes, in, out, (int64_t)n, st));
    return PG_OK;
}

}  // namespace

int clone_digest_plan(const uint8_t *d_parts, const uint64_t *d_off, const uint8_t *d_circ, uint64_t n_parts, const CloneEnzyme *d_enz,
                      uint32_t n_enz, int directional, StreamScratch &tmp, cudaStream_t st, DigestPlan *plan) {
    const uint64_t n = n_parts * n_enz;
    DigestPlan &d = *plan;
    d = DigestPlan{};
    d.n_items = n;
    d.parts = d_parts;
    d.off = d_off;
    PG_CUDA(tmp.alloc(&d.n_fwd, n));
    PG_CUDA(tmp.alloc(&d.n_rev, n));
    PG_CUDA(tmp.alloc(&d.status, n));
    PG_CUDA(tmp.alloc(&d.base, n + 1));
    uint64_t *cnt = nullptr;
    PG_CUDA(tmp.alloc(&cnt, n + 1));
    const unsigned sms = (unsigned)sm_count();
    clone_sites_kernel<false><<<grid_for(n, 8, sms * 64), 256, 0, st>>>(d_parts, d_off, d_circ, n, n_enz, d_enz, d.n_fwd, d.n_rev, d.status,
                                                                         nullptr, nullptr);
    PG_LAUNCH_CHECK("clone_sites_kernel<count>");
    // base = exclusive scan of n_fwd + n_rev (match starts); records sit at base[item] + item
    clone_sum_kernel<<<grid_for(n + 1, 256, 1u << 20), 256, 0, st>>>(d.n_fwd, d.n_rev, n, cnt);
    PG_LAUNCH_CHECK("clone_sum_kernel");
    int rc;
    if ((rc = exclusive_sum(cnt, d.base, n + 1, tmp, st)) != PG_OK) return rc;
    uint64_t n_starts = 0;
    PG_CUDA(cudaMemcpyAsync(&n_starts, d.base + n, 8, cudaMemcpyDeviceToHost, st));
    PG_CUDA(cudaStreamSynchronize(st));
    PG_CUDA(tmp.alloc(&d.starts, n_starts));
    PG_CUDA(tmp.alloc(&d.rec, n_starts + n));
    clone_sites_kernel<true><<<grid_for(n, 8, sms * 64), 256, 0, st>>>(d_parts, d_off, d_circ, n, n_enz, d_enz, d.n_fwd, d.n_rev, d.status,
                                                                        d.base, d.starts);
    PG_LAUNCH_CHECK("clone_sites_kernel<write>");
    PG_CUDA(tmp.alloc(&d.n_frag, n + 1));
    PG_CUDA(tmp.alloc(&d.seq_bytes, n + 1));
    PG_CUDA(tmp.alloc(&d.oh_bytes, n + 1));
    clone_fragments_kernel<<<grid_for(n, 128, 1u << 30), 128, 0, st>>>(d_off, d_circ, n, n_enz, d_enz, directional, d.n_fwd, d.n_rev, d.base,
                                                                       d.starts, d.status, d.rec, d.n_frag, d.seq_bytes, d.oh_bytes);
    PG_LAUNCH_CHECK("clone_fragments_kernel");
    PG_CUDA(tmp.alloc(&d.f_scan, n + 1));
    PG_CUDA(tmp.alloc(&d.s_scan, n + 1));
    PG_CUDA(tmp.alloc(&d.o_scan, n + 1));
    PG_CUDA(cudaMemsetAsync(d.n_frag + n, 0, 8, st));
    PG_CUDA(cudaMemsetAsync(d.seq_bytes + n, 0, 8, st));
    PG_CUDA(cudaMemsetAsync(d.oh_bytes + n, 0, 8, st));
    if ((rc = exclusive_sum(d.n_frag, d.f_scan, n + 1, tmp, st)) != PG_OK || (rc = exclusive_sum(d.seq_bytes, d.s_scan, n + 1, tmp, st)) != PG_OK ||
        (rc = exclusive_sum(d.oh_bytes, d.o_scan, n + 1, tmp, st)) != PG_OK)
        return rc;
    uint64_t tot[3];
    PG_CUDA(cudaMemcpyAsync(&tot[0], d.f_scan + n, 8, cudaMemcpyDeviceToHost, st));
    PG_CUDA(cudaMemcpyAsync(&tot[1], d.s_scan + n, 8, cudaMemcpyDeviceToHost, st));
    PG_CUDA(cudaMemcpyAsync(&tot[2], d.o_scan + n, 8, cudaMemcpyDeviceToHost, st));
    PG_CUDA(cudaStreamSynchronize(st));
    d.frags = tot[0];
    d.seq_total = tot[1];
    d.oh_total = tot[2];
    return PG_OK;
}

int clone_digest_write(const DigestPlan &d, uint64_t *d_seq_off, uint8_t *d_seq, uint64_t *d_oh_off, uint8_t *d_oh, StreamScratch &tmp,
                       cudaStream_t st) {
    uint64_t *frag_rec = nullptr;
    PG_CUDA(tmp.alloc(&frag_rec, d.frags));
    clone_offsets_kernel<<<grid_for(d.n_items, 128, 1u << 30), 128, 0, st>>>(d.n_items, d.n_fwd, d.n_rev, d.base, d.rec, d.n_frag, d.f_scan,
                                                                             d.s_scan, d.o_scan, d_seq_off, d_oh_off, frag_rec);
    PG_LAUNCH_CHECK("clone_offsets_kernel");
    if (d.frags == 0) return PG_OK;
    clone_copy_kernel<<<grid_for(d.frags, 8, (unsigned)sm_count() * 64), 256, 0, st>>>(d.parts, d.off, d.frags, d.rec, frag_rec, d_seq_off,
                                                                                      d_oh_off, d_seq, d_oh);
    PG_LAUNCH_CHECK("clone_copy_kernel");
    return PG_OK;
}

int launch_clone_pieces(const uint8_t *d_src, const Piece *d_pieces, uint64_t n_pieces, uint8_t *d_dst, cudaStream_t st) {
    if (n_pieces == 0) return PG_OK;
    clone_pieces_kernel<<<grid_for(n_pieces, 8, (unsigned)sm_count() * 64), 256, 0, st>>>(d_src, d_pieces, n_pieces, d_dst);
    PG_LAUNCH_CHECK("clone_pieces_kernel");
    return PG_OK;
}

}  // namespace pg
