// fragment.cu -- poly's synthesis/fragment on the GPU: Fragment / FragmentWithOverhangs of many genes,
// SetEfficiency and NextOverhangs of many overhang sets (DESIGN.md §4 "Fragment").
//
// SetEfficiency (fragment.go:24-38) of a set S multiplies, over the members o in set order,
// nCorrect(o) / nTotal(o) where nCorrect(o) = mm[o,o] and nTotal(o) = sum over o2 in S of
// mm[o,o2] + mm[o,RC(o2)].  mm is non-zero only for the 120 canonical A/C/G/T 4-mers (keys), so a member
// enters the sums only through key(o2) and key(RC(o2)), and nTotal(o) = R[key(o)] with
//     R[k] = sum over o2 in S of mm[k, key(o2)] + mm[k, key(RC(o2))]      (a missing key adds 0).
// Appending a candidate x gives R'[k] = R[k] + mm[k, key(x)] + mm[k, key(RC(x))] for every member, and x's
// own total R'[key(x)], so the efficiency of S + x takes one pass over the keyed members in set order with
// the same integer totals, the same IEEE divide and the same multiply as the reference: O(m) per candidate
// instead of O(m^2), bit for bit.  Members without a key contribute no factor and are left out of the pass.
//
// Built with -fmad=false: the product is a plain multiply of a quotient, and must stay one.
#include <algorithm>

#include "common.cuh"

namespace pg {
namespace {
#include "fragment_fidelity.inc"

constexpr int kKeys = 120;
constexpr int kWarps = 8;         // warps per CTA
constexpr int kThreads = 32 * kWarps;
constexpr int kOwnKeys = 128;     // per warp: the keyed ends (<= 2) and chosen overhangs (<= 120), or a set's first keys
constexpr int kExShared = 2048;   // keyed excludes held in shared memory; the rest are read from global memory

// A/C/G/T -> 0..3, anything else -1 (the sequence is upper-cased before it gets here)
__host__ __device__ __forceinline__ int base2(uint32_t b) { return b == 'A' ? 0 : b == 'C' ? 1 : b == 'G' ? 2 : b == 'T' ? 3 : -1; }

// the 2-bit code of a 4-byte word (first byte in the low bits, first base in the high code bits), or -1
__host__ __device__ __forceinline__ int code_of(uint32_t w) {
    int c = 0;
    for (int i = 0; i < 4; ++i) {
        const int b = base2((w >> (8 * i)) & 0xff);
        if (b < 0) return -1;
        c = c << 2 | b;
    }
    return c;
}

// code of ReverseComplement: complement each base (b ^ 3) and reverse their order
__host__ __device__ __forceinline__ int rc_code(int c) {
    return ((c & 3) ^ 3) << 6 | (((c >> 2) & 3) ^ 3) << 4 | (((c >> 4) & 3) ^ 3) << 2 | ((c >> 6) ^ 3);
}

// transform.ReverseComplement of a 4-byte word
__host__ __device__ __forceinline__ uint32_t rc_word(uint32_t w) {
    return (uint32_t)complement(w >> 24) | (uint32_t)complement((w >> 16) & 0xff) << 8 | (uint32_t)complement((w >> 8) & 0xff) << 16 |
           (uint32_t)complement(w & 0xff) << 24;
}

__device__ __forceinline__ uint32_t upper(uint32_t b) { return b - 'a' < 26u ? b - 32 : b; }

// the upper-cased 4 bytes s[q .. q + 4)
__device__ __forceinline__ uint32_t word_at(const uint8_t *s, int64_t q) {
    return upper(s[q]) | upper(s[q + 1]) << 8 | upper(s[q + 2]) << 16 | upper(s[q + 3]) << 24;
}

// candidate idx of NextOverhangs' loops over {A, T, G, C} at each position -> its code (A0 C1 G2 T3)
__device__ __forceinline__ int nest_code(int idx) {
    int c = 0;
    for (int q = 3; q >= 0; --q) c = c << 2 | ((4 - ((idx >> (2 * q)) & 3)) & 3);
    return c;
}

__device__ __forceinline__ uint8_t base_char(int b) { return b == 0 ? 'A' : b == 1 ? 'C' : b == 2 ? 'G' : 'T'; }

__device__ __forceinline__ bool bit(const uint32_t *mask, int c) { return mask[c >> 5] >> (c & 31) & 1; }

__device__ __forceinline__ bool in_list(const uint32_t *list, uint64_t n, uint32_t w) {
    for (uint64_t j = 0; j < n; ++j)
        if (list[j] == w) return true;
    return false;
}

struct Fidelity {
    uint16_t mm[kKeys * kKeys];
    int16_t key[256];  // code -> key, or -1
};

struct WarpState {
    long long R[kKeys];
    uint32_t mask[8];  // A/C/G/T codes that equal a member or a member's reverse complement
    uint8_t keys[kOwnKeys];
};

// Multiplies e by every keyed member's factor, in order, with x (key kx, RC key krx; -1 for none) appended
__device__ __forceinline__ double product(double e, const uint8_t *keys, uint64_t n, const long long *R, const uint16_t *mm, int kx, int krx) {
    for (uint64_t j = 0; j < n; ++j) {
        const int k = keys[j];
        const uint16_t *row = mm + k * kKeys;
        const long long nc = row[k];
        const long long nt = R[k] + (kx >= 0 ? row[kx] : 0) + (krx >= 0 ? row[krx] : 0);
        if (nt != nc) e = e * ((double)nc / (double)nt);
    }
    return e;
}

// x's own factor (key kx >= 0, RC key krx) as the last member of S + x
__device__ __forceinline__ double own_factor(double e, const long long *R, const uint16_t *mm, int kx, int krx) {
    const uint16_t *row = mm + kx * kKeys;
    const long long nc = row[kx];
    const long long nt = R[kx] + nc + (krx >= 0 ? row[krx] : 0);
    return nt != nc ? e * ((double)nc / (double)nt) : e;
}

// R += the contribution of one member with keys (kx, krx); lanes split the 120 keys
__device__ __forceinline__ void add_to_r(long long *R, const uint16_t *mm, int kx, int krx, int lane) {
    for (int k = lane; k < kKeys; k += 32) R[k] += (kx >= 0 ? mm[k * kKeys + kx] : 0) + (krx >= 0 ? mm[k * kKeys + krx] : 0);
}

__device__ void load_fidelity(Fidelity &sh, const uint8_t *g) {
    const uint32_t *src = (const uint32_t *)g;
    uint32_t *dst = (uint32_t *)&sh;
    for (uint32_t i = threadIdx.x; i < sizeof(Fidelity) / 4; i += blockDim.x) dst[i] = src[i];
}

// A member joins a gene's set: R, the mask of its A/C/G/T code and its reverse complement's, or (for any
// other word) the word and its reverse complement at the end of the warp's list.  Returns its key, or -1.
__device__ __forceinline__ int join(WarpState &w, const Fidelity &fid, uint32_t word, uint32_t *other, uint64_t &n_other, int lane) {
    const int c = code_of(word);
    const int kx = c >= 0 ? fid.key[c] : -1, krx = c >= 0 ? fid.key[rc_code(c)] : -1;
    add_to_r(w.R, fid.mm, kx, krx, lane);
    if (lane == 0) {
        if (c >= 0) {
            w.mask[c >> 5] |= 1u << (c & 31);
            w.mask[rc_code(c) >> 5] |= 1u << (rc_code(c) & 31);
        } else {
            other[n_other] = word;
            other[n_other + 1] = rc_word(word);
        }
    }
    if (c < 0) n_other += 2;
    __syncwarp();
    return kx;
}

// One warp per gene, grid-stride.  Per gene the warp keeps R, the exclusion mask and the keyed ends and
// chosen overhangs in shared memory; words of members that are not A/C/G/T 4-mers (and their reverse
// complements) go to the warp's slot of global scratch, which holds 2 (2 + steps) of them.
__global__ void __launch_bounds__(kThreads, 3) fragment_kernel(FragmentArgs a) {
    __shared__ Fidelity fid;
    __shared__ long long r_ex[kKeys];
    __shared__ uint32_t ex_mask[8], inc_mask[8];
    __shared__ uint8_t ex_keys[kExShared];
    __shared__ WarpState ws[kWarps];
    load_fidelity(fid, a.fid);
    for (int i = threadIdx.x; i < kKeys; i += blockDim.x) r_ex[i] = a.r_ex[i];
    if (threadIdx.x < 8) { ex_mask[threadIdx.x] = a.ex_mask[threadIdx.x]; inc_mask[threadIdx.x] = a.inc_mask[threadIdx.x]; }
    const uint64_t n_ex_sh = std::min<uint64_t>(a.n_ex_keys, kExShared);
    for (uint64_t i = threadIdx.x; i < n_ex_sh; i += blockDim.x) ex_keys[i] = a.ex_keys[i];
    __syncthreads();
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    WarpState &w = ws[wid];
    const uint64_t gw = (uint64_t)blockIdx.x * kWarps + wid, nw = (uint64_t)gridDim.x * kWarps;
    uint32_t *other = a.scratch + gw * a.slot_words;
    const uint16_t *mm = fid.mm;
    for (uint64_t item = gw; item < a.n; item += nw) {
        const uint8_t *s = a.seqs + a.off[item];
        const int64_t L = (int64_t)(a.off[item + 1] - a.off[item]);
        bool high = false;
        for (int64_t p = lane; p < L; p += 32) high |= s[p] >= 0x80;
        int32_t status = PG_ITEM_OK;
        double eff = 0;
        int64_t emin = 0, emax = 0;
        uint64_t nend = 0;
        uint64_t *ends = a.ends + a.ends_off[item];
        if (__any_sync(0xffffffffu, high)) {
            status = PG_ITEM_UNSUPPORTED;
        } else if (L < 4) {
            status = PG_ITEM_PANIC;  // sequence[:4]
        } else {
            // the starting set: [seq[:4], seq[L-4:]] ++ excludes (R and the masks of the excludes come in a)
            for (int k = lane; k < kKeys; k += 32) w.R[k] = r_ex[k];
            if (lane < 8) w.mask[lane] = ex_mask[lane];
            __syncwarp();
            int n_end_keys = 0, n_chosen = 0;
            uint64_t n_other = 0;
            for (int e = 0; e < 2; ++e) {
                const int kx = join(w, fid, word_at(s, e ? L - 4 : 0), other, n_other, lane);
                if (kx >= 0) {
                    if (lane == 0) w.keys[n_end_keys] = (uint8_t)kx;
                    ++n_end_keys;
                }
            }
            __syncwarp();
            int64_t base = 0, len = L, mn = a.min_size, mx = a.max_size;
            for (;;) {
                if (len < mx) {  // the last fragment: efficiency of the whole set
                    if (lane == 0) ends[nend] = (uint64_t)L;
                    ++nend;
                    double e = product(1.0, w.keys, n_end_keys, w.R, mm, -1, -1);
                    e = product(e, ex_keys, n_ex_sh, w.R, mm, -1, -1);
                    e = product(e, a.ex_keys + n_ex_sh, a.n_ex_keys - n_ex_sh, w.R, mm, -1, -1);
                    eff = product(e, w.keys + 2, n_chosen, w.R, mm, -1, -1);
                    break;
                }
                if (mn > mx) { status = PG_ITEM_FRAGMENT_MIN_GT_MAX; emin = mn; emax = mx; break; }
                if (mn < 12) { status = PG_ITEM_FRAGMENT_MIN_LT_12; emin = mn; emax = mx; break; }
                if (len < 2 * mx) {  // end game (fragment.go:125-133); carries into every later step
                    const int64_t d = mx - mn;
                    const int64_t buf = std::min<int64_t>((len + d) / 2, mx);
                    mn = buf - d;
                    mx = buf;
                }
                double best = 0;
                int64_t best_pos = 0;
                for (int64_t o0 = 0; o0 <= mx - mn; o0 += 32) {
                    const int64_t o = o0 + lane, pos = mx - o;
                    double v = -1;
                    if (o <= mx - mn) {
                        const uint32_t x = word_at(s, base + pos - 4);
                        const int c = code_of(x);
                        bool skip;
                        if (c >= 0) {
                            skip = bit(w.mask, c) || (a.has_include && !bit(inc_mask, c)) || rc_code(c) == c;
                        } else {
                            skip = in_list(a.ex_other, a.n_ex_other, x) || in_list(other, n_other, x) ||
                                   (a.has_include && !in_list(a.inc_other, a.n_inc_other, x)) || rc_word(x) == x;
                        }
                        if (!skip) {
                            const int kx = c >= 0 ? fid.key[c] : -1, krx = c >= 0 ? fid.key[rc_code(c)] : -1;
                            double e = product(1.0, w.keys, n_end_keys, w.R, mm, kx, krx);
                            e = product(e, ex_keys, n_ex_sh, w.R, mm, kx, krx);
                            e = product(e, a.ex_keys + n_ex_sh, a.n_ex_keys - n_ex_sh, w.R, mm, kx, krx);
                            e = product(e, w.keys + 2, n_chosen, w.R, mm, kx, krx);
                            v = kx >= 0 ? own_factor(e, w.R, mm, kx, krx) : e;
                        }
                    }
                    double m = v;
                    for (int sh = 16; sh; sh >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, sh));
                    if (m > best) {  // the first strict improvement: ties go to the larger position, the lower lane
                        const int win = __ffs(__ballot_sync(0xffffffffu, v == m)) - 1;
                        best = m;
                        best_pos = mx - (o0 + win);
                    }
                }
                if (best_pos == 0) { status = PG_ITEM_FRAGMENT_NO_POSITION; break; }
                if (lane == 0) ends[nend] = (uint64_t)(base + best_pos);
                ++nend;
                // a chosen keyed overhang is never chosen again (it joins the mask with its reverse complement),
                // so at most 120 of them join the key list
                const int kx = join(w, fid, word_at(s, base + best_pos - 4), other, n_other, lane);
                if (kx >= 0) {
                    if (lane == 0) w.keys[2 + n_chosen] = (uint8_t)kx;
                    ++n_chosen;
                }
                __syncwarp();
                base += best_pos - 4;
                len -= best_pos - 4;
            }
        }
        if (lane == 0) {
            a.status[item] = status;
            a.eff[item] = status == PG_ITEM_OK ? eff : 0.0;
            a.err_min[item] = emin;
            a.err_max[item] = emax;
            a.n_ends[item] = status == PG_ITEM_OK ? nend : 0;
        }
        __syncwarp();
    }
}

// One warp per set, grid-stride: R, the mask and the set's keys (the first kOwnKeys in shared memory, the
// rest in the warp's slot of global scratch), then SetEfficiency, or NextOverhangs with lanes over the 256
// candidates.  S + x and S + RC(x) give every member the same total, so one pass serves both.
__global__ void __launch_bounds__(kThreads) overhang_sets_kernel(SetArgs a) {
    __shared__ Fidelity fid;
    __shared__ WarpState ws[kWarps];
    load_fidelity(fid, a.fid);
    __syncthreads();
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    WarpState &w = ws[wid];
    const uint64_t gw = (uint64_t)blockIdx.x * kWarps + wid, nw = (uint64_t)gridDim.x * kWarps;
    uint8_t *spill = a.scratch + gw * a.slot_bytes;
    const uint16_t *mm = fid.mm;
    for (uint64_t set = gw; set < a.n_sets; set += nw) {
        for (int k = lane; k < kKeys; k += 32) w.R[k] = 0;
        if (lane < 8) w.mask[lane] = 0;
        __syncwarp();
        uint64_t nk = 0;
        for (uint64_t j = a.set_off[a.first + set]; j < a.set_off[a.first + set + 1]; ++j) {
            const uint64_t b = a.ov_off[j];
            if (a.ov_off[j + 1] - b != 4) continue;  // only 4-byte members can be keys, or equal a candidate
            const uint32_t x = a.ov[b] | a.ov[b + 1] << 8 | a.ov[b + 2] << 16 | (uint32_t)a.ov[b + 3] << 24;
            const int c = code_of(x);
            if (c < 0) continue;
            const int kx = fid.key[c], krx = fid.key[rc_code(c)];
            add_to_r(w.R, mm, kx, krx, lane);
            if (lane == 0) {
                w.mask[c >> 5] |= 1u << (c & 31);
                const int r = rc_code(c);
                w.mask[r >> 5] |= 1u << (r & 31);
                if (kx >= 0) {
                    if (nk < kOwnKeys) w.keys[nk] = (uint8_t)kx;
                    else spill[nk - kOwnKeys] = (uint8_t)kx;
                }
            }
            if (kx >= 0) ++nk;
            __syncwarp();
        }
        const uint64_t nsh = std::min<uint64_t>(nk, kOwnKeys);
        if (!a.next) {
            if (lane == 0) a.eff[set] = product(product(1.0, w.keys, nsh, w.R, mm, -1, -1), spill, nk - nsh, w.R, mm, -1, -1);
        } else {
            uint32_t count = 0;
            for (int r0 = 0; r0 < 256; r0 += 32) {
                const int idx = r0 + lane;  // the reference's nesting: A, T, G, C at every position
                const int c = nest_code(idx);
                const bool keep = !bit(w.mask, c) && rc_code(c) != c;
                const unsigned ball = __ballot_sync(0xffffffffu, keep);
                if (keep) {
                    const int kx = fid.key[c], krx = fid.key[rc_code(c)];
                    const double e = product(product(1.0, w.keys, nsh, w.R, mm, kx, krx), spill, nk - nsh, w.R, mm, kx, krx);
                    const double strand = kx >= 0 ? own_factor(e, w.R, mm, kx, krx) : e;
                    const double comp = krx >= 0 ? own_factor(e, w.R, mm, krx, kx) : e;
                    const uint64_t slot = set * 256 + count + __popc(ball & ((1u << lane) - 1));
                    a.eff[slot] = (strand + comp) / 2;
                    for (int q = 0; q < 4; ++q) a.cands[4 * slot + q] = base_char((c >> (6 - 2 * q)) & 3);
                }
                count += __popc(ball);
            }
            if (lane == 0) a.n_cands[set] = count;
        }
        __syncwarp();
    }
}

// ends of item i from its worst-case region to its place in the compacted list; one warp per item
__global__ void compact_ends_kernel(const uint64_t *region, const uint64_t *region_off, const uint64_t *n_ends, const uint64_t *out_off, uint64_t n,
                                    uint64_t *out) {
    const uint64_t i = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (i >= n) return;
    for (uint64_t j = threadIdx.x & 31; j < n_ends[i]; j += 32) out[out_off[i] + j] = region[region_off[i] + j];
}

int grid_for(uint64_t items, uint64_t slot_bytes, uint64_t budget) {
    uint64_t warps = std::min<uint64_t>(items, (uint64_t)sm_count() * 3 * kWarps);
    if (slot_bytes) warps = std::min<uint64_t>(warps, std::max<uint64_t>(budget / slot_bytes, 1));
    return (int)std::max<uint64_t>((warps + kWarps - 1) / kWarps, 1);
}
}  // namespace

uint64_t fragment_max_ends(uint64_t len) { return len >= 12 ? (len - 12) / 2 + 2 : 1; }

FragmentHost fragment_host(const uint8_t *ex, const uint64_t *ex_off, uint64_t n_ex, const uint8_t *inc, const uint64_t *inc_off, uint64_t n_inc) {
    FragmentHost h;
    h.fid.resize(sizeof(Fidelity));
    Fidelity &f = *(Fidelity *)h.fid.data();
    for (int i = 0; i < kKeys; ++i)
        for (int j = 0; j < kKeys; ++j) f.mm[i * kKeys + j] = k_fidelity_counts[i][j];
    std::fill(f.key, f.key + 256, (int16_t)-1);
    for (int k = 0; k < kKeys; ++k) {
        const char *s = k_fidelity_keys[k];
        f.key[code_of((uint8_t)s[0] | (uint8_t)s[1] << 8 | (uint8_t)s[2] << 16 | (uint32_t)(uint8_t)s[3] << 24)] = (int16_t)k;
    }
    h.r_ex.assign(kKeys, 0);
    h.ex_mask.assign(8, 0);
    h.inc_mask.assign(8, 0);
    auto scan = [&](const uint8_t *b, const uint64_t *off, uint64_t n, std::vector<uint32_t> &mask, std::vector<uint32_t> &other, bool exclude) {
        for (uint64_t i = 0; i < n; ++i) {
            if (off[i + 1] - off[i] != 4) continue;  // only a 4-byte member can equal a candidate or be a key
            const uint8_t *p = b + off[i];
            const uint32_t x = p[0] | p[1] << 8 | p[2] << 16 | (uint32_t)p[3] << 24;
            const int c = code_of(x);
            if (c < 0) {
                other.push_back(x);
                other.push_back(rc_word(x));
                continue;
            }
            mask[c >> 5] |= 1u << (c & 31);
            mask[rc_code(c) >> 5] |= 1u << (rc_code(c) & 31);
            if (!exclude) continue;
            const int kx = f.key[c], krx = f.key[rc_code(c)];
            for (int k = 0; k < kKeys; ++k) h.r_ex[k] += (kx >= 0 ? f.mm[k * kKeys + kx] : 0) + (krx >= 0 ? f.mm[k * kKeys + krx] : 0);
            if (kx >= 0) h.ex_keys.push_back((uint8_t)kx);
        }
    };
    scan(ex, ex_off, n_ex, h.ex_mask, h.ex_other, true);
    scan(inc, inc_off, n_inc, h.inc_mask, h.inc_other, false);
    return h;
}

int launch_fragment(FragmentArgs a, uint64_t max_len, uint64_t scratch_budget, StreamScratch &tmp, cudaStream_t st) {
    if (a.n == 0) return PG_OK;
    a.slot_words = 2 * (fragment_max_ends(max_len) + 2);
    const int grid = grid_for(a.n, a.slot_words * 4, scratch_budget);
    PG_CUDA(tmp.alloc((uint8_t **)&a.scratch, (uint64_t)grid * kWarps * a.slot_words * 4));
    fragment_kernel<<<grid, kThreads, 0, st>>>(a);
    PG_LAUNCH_CHECK("fragment_kernel");
    return PG_OK;
}

int launch_fragment_compact(const uint64_t *d_region, const uint64_t *d_region_off, const uint64_t *d_n_ends, const uint64_t *d_out_off, uint64_t n,
                            uint64_t *d_out, cudaStream_t st) {
    if (n == 0) return PG_OK;
    compact_ends_kernel<<<(unsigned)((n + 7) / 8), 256, 0, st>>>(d_region, d_region_off, d_n_ends, d_out_off, n, d_out);
    PG_LAUNCH_CHECK("fragment_compact_ends_kernel");
    return PG_OK;
}

int launch_overhang_sets(SetArgs a, uint64_t max_keys, uint64_t scratch_budget, StreamScratch &tmp, cudaStream_t st) {
    if (a.n_sets == 0) return PG_OK;
    a.slot_bytes = max_keys > kOwnKeys ? max_keys - kOwnKeys : 0;
    const int grid = grid_for(a.n_sets, a.slot_bytes, scratch_budget);
    PG_CUDA(tmp.alloc(&a.scratch, std::max<uint64_t>((uint64_t)grid * kWarps * a.slot_bytes, 16)));
    overhang_sets_kernel<<<grid, kThreads, 0, st>>>(a);
    PG_LAUNCH_CHECK(a.next ? "overhang_sets_kernel(next)" : "overhang_sets_kernel(efficiency)");
    return PG_OK;
}

}  // namespace pg
