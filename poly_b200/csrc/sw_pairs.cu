// sw_pairs.cu -- K4 pairs: Smith-Waterman / Needleman-Wunsch scores of a list of (a, b) pairs that
// index two ragged sequence sets (align.go:100-134,166 and 171-203, one call per pair).
//
// Layout.  Per pair the DP holds the SHORTER string on the rows and streams the longer one as
// columns: the SW maximum and the NW corner are the same for the transposed matrix.  A strip of
// 32*R rows is swept by one warp as an anti-diagonal wavefront: lane l owns R consecutive rows in
// registers, processes column t - l at step t, and hands its bottom row's H and the column on to
// lane l + 1 (the H by __shfl_up_sync, the column through a 64-entry per-warp ring in shared memory).
// Each cell is three DPX add-max instructions (__viaddmax_s32) and one max.
//   short pairs (shorter side <= 256): one warp per pair, R in {1, 2, 4, 5, 8} picked per pair;
//   long pairs: one CTA of PL_WARPS warps per pair; warp w sweeps strips w, w + PL_WARPS, ...; a
//            strip reads the bottom row of the strip above from global scratch (one row per warp,
//            linear in the longer length) as that strip publishes its progress in shared memory.
// Pairs are classified on the device (pair_classify_kernel: index and length checks, the first
// bad symbol of each string, the empty cases), counted per class and compacted, long pairs
// biggest-first by log2(cells); the long kernel takes them from an atomic work counter.  No host
// round trip, so the _dev entry points only enqueue work.
#include <algorithm>
#include <type_traits>

#include "align_core.cuh"

namespace pg {

namespace {

constexpr int PS_WARPS = 4;          // warps per CTA of the short-pair kernel (one pair per warp)
constexpr int PL_WARPS = 8;          // warps per CTA of the long-pair kernel (one pair per CTA)
constexpr int PL_R = 8;              // rows per lane in the long kernel: strips of 256 rows
constexpr int N_SHORT = 5;           // short classes: R = 1, 2, 4, 5, 8
constexpr int N_CLASS = N_SHORT + 64;  // + one long class per log2(la * lb), biggest first
constexpr uint8_t CLS_DONE = 0xff;   // error, empty string or bad index: the classify kernel wrote the result
constexpr int RING = 64;

__host__ __device__ constexpr int short_rows(int c) { return c == 0 ? 1 : c == 1 ? 2 : c == 2 ? 4 : c == 3 ? 5 : 8; }

struct PairParams {
    const uint8_t *a;
    const uint64_t *aoff;
    uint64_t na, max_la;
    const uint8_t *b;
    const uint64_t *boff;
    uint64_t nb, max_lb;
    const uint32_t *pa, *pb;
    uint64_t n;
    int n_a, n_b;
    int min_class;  // 64-bit scores: every short pair takes the R = 8 kernel
};

// Device parameter block: the two byte LUTs, then the table twice: [n_a + 1][n_b] (rows = a) and
// [n_b + 1][n_a] (rows = b), each with a last row of NegBig for rows beyond the shorter string.
template <typename T>
struct Blob {
    const int16_t *lut_a, *lut_b;
    const T *tab_ab, *tab_ba;
};

// Per-call control block on the device
struct Ctl {
    unsigned int count[N_CLASS];
    unsigned int start[N_CLASS];
    unsigned int cursor[N_CLASS];
    unsigned int n_long, long_start, work;
};

// first i < len with lut[s[i]] < 0, or -1 (all lanes of the warp return it)
__device__ __forceinline__ int64_t warp_first_bad(const uint8_t *s, uint64_t len, const int16_t *lut) {
    const int lane = threadIdx.x & 31;
    for (uint64_t base = 0; base < len; base += 32) {
        const uint64_t i = base + lane;
        const bool bad = i < len && lut[s[i]] < 0;
        const unsigned m = __ballot_sync(0xffffffffu, bad);
        if (m) return (int64_t)(base + __ffs(m) - 1);
    }
    return -1;
}

__device__ __forceinline__ int class_of(uint64_t m, uint64_t cells, int min_class) {
    if (m > 32 * PL_R) return N_SHORT + __clzll((long long)cells);  // bigger cells -> smaller class
    return max(min_class, m <= 32 ? 0 : m <= 64 ? 1 : m <= 128 ? 2 : m <= 160 ? 3 : 4);
}

// One warp per pair: index/length checks, errors in the reference's order, empty strings; the rest
// are counted per class.
__global__ void __launch_bounds__(256)
pair_classify_kernel(PairParams p, const int16_t *__restrict__ g_lut_a, const int16_t *__restrict__ g_lut_b, int64_t gap, int global,
                     int64_t *__restrict__ score, int32_t *__restrict__ err, int64_t *__restrict__ errpos, uint8_t *__restrict__ cls,
                     Ctl *__restrict__ ctl) {
    __shared__ int16_t lut_a[256], lut_b[256];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) { lut_a[i] = g_lut_a[i]; lut_b[i] = g_lut_b[i]; }
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const uint64_t nw = (uint64_t)gridDim.x * (blockDim.x / 32);
    for (uint64_t k = (uint64_t)blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32; k < p.n; k += nw) {
        const uint32_t ia = p.pa[k], ib = p.pb[k];
        int32_t ec = 0;
        int64_t ep = -1, sc = 0;
        uint8_t c = CLS_DONE;
        uint64_t la = 0, lb = 0;
        if (ia < p.na && ib < p.nb) {
            const uint64_t a0 = p.aoff[ia], b0 = p.boff[ib];
            la = p.aoff[ia + 1] - a0;
            lb = p.boff[ib + 1] - b0;
            if (la > p.max_la || lb > p.max_lb) {
                ec = PG_PAIR_OUT_OF_RANGE;
            } else if (la > 0 && lb > 0) {
                const int64_t bad_a = warp_first_bad(p.a + a0, la, lut_a), bad_b = warp_first_bad(p.b + b0, lb, lut_b);
                first_error(bad_a, bad_b, ec, ep);
                if (!ec) c = (uint8_t)class_of(min(la, lb), la * lb, p.min_class);
            } else if (global) {
                sc = (int64_t)(la + lb) * gap;  // a pure gap ramp (align.go:115-122,166)
            }
        } else {
            ec = PG_PAIR_OUT_OF_RANGE;
        }
        if (lane == 0) {
            if (c == CLS_DONE) score[k] = sc;
            if (err) err[k] = ec;
            if (errpos) errpos[k] = ep;
            cls[k] = c;
            if (c != CLS_DONE) atomicAdd(&ctl->count[c], 1u);
        }
    }
}

__global__ void pair_scan_kernel(Ctl *ctl) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    unsigned int s = 0;
    for (int c = 0; c < N_CLASS; ++c) {
        ctl->start[c] = ctl->cursor[c] = s;
        s += ctl->count[c];
    }
    ctl->long_start = ctl->start[N_SHORT];
    ctl->n_long = s - ctl->long_start;
    ctl->work = 0;
}

__global__ void pair_scatter_kernel(uint64_t n, const uint8_t *__restrict__ cls, Ctl *__restrict__ ctl, uint32_t *__restrict__ list) {
    for (uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (uint64_t)gridDim.x * blockDim.x) {
        const uint8_t c = cls[k];
        if (c != CLS_DONE) list[atomicAdd(&ctl->cursor[c], 1u)] = (uint32_t)k;
    }
}

// A pair as the DP sees it: S (m symbols) on the rows, L (n symbols) on the columns
template <typename T>
struct PairView {
    const uint8_t *S, *L;
    uint32_t m, n;
    const int16_t *lut_row, *lut_col;
    const T *tab;  // [rows: S symbol or the NegBig row][n_col]
    int n_row, n_col;
};

template <typename T>
__device__ __forceinline__ PairView<T> view_of(const PairParams &p, const Blob<T> &bl, uint32_t k) {
    const uint32_t ia = p.pa[k], ib = p.pb[k];
    const uint64_t a0 = p.aoff[ia], b0 = p.boff[ib];
    const uint32_t la = (uint32_t)(p.aoff[ia + 1] - a0), lb = (uint32_t)(p.boff[ib + 1] - b0);
    PairView<T> v;
    if (la <= lb) {
        v.S = p.a + a0; v.m = la; v.L = p.b + b0; v.n = lb;
        v.lut_row = bl.lut_a; v.lut_col = bl.lut_b; v.tab = bl.tab_ab; v.n_row = p.n_a; v.n_col = p.n_b;
    } else {
        v.S = p.b + b0; v.m = lb; v.L = p.a + a0; v.n = la;
        v.lut_row = bl.lut_b; v.lut_col = bl.lut_a; v.tab = bl.tab_ba; v.n_row = p.n_b; v.n_col = p.n_a;
    }
    return v;
}

// One warp sweeps rows [row0, row0 + 32 R) of v over all n columns.
//   in_row:  H[row0 - 1][j] written by the strip above (nullptr: the first strip, whose top row is the
//            boundary align.go:120-122); its writer publishes "strip tag << 32 | columns done" at prod.
//   out_row: where this strip's bottom row goes (nullptr: no strip below); progress is published at mine.
// best: the running SW maximum of this lane's valid rows.  corner: NW H[m-1][n-1] (last strip only).
template <typename T, int R, bool GLOBAL, bool MASK>
__device__ __forceinline__ void sweep(const PairView<T> &v, uint32_t row0, T gap, const T *in_row, T *out_row,
                                      const volatile unsigned long long *prod, unsigned long long prod_tag,
                                      volatile unsigned long long *mine, unsigned long long my_tag, int *ring_col, T *ring_in,
                                      T &best, T &corner) {
    const int lane = threadIdx.x & 31;
    const uint32_t rows = min(v.m - row0, (uint32_t)(32 * R));
    const int used = (int)((rows + R - 1) / R);  // lanes with at least one row
    const int last = used - 1;
    int rowoff[R];
    T H[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
        const uint32_t i = row0 + (uint32_t)lane * R + r;
        rowoff[r] = (i < v.m ? (int)v.lut_row[v.S[i]] : v.n_row) * v.n_col;
        H[r] = GLOBAL ? (T)(i + 1) * gap : (T)0;  // H[i][-1], align.go:115-117
    }
    const int nvalid = (int)min((int64_t)R, max((int64_t)0, (int64_t)v.m - (int64_t)(row0 + (uint32_t)lane * R)));
    T prev_up = GLOBAL ? (T)(row0 + (uint32_t)lane * R) * gap : (T)0;  // H[row0 + lane R - 1][-1]
    const uint32_t steps = v.n + (uint32_t)last;
    for (uint32_t t = 0; t < steps; ++t) {
        if ((t & 31) == 0) {
            __syncwarp();
            const uint32_t j = t + lane;
            ring_col[j & (RING - 1)] = j < v.n ? (int)v.lut_col[v.L[j]] : 0;
            if (in_row) {
                if (lane == 0) {
                    const unsigned long long need = prod_tag | (unsigned long long)min(v.n, t + 32);
                    while (*prod < need) __nanosleep(20);
                    __threadfence_block();
                }
                __syncwarp();
                ring_in[j & (RING - 1)] = j < v.n ? in_row[j] : (T)0;
            }
            if (out_row && lane == last) {  // columns [0, t - last) of the bottom row are stored
                __threadfence_block();
                *mine = my_tag | (unsigned long long)(t > (uint32_t)last ? t - last : 0);
            }
            __syncwarp();
        }
        const T recv = __shfl_up_sync(0xffffffffu, H[R - 1], 1);
        const uint32_t j = t - (uint32_t)lane;
        if (lane <= last && t >= (uint32_t)lane && j < v.n) {
            const T up_in = lane ? recv : (in_row ? ring_in[j & (RING - 1)] : (GLOBAL ? (T)(j + 1) * gap : (T)0));
            T diag = prev_up, up = up_in;
            prev_up = up_in;
            const int cv = ring_col[j & (RING - 1)];
#pragma unroll
            for (int r = 0; r < R; ++r) {
                const T old = H[r];  // H[i][j-1]
                const T x = sw_cell<T, GLOBAL>(diag, v.tab[rowoff[r] + cv], old, up, gap);
                if (!GLOBAL && (!MASK || r < nvalid)) best = x > best ? x : best;  // align.go:197-201
                diag = old;
                up = x;
                H[r] = x;
            }
            if (out_row && lane == last) out_row[j] = H[R - 1];
        }
    }
    if (out_row && lane == last) {
        __threadfence_block();
        *mine = my_tag | (unsigned long long)v.n;
    }
    if (GLOBAL && row0 + 32u * R >= v.m) {  // the strip holding row m - 1
        const int owner = (int)((v.m - 1 - row0) / R), rr = (int)((v.m - 1 - row0) % R);
        T h = 0;
#pragma unroll
        for (int r = 0; r < R; ++r)
            if (r == rr) h = H[r];
        corner = __shfl_sync(0xffffffffu, h, owner);
    }
}

template <typename T>
__device__ __forceinline__ T warp_max(T x) {
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        const T y = __shfl_xor_sync(0xffffffffu, x, o);
        x = y > x ? y : x;
    }
    return x;
}

// the tables in shared memory when they fit (smem_tab), else read through L1
template <typename T>
__device__ __forceinline__ Blob<T> stage_blob(const Blob<T> &g, int n_a, int n_b, bool smem_tab, T *s_tab) {
    Blob<T> b = g;
    if (smem_tab) {
        const int nab = (n_a + 1) * n_b, nba = (n_b + 1) * n_a;
        for (int i = threadIdx.x; i < nab; i += blockDim.x) s_tab[i] = g.tab_ab[i];
        for (int i = threadIdx.x; i < nba; i += blockDim.x) s_tab[nab + i] = g.tab_ba[i];
        b.tab_ab = s_tab;
        b.tab_ba = s_tab + nab;
    }
    __syncthreads();
    return b;
}

// short pairs of class CLS: one warp per pair, grid-stride over the class's list
template <typename T, int R, bool GLOBAL, bool MASK>
__global__ void __launch_bounds__(PS_WARPS * 32, 8)
pair_short_kernel(PairParams p, Blob<T> g, bool smem_tab, T gap, int cls, const Ctl *__restrict__ ctl, const uint32_t *__restrict__ list,
                  int64_t *__restrict__ score) {
    extern __shared__ __align__(16) uint8_t sm[];
    __shared__ int s_ring_col[PS_WARPS][RING];
    const Blob<T> bl = stage_blob<T>(g, p.n_a, p.n_b, smem_tab, reinterpret_cast<T *>(sm));
    const int warp = threadIdx.x / 32;
    const unsigned int cnt = ctl->count[cls], first = ctl->start[cls];
    for (unsigned int k = blockIdx.x * PS_WARPS + warp; k < cnt; k += gridDim.x * PS_WARPS) {
        const uint32_t pair = list[first + k];
        const PairView<T> v = view_of<T>(p, bl, pair);
        T best = 0, corner = 0;
        sweep<T, R, GLOBAL, MASK>(v, 0, gap, nullptr, nullptr, nullptr, 0, nullptr, 0, s_ring_col[warp], nullptr, best, corner);
        best = warp_max<T>(best);
        if ((threadIdx.x & 31) == 0) score[pair] = (int64_t)(GLOBAL ? corner : best);
    }
}

// long pairs: one CTA per pair, biggest first from the work counter; strips of 32 PL_R rows
template <typename T, bool GLOBAL, bool MASK>
__global__ void __launch_bounds__(PL_WARPS * 32)
pair_long_kernel(PairParams p, Blob<T> g, bool smem_tab, T gap, Ctl *__restrict__ ctl, const uint32_t *__restrict__ list,
                 T *__restrict__ scratch, uint64_t row_cap, int64_t *__restrict__ score) {
    extern __shared__ __align__(16) uint8_t sm[];
    __shared__ int s_ring_col[PL_WARPS][RING];
    __shared__ T s_ring_in[PL_WARPS][RING];
    __shared__ unsigned long long s_prog[PL_WARPS];
    __shared__ unsigned int s_item;
    __shared__ unsigned long long s_best;
    __shared__ long long s_corner;
    const Blob<T> bl = stage_blob<T>(g, p.n_a, p.n_b, smem_tab, reinterpret_cast<T *>(sm));
    const int warp = threadIdx.x / 32, lane = threadIdx.x & 31;
    T *rows = scratch + (uint64_t)blockIdx.x * PL_WARPS * row_cap;  // one bottom row per warp
    const unsigned int n_long = ctl->n_long, first = ctl->long_start;
    for (;;) {
        if (threadIdx.x == 0) { s_item = atomicAdd(&ctl->work, 1u); s_best = 0; s_corner = 0; }
        if (lane == 0) s_prog[warp] = 0;
        __syncthreads();
        const unsigned int item = s_item;
        if (item >= n_long) break;
        const uint32_t pair = list[first + item];
        const PairView<T> v = view_of<T>(p, bl, pair);
        const uint32_t strips = (v.m + 32 * PL_R - 1) / (32 * PL_R);
        T best = 0, corner = 0;
        for (uint32_t s = warp; s < strips; s += PL_WARPS) {
            const int pw = (int)((s + PL_WARPS - 1) % PL_WARPS);
            sweep<T, PL_R, GLOBAL, MASK>(v, s * 32 * PL_R, gap, s ? rows + (uint64_t)pw * row_cap : nullptr,
                                         s + 1 < strips ? rows + (uint64_t)warp * row_cap : nullptr, &s_prog[pw],
                                         (unsigned long long)(s - 1) << 32, &s_prog[warp], (unsigned long long)s << 32,
                                         s_ring_col[warp], s_ring_in[warp], best, corner);
            if (GLOBAL && s + 1 == strips && lane == 0) s_corner = (long long)corner;
        }
        if (!GLOBAL) {
            best = warp_max<T>(best);
            if (lane == 0) atomicMax(&s_best, (unsigned long long)(long long)best);  // best >= 0
        }
        __syncthreads();
        if (threadIdx.x == 0) score[pair] = GLOBAL ? (int64_t)s_corner : (int64_t)s_best;
        __syncthreads();
    }
}

template <typename T>
int run_pairs(const PairParams &p0, const AlignScoring &s, int64_t *d_score, int32_t *d_err, int64_t *d_errpos, cudaStream_t st) {
    PairParams p = p0;
    p.min_class = sizeof(T) == 4 ? 0 : N_SHORT - 1;
    const int64_t gap = s.gap;
    const int global = s.global;
    const size_t nab = (size_t)(s.n_a + 1) * s.n_b, nba = (size_t)(s.n_b + 1) * s.n_a;
    StreamScratch tmp(st);
    AlignTables<T> d;  // the LUTs, then the table with a rows and with b rows
    int rc = upload_tables<T>(s, {true, false}, true, tmp, st, &d);
    if (rc != PG_OK) return rc;
    uint8_t *d_cls = nullptr;
    Ctl *d_ctl = nullptr;
    uint32_t *d_list = nullptr;
    PG_CUDA(tmp.alloc(&d_ctl, 1));
    PG_CUDA(tmp.alloc(&d_cls, p.n));
    PG_CUDA(tmp.alloc(&d_list, p.n));
    PG_CUDA(cudaMemsetAsync(d_ctl, 0, sizeof(Ctl), st));
    Blob<T> g;
    g.lut_a = d.lut_row;
    g.lut_b = d.lut_col;
    g.tab_ab = d.tab;
    g.tab_ba = d.tab + nab;
    const size_t tab_bytes = (nab + nba) * sizeof(T);
    const bool smem_tab = tab_bytes <= 48 * 1024;
    const size_t smem = smem_tab ? tab_bytes : 0;

    const int sms = sm_count();
    const unsigned cgrid = (unsigned)std::min<uint64_t>((p.n + 7) / 8, (uint64_t)sms * 16);
    pair_classify_kernel<<<cgrid, 256, 0, st>>>(p, g.lut_a, g.lut_b, gap, global, d_score, d_err, d_errpos, d_cls, d_ctl);
    PG_LAUNCH_CHECK("pair_classify_kernel");
    pair_scan_kernel<<<1, 32, 0, st>>>(d_ctl);
    PG_LAUNCH_CHECK("pair_scan_kernel");
    pair_scatter_kernel<<<(unsigned)std::min<uint64_t>((p.n + 255) / 256, (uint64_t)sms * 8), 256, 0, st>>>(p.n, d_cls, d_ctl, d_list);
    PG_LAUNCH_CHECK("pair_scatter_kernel");

    const bool mask = !global && gap > 0;  // a positive gap can lift the rows beyond the shorter string
    const uint64_t max_m = std::min(p.max_la, p.max_lb);
    auto launch_short = [&](auto rows_tag, int cls) -> int {
        constexpr int R = decltype(rows_tag)::value;
        if constexpr (sizeof(T) == 8 && R != 8) return PG_OK;  // 64-bit scores: R = 8 only
        else {
        if (cls < p.min_class || max_m == 0 || (cls > p.min_class && max_m <= (uint64_t)32 * short_rows(cls - 1))) return PG_OK;  // no pair can be in it
        const unsigned grid = (unsigned)std::min<uint64_t>((p.n + PS_WARPS - 1) / PS_WARPS, (uint64_t)sms * 16);
#define PG_PS(G, M)                                                                                                  \
        do {                                                                                                         \
            int rc = func_smem((const void *)pair_short_kernel<T, R, G, M>, smem);                                   \
            if (rc != PG_OK) return rc;                                                                              \
            pair_short_kernel<T, R, G, M><<<grid, PS_WARPS * 32, smem, st>>>(p, g, smem_tab, (T)gap, cls, d_ctl, d_list, d_score); \
        } while (0)
        if (global) PG_PS(true, false);
        else if (mask) PG_PS(false, true);
        else PG_PS(false, false);
#undef PG_PS
        PG_LAUNCH_CHECK(global ? "nw_pair_short_kernel" : "sw_pair_short_kernel");
        return PG_OK;
        }
    };
    if ((rc = launch_short(std::integral_constant<int, 1>{}, 0)) != PG_OK) return rc;
    if ((rc = launch_short(std::integral_constant<int, 2>{}, 1)) != PG_OK) return rc;
    if ((rc = launch_short(std::integral_constant<int, 4>{}, 2)) != PG_OK) return rc;
    if ((rc = launch_short(std::integral_constant<int, 5>{}, 3)) != PG_OK) return rc;
    if ((rc = launch_short(std::integral_constant<int, 8>{}, 4)) != PG_OK) return rc;

    if (max_m > (uint64_t)32 * PL_R) {  // long pairs are possible
        const uint64_t row_cap = std::max(p.max_la, p.max_lb);
        const void *fn = global ? (const void *)pair_long_kernel<T, true, false>
                                : mask ? (const void *)pair_long_kernel<T, false, true> : (const void *)pair_long_kernel<T, false, false>;
        if ((rc = func_smem(fn, smem)) != PG_OK) return rc;
        int occ = 1;
        PG_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fn, PL_WARPS * 32, smem));
        // one CTA per resident slot, capped so that the boundary rows stay under 1 GiB
        uint64_t ctas = std::min<uint64_t>((uint64_t)sms * std::max(occ, 1), p.n);
        ctas = std::max<uint64_t>(1, std::min<uint64_t>(ctas, (1ull << 30) / ((uint64_t)PL_WARPS * row_cap * sizeof(T))));
        T *d_rows = nullptr;
        while (tmp.alloc(&d_rows, ctas * PL_WARPS * row_cap) != cudaSuccess) {  // fewer CTAs, down to one pair's rows
            cudaGetLastError();
            if (ctas == 1) {
                set_error("pair scratch of %llu bytes does not fit", (unsigned long long)(PL_WARPS * row_cap * sizeof(T)));
                return PG_ERR_NOMEM;
            }
            ctas /= 2;
        }
        if (global)
            pair_long_kernel<T, true, false><<<(unsigned)ctas, PL_WARPS * 32, smem, st>>>(p, g, smem_tab, (T)gap, d_ctl, d_list, d_rows, row_cap, d_score);
        else if (mask)
            pair_long_kernel<T, false, true><<<(unsigned)ctas, PL_WARPS * 32, smem, st>>>(p, g, smem_tab, (T)gap, d_ctl, d_list, d_rows, row_cap, d_score);
        else
            pair_long_kernel<T, false, false><<<(unsigned)ctas, PL_WARPS * 32, smem, st>>>(p, g, smem_tab, (T)gap, d_ctl, d_list, d_rows, row_cap, d_score);
        PG_LAUNCH_CHECK(global ? "nw_pair_long_kernel" : "sw_pair_long_kernel");
    }
    return PG_OK;
}

}  // namespace

int launch_sw_score_pairs(const uint8_t *d_a, const uint64_t *d_aoff, uint64_t na, uint64_t max_la, const uint8_t *d_b,
                          const uint64_t *d_boff, uint64_t nb, uint64_t max_lb, const uint32_t *d_pa, const uint32_t *d_pb,
                          uint64_t n_pairs, const AlignScoring &s, int64_t *d_score, int32_t *d_err, int64_t *d_errpos,
                          cudaStream_t st) {
    int rc = s.check();
    if (rc != PG_OK) return rc;
    if (n_pairs == 0) return PG_OK;
    if (n_pairs > 0xffffffffull || max_la > 0xffffffffull || max_lb > 0xffffffffull) {
        set_error("pair lists are limited to 2^32 - 1 pairs and sequences to 2^32 - 1 symbols");
        return PG_ERR_ARG;
    }
    PairParams p;
    p.a = d_a; p.aoff = d_aoff; p.na = na; p.max_la = max_la;
    p.b = d_b; p.boff = d_boff; p.nb = nb; p.max_lb = max_lb;
    p.pa = d_pa; p.pb = d_pb; p.n = n_pairs; p.n_a = s.n_a; p.n_b = s.n_b; p.min_class = 0;
    // the longest a and b of the call
    if (score_bound(s.global, s.abs_max(), s.gap, std::min(max_la, max_lb), max_la + max_lb) < SCORE32_LIMIT)
        return run_pairs<int>(p, s, d_score, d_err, d_errpos, st);
    return run_pairs<long long>(p, s, d_score, d_err, d_errpos, st);
}

}  // namespace pg
