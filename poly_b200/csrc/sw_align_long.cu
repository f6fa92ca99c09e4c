// sw_align_long.cu -- aligned strings of align.SmithWaterman / align.NeedlemanWunsch
// (/root/reference/search/align/align.go:100-166, 171-232) when BOTH strings are longer than the 64
// symbols the register-column kernel (sw_align.cu) holds.  Like the reference it keeps the whole
// (len(a)+1) x (len(b)+1) matrix (align.go:104-110, 175-178) -- here in HBM -- so the traceback is the
// reference's literal walk.  One CTA per pair:
//   fill   anti-diagonal wavefront (cells of one diagonal are independent), one CTA barrier per
//          diagonal; Smith-Waterman also records the first cell (row-major, stringA outer) that holds
//          the best score B, which the score kernel computed before (align.go:197-201);
//   walk   one thread follows align.go:141-160 / 209-229 (diagonal > up > left), writes the strings
//          reversed and flips them.
// Generality path (memory-bound on the matrix, 4 bytes per cell); scores must fit 32 bits.
#include <algorithm>

#include "align_core.cuh"

namespace pg {

namespace {

constexpr int ALL_THREADS = 256;

struct LongParams {
    const uint8_t *q;
    const uint64_t *qoff;
    uint64_t q_first, n;
    const uint8_t *t;
    uint64_t tlen;
    int query_is_a, n_b, gap;
    uint64_t out_stride;
    uint64_t cells_per_pair;  // (max_qlen + 1) * (tlen + 1): stride of a pair's matrix
    const uint64_t *toff;     // non-null: item k is query pq[k] against template pt[k] of (t, toff)
    const uint32_t *pq, *pt;
};

template <bool GLOBAL>
__global__ void __launch_bounds__(ALL_THREADS)
align_long_kernel(LongParams p, const int16_t *__restrict__ lut_a, const int16_t *__restrict__ lut_b,
                  const int *__restrict__ tab, const int64_t *__restrict__ score, const int32_t *__restrict__ err,
                  int *__restrict__ matrices, uint8_t *__restrict__ out_a, uint8_t *__restrict__ out_b,
                  uint32_t *__restrict__ out_len, int32_t *__restrict__ status) {
    __shared__ unsigned long long s_first;  // SW: smallest (i << 32 | j) with H[i][j] == B
    const uint64_t qi = p.q_first + blockIdx.x;  // the item: index of every output
    const uint64_t qs = p.toff ? p.pq[qi] : qi;
    const uint64_t qbeg = p.qoff[qs];
    const uint64_t qlen = p.qoff[qs + 1] - qbeg;
    const uint8_t *tp = p.toff ? p.t + p.toff[p.pt[qi]] : p.t;
    const uint64_t tlen = p.toff ? p.toff[p.pt[qi] + 1] - p.toff[p.pt[qi]] : p.tlen;
    // stringA indexes the rows (outer loop of the reference), stringB the columns
    const uint8_t *A = p.query_is_a ? p.q + qbeg : tp, *B = p.query_is_a ? tp : p.q + qbeg;
    const uint64_t la = p.query_is_a ? qlen : tlen, lb = p.query_is_a ? tlen : qlen;
    const int best = err[qi] ? 0 : (int)score[qi];
    const bool active = GLOBAL ? (!err[qi] && la > 0 && lb > 0) : best > 0;
    if (!active) {  // SW: maxScore never updated, the loop does not run; NW: a string is empty
        if (threadIdx.x == 0) { out_len[qi] = 0; status[qi] = PG_ITEM_OK; }
        return;
    }
    int *M = matrices + (uint64_t)blockIdx.x * p.cells_per_pair;
    const uint64_t W = lb + 1;
    const int gap = p.gap;
    for (uint64_t i = threadIdx.x; i <= la; i += ALL_THREADS) M[i * W] = GLOBAL ? (int)i * gap : 0;       // align.go:115-117
    for (uint64_t j = threadIdx.x; j <= lb; j += ALL_THREADS) M[j] = GLOBAL ? (int)j * gap : 0;           // align.go:120-122
    if (threadIdx.x == 0) s_first = ~0ull;
    __syncthreads();
    for (uint64_t d = 2; d <= la + lb; ++d) {  // cells (i, d - i)
        const uint64_t i_lo = d > lb ? d - lb : 1, i_hi = min(la, d - 1);
        for (uint64_t i = i_lo + threadIdx.x; i <= i_hi; i += ALL_THREADS) {
            const uint64_t j = d - i;
            const int ia = lut_a[A[i - 1]], ib = lut_b[B[j - 1]];
            const int sc = (ia < 0 || ib < 0) ? 0 : tab[ia * p.n_b + ib];  // bad symbols were reported by the score kernel
            const int v = sw_cell<int, GLOBAL>(M[(i - 1) * W + j - 1], sc, M[i * W + j - 1], M[(i - 1) * W + j], gap);
            if (!GLOBAL && v == best) atomicMin(&s_first, ((unsigned long long)i << 32) | (unsigned long long)j);  // align.go:197-201
            M[i * W + j] = v;
        }
        __syncthreads();
    }
    if (threadIdx.x != 0) return;
    uint64_t i = la, j = lb;
    if (!GLOBAL) { i = s_first >> 32; j = s_first & 0xffffffffull; }
    uint8_t *oa = out_a + qi * p.out_stride, *ob = out_b + qi * p.out_stride;
    uint32_t len = 0;
    bool overflow = false;
    while (GLOBAL ? (i > 0 && j > 0) : M[i * W + j] > 0) {
        const int ia = lut_a[A[i - 1]], ib = lut_b[B[j - 1]];
        const int sc = (ia < 0 || ib < 0) ? 0 : tab[ia * p.n_b + ib];
        const TraceStep step = trace_step<GLOBAL>(M[i * W + j], M[(i - 1) * W + j - 1], M[(i - 1) * W + j], M[i * W + j - 1], sc, gap);
        if (step == STEP_DIAG) { trace_put(oa, ob, p.out_stride, A[i - 1], B[j - 1], len, overflow); --i; --j; }
        else if (step == STEP_UP) { trace_put(oa, ob, p.out_stride, A[i - 1], '-', len, overflow); --i; }
        else if (step == STEP_LEFT) { trace_put(oa, ob, p.out_stride, '-', B[j - 1], len, overflow); --j; }
        else break;
    }
    trace_finish(oa, ob, p.out_stride, len, overflow, out_len, status, qi);
}

}  // namespace

// scores (and the reference's first error) come from launch_sw_score; this adds the strings
int launch_sw_align_long(const uint8_t *d_q, const uint64_t *d_qoff, uint64_t nq, uint64_t max_qlen, const uint8_t *d_t,
                         uint64_t tlen, int query_is_a, const AlignScoring &s, const int64_t *d_score, const int32_t *d_err,
                         uint8_t *d_align_a, uint8_t *d_align_b, uint64_t out_stride, uint32_t *d_len, int32_t *d_status,
                         cudaStream_t st, const uint64_t *d_toff, const uint32_t *d_pq, const uint32_t *d_pt) {
    if (nq == 0) return PG_OK;
    if (score_bound(1, s.abs_max(), s.gap, 0, max_qlen + tlen) >= SCORE32_LIMIT) {  // the NW bound for SW too
        set_error("aligned strings need scores that fit 32 bits");
        return PG_ERR_UNSUPPORTED;
    }
    const uint64_t cells = (max_qlen + 1) * (tlen + 1);
    if (cells > (16ull << 30)) {  // 64 GiB of matrix for ONE pair
        set_error("alignment matrix of %llu x %llu cells does not fit", (unsigned long long)max_qlen, (unsigned long long)tlen);
        return PG_ERR_UNSUPPORTED;
    }
    StreamScratch tmp(st);
    AlignTables<int> d;  // a's symbol on the table's rows
    int rc = upload_tables<int>(s, {true}, false, tmp, st, &d);
    if (rc != PG_OK) return rc;
    const uint64_t per = std::max<uint64_t>(1, std::min<uint64_t>((512ull << 20) / cells, 65535));  // <= 2 GiB of matrices per launch
    int *d_m = nullptr;
    PG_CUDA(tmp.alloc(&d_m, std::min(per, nq) * cells));
    LongParams p;
    p.q = d_q; p.qoff = d_qoff; p.t = d_t; p.tlen = tlen; p.query_is_a = query_is_a; p.n_b = s.n_b; p.gap = (int)s.gap;
    p.out_stride = out_stride; p.cells_per_pair = cells;
    p.toff = d_toff; p.pq = d_pq; p.pt = d_pt;
    for (uint64_t q0 = 0; q0 < nq; q0 += per) {
        p.q_first = q0;
        p.n = std::min(per, nq - q0);
        (s.global ? align_long_kernel<true> : align_long_kernel<false>)<<<(unsigned)p.n, ALL_THREADS, 0, st>>>(
            p, d.lut_row, d.lut_col, d.tab, d_score, d_err, d_m, d_align_a, d_align_b, d_len, d_status);
        PG_LAUNCH_CHECK("align_long_kernel");
    }
    return PG_OK;
}

}  // namespace pg
