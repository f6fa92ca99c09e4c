// sw_align.cu -- Smith-Waterman WITH the aligned strings for short queries: the part of
// /root/reference/search/align/align.go:171-232 that K4 (sw_score.cu) leaves out -- the
// first-max position in the reference's row-major order (align.go:197-201) and the traceback
// (align.go:205-229: diagonal, then "up" (a consumed, '-' in B), then "left"; strings built by
// prepending).  SURVEY.md 8f.1 ("next").
//
// One thread per query, DP column in registers (queries <= 64 cells, 32-bit scores), given the
// best score B from the score kernel:
//   sweep 1  locate the first cell with H == B in the reference's visiting order
//            (stringA outer): smallest a-index, then smallest b-index;
//   sweep 2  recompute the DP up to the end column, storing the last W columns in a global ring
//            ([slot][row][query]: coalesced across the warp);
//   walk     trace back from (end row, end column) through the ring until H == 0, writing the two
//            strings reversed, then reverse them in place.
// A path that leaves the W-column window is reported (status 2) and the host re-runs that query
// with W = template length.
#include <algorithm>
#include <vector>

#include "align_core.cuh"

namespace pg {

namespace {

constexpr int AL_THREADS = 128;
constexpr int AL_TCHUNK = 4096;

struct AlignParams {
    const uint8_t *q;
    const uint64_t *qoff;
    const uint32_t *qlist;  // optional list of query indices (retries); nullptr = [q_first, q_first + n)
    uint64_t q_first, n;
    const uint8_t *t;
    uint64_t tlen;
    int query_is_a, n_q, n_t, gap;
    int global;           // 1: Needleman-Wunsch traceback (align.go:136-166) instead of Smith-Waterman
    uint32_t W;           // ring columns
    uint64_t out_stride;  // bytes per aligned string
};

template <int ROWS, bool GLOBAL>
__global__ void __launch_bounds__(AL_THREADS)
sw_align_kernel(AlignParams p, const int16_t *__restrict__ lut_q, const int16_t *__restrict__ lut_t,
                const int *__restrict__ tab, const int64_t *__restrict__ score, const int32_t *__restrict__ err,
                int *__restrict__ ring, uint8_t *__restrict__ out_a, uint8_t *__restrict__ out_b,
                uint32_t *__restrict__ out_len, int32_t *__restrict__ status) {
    extern __shared__ __align__(16) uint8_t sm[];
    uint8_t *s_tidx = sm;                                              // [AL_TCHUNK]
    int16_t *s_lut_t = reinterpret_cast<int16_t *>(sm + AL_TCHUNK);    // [256]
    int *s_tab = reinterpret_cast<int *>(sm + AL_TCHUNK + 512);        // [n_q * n_t]
    const uint32_t tid = threadIdx.x;
    for (int i = tid; i < p.n_q * p.n_t; i += AL_THREADS) s_tab[i] = tab[i];
    for (int i = tid; i < 256; i += AL_THREADS) s_lut_t[i] = lut_t[i];
    __syncthreads();

    const uint64_t b = (uint64_t)blockIdx.x * AL_THREADS + tid;  // slot in this launch
    const bool in_range = b < p.n;
    const uint64_t qi = in_range ? (p.qlist ? p.qlist[b] : p.q_first + b) : 0;
    uint64_t qbeg = 0;
    uint32_t qlen = 0;
    int B = 0;
    bool active = false;
    if (in_range) {
        qbeg = p.qoff[qi];
        qlen = (uint32_t)(p.qoff[qi + 1] - qbeg);
        B = err[qi] ? 0 : (int)score[qi];
        // SW: B == 0 means maxScore was never updated and the traceback loop does not run.
        // NW: the loop runs while both indices are positive (align.go:141).
        active = GLOBAL ? (!err[qi] && qlen > 0 && p.tlen > 0) : B > 0;
        if (!active) {
            out_len[qi] = 0;
            status[qi] = PG_ITEM_OK;
        }
    }
    int qrow[ROWS];
#pragma unroll
    for (int i = 0; i < ROWS; ++i) {
        qrow[i] = 0;
        if (active && i < (int)qlen) {
            const int ix = lut_q[__ldg(p.q + qbeg + i)];
            qrow[i] = ix < 0 ? 0 : ix * p.n_t;
        }
    }
    const int gap = p.gap;

    // ---- sweep 1: first cell with H == B in the reference's order ---------------------
    int col[ROWS];
#pragma unroll
    for (int i = 0; i < ROWS; ++i) col[i] = 0;
    uint32_t bq = 0xffffffffu, bt = 0xffffffffu;  // 1-based query / template index of the end cell
    if (GLOBAL) { bq = qlen; bt = (uint32_t)p.tlen; }  // NW starts at (len(a), len(b))
    for (uint64_t t0 = 0; !GLOBAL && t0 < p.tlen; t0 += AL_TCHUNK) {
        const uint32_t tc = (uint32_t)min((uint64_t)AL_TCHUNK, p.tlen - t0);
        __syncthreads();
        for (uint32_t j = tid; j < tc; j += AL_THREADS) {
            const int ix = s_lut_t[__ldg(p.t + t0 + j)];
            s_tidx[j] = ix < 0 ? 0 : (uint8_t)ix;
        }
        __syncthreads();
        if (active) {
            for (uint32_t j = 0; j < tc; ++j) {
                const int tj = s_tidx[j];
                int diag = 0, up = 0;
#pragma unroll
                for (int i = 0; i < ROWS; ++i) {
                    if (i < (int)qlen) {
                        const int old = col[i];
                        const int v = sw_cell<int, false>(diag, s_tab[qrow[i] + tj], old, up, gap);
                        if (v == B) {
                            const uint32_t cq = i + 1, ct = (uint32_t)(t0 + j) + 1;
                            // stringA outer: query_is_a -> (query, template) lexicographic, else (template, query)
                            const bool better = p.query_is_a ? (cq < bq || (cq == bq && ct < bt))
                                                             : (ct < bt || (ct == bt && cq < bq));
                            if (better) { bq = cq; bt = ct; }
                        }
                        diag = old;
                        up = v;
                        col[i] = v;
                    }
                }
            }
        }
    }

    // ---- sweep 2: recompute up to column bt, keep the last W columns in the ring ------
    const uint32_t W = p.W;
    const uint32_t first_kept = active ? (bt > W ? bt - W + 1 : 1) : 0;  // 1-based template index
#pragma unroll
    for (int i = 0; i < ROWS; ++i) col[i] = GLOBAL ? (i + 1) * gap : 0;
    int edge = 0;  // NW: H[0][j-1]
    for (uint64_t t0 = 0; t0 < p.tlen; t0 += AL_TCHUNK) {
        const uint32_t tc = (uint32_t)min((uint64_t)AL_TCHUNK, p.tlen - t0);
        __syncthreads();
        for (uint32_t j = tid; j < tc; j += AL_THREADS) {
            const int ix = s_lut_t[__ldg(p.t + t0 + j)];
            s_tidx[j] = ix < 0 ? 0 : (uint8_t)ix;
        }
        __syncthreads();
        if (active && t0 < bt) {
            const uint32_t jend = (uint32_t)min((uint64_t)tc, (uint64_t)bt - t0);
            for (uint32_t j = 0; j < jend; ++j) {
                const int tj = s_tidx[j];
                const uint32_t ct = (uint32_t)(t0 + j) + 1;
                const bool keep = ct >= first_kept;
                int *slot = ring + ((uint64_t)(ct % W) * ROWS) * p.n + b;
                int diag = GLOBAL ? edge : 0, up = GLOBAL ? edge + gap : 0;
                if (GLOBAL) edge += gap;
#pragma unroll
                for (int i = 0; i < ROWS; ++i) {
                    if (i < (int)qlen) {
                        const int old = col[i];
                        const int v = sw_cell<int, GLOBAL>(diag, s_tab[qrow[i] + tj], old, up, gap);
                        if (keep) slot[(uint64_t)i * p.n] = v;
                        diag = old;
                        up = v;
                        col[i] = v;
                    }
                }
            }
        }
    }
    if (!active) return;

    // ---- walk: align.go:205-229 ----------------------------------------------------------
    auto H = [&](uint32_t cq, uint32_t ct, bool &outside) -> int {
        if (cq == 0 || ct == 0) return GLOBAL ? (int)(cq + ct) * gap : 0;  // NW gap ramps on the first row / column
        if (ct < first_kept) { outside = true; return 0; }
        return ring[((uint64_t)(ct % W) * ROWS + (cq - 1)) * p.n + b];
    };
    uint8_t *oa = out_a + qi * p.out_stride, *ob = out_b + qi * p.out_stride;
    uint32_t cq = bq, ct = bt, len = 0;
    bool outside = false, overflow = false;
    int h = H(cq, ct, outside);
    while ((GLOBAL ? (cq > 0 && ct > 0) : h > 0) && !outside) {
        const uint8_t qc = __ldg(p.q + qbeg + cq - 1), tc_ = __ldg(p.t + ct - 1);
        const int lq = lut_q[qc], lt = lut_t[tc_];
        const int sc = (lq < 0 || lt < 0) ? 0 : s_tab[lq * p.n_t + lt];
        const int hd = H(cq - 1, ct - 1, outside);
        // "up" = previous index of stringA, "left" = previous index of stringB
        const int h_up = p.query_is_a ? H(cq - 1, ct, outside) : H(cq, ct - 1, outside);
        const int h_left = p.query_is_a ? H(cq, ct - 1, outside) : H(cq - 1, ct, outside);
        if (outside) break;
        uint8_t ca, cb;
        // trace_step's choice, written out: calling trace_step and trace_finish changes this kernel's machine code
        if (h == hd + sc) {                 // align.go:215-219
            ca = p.query_is_a ? qc : tc_;
            cb = p.query_is_a ? tc_ : qc;
            --cq; --ct;
        } else if (h == h_up + gap) {       // align.go:220-223: stringA consumed, '-' in B
            ca = p.query_is_a ? qc : tc_;
            cb = '-';
            if (p.query_is_a) --cq; else --ct;
        } else if (GLOBAL || h == h_left + gap) {  // align.go:224-228 (SW) / the plain else of align.go:155-159 (NW)
            ca = '-';
            cb = p.query_is_a ? tc_ : qc;
            if (p.query_is_a) --ct; else --cq;
        } else {
            break;  // unreachable for a max of the three (the reference would not terminate)
        }
        trace_put(oa, ob, p.out_stride, ca, cb, len, overflow);
        h = H(cq, ct, outside);
    }
    if (outside) {
        status[qi] = 2;  // window too small: host retries with W = template length
        return;
    }
    const uint32_t n_written = min(len, (uint32_t)p.out_stride);  // trace_finish, written out as above
    for (uint32_t x = 0; x < n_written / 2; ++x) {
        uint8_t t1 = oa[x]; oa[x] = oa[n_written - 1 - x]; oa[n_written - 1 - x] = t1;
        t1 = ob[x]; ob[x] = ob[n_written - 1 - x]; ob[n_written - 1 - x] = t1;
    }
    out_len[qi] = len;
    status[qi] = overflow ? PG_ITEM_UNSUPPORTED : PG_ITEM_OK;
}

template <int ROWS, bool GLOBAL>
int run_align(const AlignParams &p, const AlignTables<int> &d, const int64_t *d_score, const int32_t *d_err, uint8_t *d_a,
              uint8_t *d_b, uint32_t *d_len, int32_t *d_status, cudaStream_t st) {
    if (p.n == 0) return PG_OK;
    StreamScratch tmp(st);
    int *d_ring = nullptr;
    PG_CUDA(tmp.alloc(&d_ring, (size_t)p.W * ROWS * p.n));
    const size_t smem = AL_TCHUNK + 512 + (size_t)p.n_q * p.n_t * sizeof(int);
    return launch_smem(sw_align_kernel<ROWS, GLOBAL>, (unsigned)((p.n + AL_THREADS - 1) / AL_THREADS), AL_THREADS, smem, st,
                       GLOBAL ? "nw_align_kernel" : "sw_align_kernel", p, d.lut_row, d.lut_col, d.tab, d_score, d_err, d_ring, d_a,
                       d_b, d_len, d_status);
}

}  // namespace

// Device-resident driver: scores (K4) first, then the traceback kernel in batches; queries whose
// path leaves the default window are re-run with a full-length window.
int launch_sw_align(const uint8_t *d_q, const uint64_t *d_qoff, uint64_t nq, uint64_t max_qlen, const uint8_t *d_t, uint64_t tlen,
                    int query_is_a, const AlignScoring &s, int64_t *d_score, int32_t *d_err, int64_t *d_errpos, uint8_t *d_align_a,
                    uint8_t *d_align_b, uint64_t out_stride, uint32_t *d_len, int32_t *d_status, cudaStream_t st) {
    if (nq == 0) return PG_OK;
    if (max_qlen > 64) {  // both strings may be long: whole matrix in HBM, literal traceback (sw_align_long.cu)
        int rc = launch_sw_score(d_q, d_qoff, nq, max_qlen, d_t, tlen, query_is_a, s, d_score, d_err, d_errpos, st);
        if (rc != PG_OK) return rc;
        return launch_sw_align_long(d_q, d_qoff, nq, max_qlen, d_t, tlen, query_is_a, s, d_score, d_err, d_align_a, d_align_b,
                                    out_stride, d_len, d_status, st);
    }
    if (score_bound(s.global, s.abs_max(), s.gap, 64, 64 + tlen) >= SCORE32_LIMIT) {
        set_error("aligned strings need scores that fit 32 bits");
        return PG_ERR_UNSUPPORTED;
    }
    int rc = launch_sw_score(d_q, d_qoff, nq, max_qlen, d_t, tlen, query_is_a, s, d_score, d_err, d_errpos, st);
    if (rc != PG_OK) return rc;

    AlignParams p;
    p.q = d_q; p.qoff = d_qoff; p.qlist = nullptr; p.t = d_t; p.tlen = tlen; p.query_is_a = query_is_a;
    p.n_q = query_is_a ? s.n_a : s.n_b;
    p.n_t = query_is_a ? s.n_b : s.n_a;
    p.gap = (int)s.gap;
    p.global = s.global;
    p.out_stride = out_stride;
    StreamScratch tmp(st);
    AlignTables<int> d;  // the query symbol on the table's rows
    if ((rc = upload_tables<int>(s, {query_is_a != 0}, false, tmp, st, &d)) != PG_OK) return rc;

    const int rows = max_qlen <= 32 ? 32 : 64;
    auto run = [&]() {
        return s.global ? (rows == 32 ? run_align<32, true>(p, d, d_score, d_err, d_align_a, d_align_b, d_len, d_status, st)
                                      : run_align<64, true>(p, d, d_score, d_err, d_align_a, d_align_b, d_len, d_status, st))
                        : (rows == 32 ? run_align<32, false>(p, d, d_score, d_err, d_align_a, d_align_b, d_len, d_status, st)
                                      : run_align<64, false>(p, d, d_score, d_err, d_align_a, d_align_b, d_len, d_status, st));
    };
    // NW walks the whole matrix: keep every column
    const uint32_t W0 = s.global ? (uint32_t)std::max<uint64_t>(tlen, 1) : (uint32_t)std::min<uint64_t>(std::max<uint64_t>(tlen, 1), 2 * rows + 32);
    // batches bounded by ~1 GiB of ring
    const uint64_t per = std::max<uint64_t>(1, ((1ull << 30) / ((uint64_t)W0 * rows * 4)));
    for (uint64_t q0 = 0; q0 < nq && rc == PG_OK; q0 += per) {
        p.q_first = q0; p.n = std::min<uint64_t>(per, nq - q0); p.W = W0;
        rc = run();
    }
    // retries with a full-length window (rare: long gap runs)
    if (rc == PG_OK && !s.global && W0 < tlen) {
        std::vector<int32_t> hst(nq);
        PG_CUDA(cudaMemcpyAsync(hst.data(), d_status, nq * 4, cudaMemcpyDeviceToHost, st));
        PG_CUDA(cudaStreamSynchronize(st));
        std::vector<uint32_t> redo;
        for (uint64_t i = 0; i < nq; ++i)
            if (hst[i] == 2) redo.push_back((uint32_t)i);
        if (!redo.empty()) {
            uint32_t *d_list = nullptr;
            PG_CUDA(tmp.alloc(&d_list, redo.size()));
            PG_CUDA(cudaMemcpyAsync(d_list, redo.data(), redo.size() * 4, cudaMemcpyHostToDevice, st));
            const uint64_t per2 = std::max<uint64_t>(1, (1ull << 30) / (tlen * rows * 4));
            for (uint64_t r0 = 0; r0 < redo.size() && rc == PG_OK; r0 += per2) {
                p.qlist = d_list + r0; p.q_first = 0; p.n = std::min<uint64_t>(per2, redo.size() - r0); p.W = (uint32_t)tlen;
                rc = run();
            }
        }
    }
    return rc;
}

}  // namespace pg
