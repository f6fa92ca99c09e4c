// api_align.cu -- the C ABI of poly's align: Smith-Waterman / Needleman-Wunsch scores and aligned strings
// of queries against one template, and of pair lists.
#include <algorithm>
#include <vector>

#include "align_core.cuh"
#include "runtime.cuh"

namespace pg {
namespace {

static int align_score_dev(const AlignScoring &s, const uint8_t *d_queries, const uint64_t *d_q_offsets, uint64_t n_queries,
                           uint64_t max_query_len, const uint8_t *d_templ, uint64_t templ_len, int32_t query_is_a, int64_t *d_score,
                           int32_t *d_err_code, int64_t *d_err_pos, void *stream) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if (s.has_null() || (n_queries && (!d_q_offsets || !d_score))) { set_error("null buffer"); return PG_ERR_ARG; }
    return launch_sw_score(d_queries, d_q_offsets, n_queries, max_query_len, d_templ, templ_len, query_is_a, s, d_score, d_err_code,
                           d_err_pos, (cudaStream_t)stream);
}

static int align_score_host(const AlignScoring &s, const uint8_t *queries, const uint64_t *q_offsets, uint64_t n_queries,
                            const uint8_t *templ, uint64_t templ_len, int32_t query_is_a, int64_t *score, int32_t *err_code,
                            int64_t *err_pos) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if (n_queries == 0) return PG_OK;
    if (!q_offsets || !score || s.has_null()) { set_error("null buffer"); return PG_ERR_ARG; }
    HostCall c;
    const Ragged<uint8_t> q = c.ragged(queries, q_offsets, n_queries);
    const uint8_t *d_t = c.upload(templ, templ_len);
    int64_t *d_sc = c.alloc<int64_t>(n_queries), *d_ep = c.alloc<int64_t>(n_queries);
    int32_t *d_ec = c.alloc<int32_t>(n_queries);
    if ((rc = c.error()) || (rc = launch_sw_score(q.base, q.off, n_queries, q.max_len, d_t, templ_len, query_is_a, s, d_sc, d_ec, d_ep, c.st)))
        return rc;
    c.download(score, d_sc, n_queries);
    c.download(err_code, d_ec, n_queries);
    c.download(err_pos, d_ep, n_queries);
    return c.finish();
}

static int align_strings_host(const AlignScoring &s, const uint8_t *queries, const uint64_t *q_offsets, uint64_t n_queries,
                              const uint8_t *templ, uint64_t templ_len, int32_t query_is_a, int64_t *score, int32_t *err_code,
                              int64_t *err_pos, uint8_t *align_a, uint8_t *align_b, uint64_t out_stride, uint32_t *align_len,
                              int32_t *status) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if (n_queries == 0) return PG_OK;
    if (!q_offsets || !score || s.has_null() || !align_a || !align_b || !align_len || s.n_a <= 0 || s.n_b <= 0) {
        set_error("null buffer");
        return PG_ERR_ARG;
    }
    HostCall c;
    const Ragged<uint8_t> q = c.ragged(queries, q_offsets, n_queries);
    const uint8_t *d_t = c.upload(templ, templ_len);
    int64_t *d_sc = c.alloc<int64_t>(n_queries), *d_ep = c.alloc<int64_t>(n_queries);
    int32_t *d_ec = c.alloc<int32_t>(n_queries);
    uint8_t *d_a = c.alloc<uint8_t>(n_queries * out_stride), *d_b = c.alloc<uint8_t>(n_queries * out_stride);
    uint32_t *d_len = c.alloc<uint32_t>(n_queries, true);
    int32_t *d_st = c.alloc<int32_t>(n_queries, true);
    if ((rc = c.error()) || (rc = launch_sw_align(q.base, q.off, n_queries, q.max_len, d_t, templ_len, query_is_a, s, d_sc, d_ec, d_ep, d_a,
                                                  d_b, out_stride, d_len, d_st, c.st)))
        return rc;
    c.download(score, d_sc, n_queries);
    c.download(err_code, d_ec, n_queries);
    c.download(err_pos, d_ep, n_queries);
    c.download(align_a, d_a, n_queries * out_stride);
    c.download(align_b, d_b, n_queries * out_stride);
    c.download(align_len, d_len, n_queries);
    c.download(status, d_st, n_queries);
    return c.finish();
}

// device bytes per pair of a host pair call: indices, outputs and the classify / list scratch
static constexpr uint64_t PAIR_BYTES = 4 + 4 + 8 + 4 + 8 + 1 + 4;
static constexpr uint64_t PAIR_GROUP_BYTES = 1ull << 30;

static int align_pairs_host(const AlignScoring &s, bool strings, const uint8_t *seqs_a, const uint64_t *offsets_a, uint64_t n_seqs_a,
                            const uint8_t *seqs_b, const uint64_t *offsets_b, uint64_t n_seqs_b, const uint32_t *pair_a,
                            const uint32_t *pair_b, uint64_t n_pairs, int64_t *score, int32_t *err_code, int64_t *err_pos,
                            uint8_t *align_a, uint8_t *align_b, uint64_t out_stride, uint32_t *align_len, int32_t *status) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if (n_pairs == 0) return PG_OK;
    if (!offsets_a || !offsets_b || !pair_a || !pair_b || !score || s.has_null() ||
        (strings && (!align_a || !align_b || !align_len))) {
        set_error("null buffer");
        return PG_ERR_ARG;
    }
    // the whole call is checked before anything is uploaded or launched
    uint64_t set_max = 0;
    if ((rc = check_ragged(offsets_a, n_seqs_a, &set_max)) != PG_OK || (rc = check_ragged(offsets_b, n_seqs_b, &set_max)) != PG_OK) return rc;
    // the longest a and b the pairs reference: a long sequence no pair uses widens neither the score type nor any scratch
    uint64_t max_la = 0, max_lb = 0;
    for (uint64_t k = 0; k < n_pairs; ++k) {
        if (pair_a[k] >= n_seqs_a || pair_b[k] >= n_seqs_b) {
            set_error("pair %llu = (%u, %u) is out of range (%llu, %llu sequences)", (unsigned long long)k, pair_a[k], pair_b[k],
                      (unsigned long long)n_seqs_a, (unsigned long long)n_seqs_b);
            return PG_ERR_ARG;
        }
        max_la = std::max(max_la, offsets_a[pair_a[k] + 1] - offsets_a[pair_a[k]]);
        max_lb = std::max(max_lb, offsets_b[pair_b[k] + 1] - offsets_b[pair_b[k]]);
    }
    HostCall c;
    const Ragged<uint8_t> A = c.ragged(seqs_a, offsets_a, n_seqs_a);
    const bool same = seqs_a == seqs_b && offsets_a == offsets_b && n_seqs_a == n_seqs_b;
    const Ragged<uint8_t> B = same ? A : c.ragged(seqs_b, offsets_b, n_seqs_b);
    if ((rc = c.sync()) != PG_OK) return rc;  // the sets are resident: what is free now bounds a group
    size_t free_b = 0, total_b = 0;
    PG_CUDA(cudaMemGetInfo(&free_b, &total_b));
    // half of the free memory (the rest for the long-pair rows and the aligned-string matrices), at most 1 GiB
    const uint64_t per_pair = PAIR_BYTES + (strings ? 2 * out_stride + 8 : 0);
    const uint64_t budget = group_budget(std::min<uint64_t>(PAIR_GROUP_BYTES, free_b / 2));
    const uint64_t group = std::min<uint64_t>(n_pairs, std::max<uint64_t>(1, budget / per_pair));
    uint32_t *d_pa = c.alloc<uint32_t>(group), *d_pb = c.alloc<uint32_t>(group);
    int64_t *d_sc = c.alloc<int64_t>(group), *d_ep = c.alloc<int64_t>(group);
    int32_t *d_ec = c.alloc<int32_t>(group);
    uint8_t *d_oa = nullptr, *d_ob = nullptr;
    uint32_t *d_len = nullptr;
    int32_t *d_st = nullptr;
    if (strings) {
        d_oa = c.alloc<uint8_t>(group * out_stride);
        d_ob = c.alloc<uint8_t>(group * out_stride);
        d_len = c.alloc<uint32_t>(group);
        d_st = c.alloc<int32_t>(group);
    }
    for (uint64_t g0 = 0; g0 < n_pairs; g0 += group) {
        const uint64_t ng = std::min(group, n_pairs - g0);
        c.put(d_pa, pair_a + g0, ng);
        c.put(d_pb, pair_b + g0, ng);
        if ((rc = c.error()) || (rc = launch_sw_score_pairs(A.base, A.off, n_seqs_a, max_la, B.base, B.off, n_seqs_b, max_lb, d_pa, d_pb, ng,
                                                            s, d_sc, d_ec, d_ep, c.st)))
            return rc;
        if (strings) {  // matrices sized by this group's longest a and b
            uint64_t ga = 0, gb = 0;
            for (uint64_t k = g0; k < g0 + ng; ++k) {
                ga = std::max(ga, offsets_a[pair_a[k] + 1] - offsets_a[pair_a[k]]);
                gb = std::max(gb, offsets_b[pair_b[k] + 1] - offsets_b[pair_b[k]]);
            }
            if ((rc = launch_sw_align_long(A.base, A.off, ng, ga, B.base, gb, 1, s, d_sc, d_ec, d_oa, d_ob, out_stride, d_len, d_st, c.st,
                                           B.off, d_pa, d_pb)))
                return rc;
        }
        c.download(score + g0, d_sc, ng);
        if (err_code) c.download(err_code + g0, d_ec, ng);
        if (err_pos) c.download(err_pos + g0, d_ep, ng);
        if (strings) {
            c.download(align_a + g0 * out_stride, d_oa, ng * out_stride);
            c.download(align_b + g0 * out_stride, d_ob, ng * out_stride);
            c.download(align_len + g0, d_len, ng);
            if (status) c.download(status + g0, d_st, ng);
        }
    }
    return c.finish();
}

static int score_pairs_dev(const AlignScoring &s, const uint8_t *d_seqs_a, const uint64_t *d_offsets_a, uint64_t n_seqs_a,
                           uint64_t max_len_a, const uint8_t *d_seqs_b, const uint64_t *d_offsets_b, uint64_t n_seqs_b,
                           uint64_t max_len_b, const uint32_t *d_pair_a, const uint32_t *d_pair_b, uint64_t n_pairs, int64_t *d_score,
                           int32_t *d_err_code, int64_t *d_err_pos, void *stream) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if (s.has_null() || (n_pairs && (!d_offsets_a || !d_offsets_b || !d_pair_a || !d_pair_b || !d_score))) {
        set_error("null buffer");
        return PG_ERR_ARG;
    }
    return launch_sw_score_pairs(d_seqs_a, d_offsets_a, n_seqs_a, max_len_a, d_seqs_b, d_offsets_b, n_seqs_b, max_len_b, d_pair_a,
                                 d_pair_b, n_pairs, s, d_score, d_err_code, d_err_pos, (cudaStream_t)stream);
}

}  // namespace
}  // namespace pg

using namespace pg;

extern "C" {

// ---------------------------------------------------------------------------------
// Smith-Waterman score
// ---------------------------------------------------------------------------------
int pg_sw_score_batch_dev(const uint8_t *d_queries, const uint64_t *d_q_offsets, uint64_t n_queries,
                          uint64_t max_query_len, const uint8_t *d_templ, uint64_t templ_len,
                          int32_t query_is_a, const int16_t *lut_a_host, const int16_t *lut_b_host,
                          const int64_t *table_host, int32_t n_a, int32_t n_b, int64_t gap,
                          int64_t *d_score, int32_t *d_err_code, int64_t *d_err_pos, void *stream) {
    return align_score_dev({lut_a_host, lut_b_host, table_host, n_a, n_b, gap, 0}, d_queries, d_q_offsets, n_queries, max_query_len,
                           d_templ, templ_len, query_is_a, d_score, d_err_code, d_err_pos, stream);
}
int pg_nw_score_batch_dev(const uint8_t *d_queries, const uint64_t *d_q_offsets, uint64_t n_queries,
                          uint64_t max_query_len, const uint8_t *d_templ, uint64_t templ_len,
                          int32_t query_is_a, const int16_t *lut_a_host, const int16_t *lut_b_host,
                          const int64_t *table_host, int32_t n_a, int32_t n_b, int64_t gap,
                          int64_t *d_score, int32_t *d_err_code, int64_t *d_err_pos, void *stream) {
    return align_score_dev({lut_a_host, lut_b_host, table_host, n_a, n_b, gap, 1}, d_queries, d_q_offsets, n_queries, max_query_len,
                           d_templ, templ_len, query_is_a, d_score, d_err_code, d_err_pos, stream);
}
int pg_sw_score_batch(const uint8_t *queries, const uint64_t *q_offsets, uint64_t n_queries,
                      const uint8_t *templ, uint64_t templ_len, int32_t query_is_a,
                      const int16_t *lut_a, const int16_t *lut_b, const int64_t *table, int32_t n_a,
                      int32_t n_b, int64_t gap, int64_t *score, int32_t *err_code, int64_t *err_pos) {
    return align_score_host({lut_a, lut_b, table, n_a, n_b, gap, 0}, queries, q_offsets, n_queries, templ, templ_len, query_is_a, score,
                            err_code, err_pos);
}
int pg_nw_score_batch(const uint8_t *queries, const uint64_t *q_offsets, uint64_t n_queries,
                      const uint8_t *templ, uint64_t templ_len, int32_t query_is_a,
                      const int16_t *lut_a, const int16_t *lut_b, const int64_t *table, int32_t n_a,
                      int32_t n_b, int64_t gap, int64_t *score, int32_t *err_code, int64_t *err_pos) {
    return align_score_host({lut_a, lut_b, table, n_a, n_b, gap, 1}, queries, q_offsets, n_queries, templ, templ_len, query_is_a, score,
                            err_code, err_pos);
}

int pg_sw_align_batch(const uint8_t *queries, const uint64_t *q_offsets, uint64_t n_queries,
                      const uint8_t *templ, uint64_t templ_len, int32_t query_is_a,
                      const int16_t *lut_a, const int16_t *lut_b, const int64_t *table, int32_t n_a,
                      int32_t n_b, int64_t gap, int64_t *score, int32_t *err_code, int64_t *err_pos,
                      uint8_t *align_a, uint8_t *align_b, uint64_t out_stride, uint32_t *align_len,
                      int32_t *status) {
    return align_strings_host({lut_a, lut_b, table, n_a, n_b, gap, 0}, queries, q_offsets, n_queries, templ, templ_len, query_is_a, score,
                              err_code, err_pos, align_a, align_b, out_stride, align_len, status);
}
int pg_nw_align_batch(const uint8_t *queries, const uint64_t *q_offsets, uint64_t n_queries,
                      const uint8_t *templ, uint64_t templ_len, int32_t query_is_a,
                      const int16_t *lut_a, const int16_t *lut_b, const int64_t *table, int32_t n_a,
                      int32_t n_b, int64_t gap, int64_t *score, int32_t *err_code, int64_t *err_pos,
                      uint8_t *align_a, uint8_t *align_b, uint64_t out_stride, uint32_t *align_len,
                      int32_t *status) {
    return align_strings_host({lut_a, lut_b, table, n_a, n_b, gap, 1}, queries, q_offsets, n_queries, templ, templ_len, query_is_a, score,
                              err_code, err_pos, align_a, align_b, out_stride, align_len, status);
}

// ---------------------------------------------------------------------------------
// Smith-Waterman / Needleman-Wunsch over pair lists
// ---------------------------------------------------------------------------------
int pg_sw_score_pairs(const uint8_t *seqs_a, const uint64_t *offsets_a, uint64_t n_seqs_a, const uint8_t *seqs_b,
                      const uint64_t *offsets_b, uint64_t n_seqs_b, const uint32_t *pair_a, const uint32_t *pair_b, uint64_t n_pairs,
                      const int16_t *lut_a, const int16_t *lut_b, const int64_t *table, int32_t n_a, int32_t n_b, int64_t gap,
                      int64_t *score, int32_t *err_code, int64_t *err_pos) {
    return align_pairs_host({lut_a, lut_b, table, n_a, n_b, gap, 0}, false, seqs_a, offsets_a, n_seqs_a, seqs_b, offsets_b, n_seqs_b,
                            pair_a, pair_b, n_pairs, score, err_code, err_pos, nullptr, nullptr, 0, nullptr, nullptr);
}
int pg_nw_score_pairs(const uint8_t *seqs_a, const uint64_t *offsets_a, uint64_t n_seqs_a, const uint8_t *seqs_b,
                      const uint64_t *offsets_b, uint64_t n_seqs_b, const uint32_t *pair_a, const uint32_t *pair_b, uint64_t n_pairs,
                      const int16_t *lut_a, const int16_t *lut_b, const int64_t *table, int32_t n_a, int32_t n_b, int64_t gap,
                      int64_t *score, int32_t *err_code, int64_t *err_pos) {
    return align_pairs_host({lut_a, lut_b, table, n_a, n_b, gap, 1}, false, seqs_a, offsets_a, n_seqs_a, seqs_b, offsets_b, n_seqs_b,
                            pair_a, pair_b, n_pairs, score, err_code, err_pos, nullptr, nullptr, 0, nullptr, nullptr);
}
int pg_sw_score_pairs_dev(const uint8_t *d_seqs_a, const uint64_t *d_offsets_a, uint64_t n_seqs_a, uint64_t max_len_a,
                          const uint8_t *d_seqs_b, const uint64_t *d_offsets_b, uint64_t n_seqs_b, uint64_t max_len_b,
                          const uint32_t *d_pair_a, const uint32_t *d_pair_b, uint64_t n_pairs, const int16_t *lut_a_host,
                          const int16_t *lut_b_host, const int64_t *table_host, int32_t n_a, int32_t n_b, int64_t gap,
                          int64_t *d_score, int32_t *d_err_code, int64_t *d_err_pos, void *stream) {
    return score_pairs_dev({lut_a_host, lut_b_host, table_host, n_a, n_b, gap, 0}, d_seqs_a, d_offsets_a, n_seqs_a, max_len_a, d_seqs_b,
                           d_offsets_b, n_seqs_b, max_len_b, d_pair_a, d_pair_b, n_pairs, d_score, d_err_code, d_err_pos, stream);
}
int pg_nw_score_pairs_dev(const uint8_t *d_seqs_a, const uint64_t *d_offsets_a, uint64_t n_seqs_a, uint64_t max_len_a,
                          const uint8_t *d_seqs_b, const uint64_t *d_offsets_b, uint64_t n_seqs_b, uint64_t max_len_b,
                          const uint32_t *d_pair_a, const uint32_t *d_pair_b, uint64_t n_pairs, const int16_t *lut_a_host,
                          const int16_t *lut_b_host, const int64_t *table_host, int32_t n_a, int32_t n_b, int64_t gap,
                          int64_t *d_score, int32_t *d_err_code, int64_t *d_err_pos, void *stream) {
    return score_pairs_dev({lut_a_host, lut_b_host, table_host, n_a, n_b, gap, 1}, d_seqs_a, d_offsets_a, n_seqs_a, max_len_a, d_seqs_b,
                           d_offsets_b, n_seqs_b, max_len_b, d_pair_a, d_pair_b, n_pairs, d_score, d_err_code, d_err_pos, stream);
}
int pg_sw_align_pairs(const uint8_t *seqs_a, const uint64_t *offsets_a, uint64_t n_seqs_a, const uint8_t *seqs_b,
                      const uint64_t *offsets_b, uint64_t n_seqs_b, const uint32_t *pair_a, const uint32_t *pair_b, uint64_t n_pairs,
                      const int16_t *lut_a, const int16_t *lut_b, const int64_t *table, int32_t n_a, int32_t n_b, int64_t gap,
                      int64_t *score, int32_t *err_code, int64_t *err_pos, uint8_t *align_a, uint8_t *align_b, uint64_t out_stride,
                      uint32_t *align_len, int32_t *status) {
    return align_pairs_host({lut_a, lut_b, table, n_a, n_b, gap, 0}, true, seqs_a, offsets_a, n_seqs_a, seqs_b, offsets_b, n_seqs_b,
                            pair_a, pair_b, n_pairs, score, err_code, err_pos, align_a, align_b, out_stride, align_len, status);
}
int pg_nw_align_pairs(const uint8_t *seqs_a, const uint64_t *offsets_a, uint64_t n_seqs_a, const uint8_t *seqs_b,
                      const uint64_t *offsets_b, uint64_t n_seqs_b, const uint32_t *pair_a, const uint32_t *pair_b, uint64_t n_pairs,
                      const int16_t *lut_a, const int16_t *lut_b, const int64_t *table, int32_t n_a, int32_t n_b, int64_t gap,
                      int64_t *score, int32_t *err_code, int64_t *err_pos, uint8_t *align_a, uint8_t *align_b, uint64_t out_stride,
                      uint32_t *align_len, int32_t *status) {
    return align_pairs_host({lut_a, lut_b, table, n_a, n_b, gap, 1}, true, seqs_a, offsets_a, n_seqs_a, seqs_b, offsets_b, n_seqs_b,
                            pair_a, pair_b, n_pairs, score, err_code, err_pos, align_a, align_b, out_stride, align_len, status);
}

}  // extern "C"
