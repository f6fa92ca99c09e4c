/*
 * oracle/pair_oracle.c -- pair-list driver over the restated po_sw_score / po_nw_score (TEST
 * INFRASTRUCTURE: the oracle of tests/test_gpu_align_pairs.py and the CPU arm of
 * tools/bench_align_pairs.py; see oracle/poly_oracle.h).  The reference has no pair API: a caller loops
 * over the pairs and calls align.SmithWaterman / align.NeedlemanWunsch once per pair, so that is what
 * each worker does here.  Workers take blocks of pairs from a shared counter (at most 64, and small
 * enough for every thread to get several), so that a few long pairs do not leave threads idle.
 */
#include <stdint.h>

#include "parallel.h"
#include "poly_oracle.h"

typedef struct {
    int global;
    const uint8_t *a, *b;
    const uint64_t *off_a, *off_b;
    const uint32_t *pair_a, *pair_b;
    const int16_t *lut_a, *lut_b;
    const int64_t *table;
    int n_b;
    int64_t gap;
    int64_t *score;
    int32_t *err_code;
    int64_t *err_pos;
    int rc;
} pair_job;

static void pair_one(void *p, uint64_t k) {
    pair_job *j = (pair_job *)p;
    const uint32_t ia = j->pair_a[k], ib = j->pair_b[k];
    const uint8_t *a = j->a + j->off_a[ia], *b = j->b + j->off_b[ib];
    const int64_t la = (int64_t)(j->off_a[ia + 1] - j->off_a[ia]), lb = (int64_t)(j->off_b[ib + 1] - j->off_b[ib]);
    int64_t sc = 0, mr = 0, mc = 0, ep = 0;
    int32_t ec = 0;
    const int rc = j->global ? po_nw_score(a, la, b, lb, j->lut_a, j->lut_b, j->table, j->n_b, j->gap, &sc, &ec, &ep)
                             : po_sw_score(a, la, b, lb, j->lut_a, j->lut_b, j->table, j->n_b, j->gap, &sc, &mr, &mc, &ec, &ep);
    if (rc != PO_OK) __atomic_store_n(&j->rc, rc, __ATOMIC_RELAXED);
    j->score[k] = sc;
    j->err_code[k] = ec;
    j->err_pos[k] = ep;
}

/* pair k: po_sw_score (global = 0) or po_nw_score (global = 1) of a = A[pair_a[k]], b = B[pair_b[k]];
 * indices must be in range (the caller checks them).  Returns PO_OK or the first failing code. */
int po_pair_scores(int global, const uint8_t *a, const uint64_t *off_a, const uint8_t *b, const uint64_t *off_b, const uint32_t *pair_a,
                   const uint32_t *pair_b, uint64_t n, const int16_t *lut_a, const int16_t *lut_b, const int64_t *table, int n_b,
                   int64_t gap, int nthreads, int64_t *score, int32_t *err_code, int64_t *err_pos) {
    if (nthreads < 1) nthreads = 1;
    uint64_t block = n / ((uint64_t)nthreads * 16);
    block = block < 1 ? 1 : block > 64 ? 64 : block;
    pair_job j = {global, a, b, off_a, off_b, pair_a, pair_b, lut_a, lut_b, table, n_b, gap, score, err_code, err_pos, PO_OK};
    const int rc = po_parallel_for(n, nthreads, block, pair_one, &j);
    return rc != PO_OK ? rc : j.rc;
}
