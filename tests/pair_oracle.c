/*
 * tests/pair_oracle.c -- pair-list driver over the restated po_sw_score / po_nw_score (TEST
 * INFRASTRUCTURE: the oracle of tests/test_gpu_align_pairs.py and the CPU arm of
 * tools/bench_align_pairs.py; see oracle/poly_oracle.h).  The reference has no pair API: a caller loops
 * over the pairs and calls align.SmithWaterman / align.NeedlemanWunsch once per pair, so that is what
 * each worker does here.  Workers take blocks of pairs from a shared counter (at most 64, and small
 * enough for every thread to get several), so that a few long pairs do not leave threads idle.  Linked against oracle/liboracle.so.
 */
#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>

#include "poly_oracle.h"

typedef struct {
    int global;
    const uint8_t *a, *b;
    const uint64_t *off_a, *off_b;
    const uint32_t *pair_a, *pair_b;
    uint64_t n;
    const int16_t *lut_a, *lut_b;
    const int64_t *table;
    int n_b;
    int64_t gap;
    int64_t *score;
    int32_t *err_code;
    int64_t *err_pos;
    uint64_t next, block; /* shared counter, pairs per take */
    int rc;
} pair_job;

static void *pair_worker(void *p) {
    pair_job *j = (pair_job *)p;
    for (;;) {
        const uint64_t lo = __atomic_fetch_add(&j->next, j->block, __ATOMIC_RELAXED);
        if (lo >= j->n) break;
        const uint64_t hi = lo + j->block < j->n ? lo + j->block : j->n;
        for (uint64_t k = lo; k < hi; k++) {
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
    }
    return NULL;
}

/* pair k: po_sw_score (global = 0) or po_nw_score (global = 1) of a = A[pair_a[k]], b = B[pair_b[k]];
 * indices must be in range (the caller checks them).  Returns PO_OK or the first failing code. */
int po_pair_scores(int global, const uint8_t *a, const uint64_t *off_a, const uint8_t *b, const uint64_t *off_b, const uint32_t *pair_a,
                   const uint32_t *pair_b, uint64_t n, const int16_t *lut_a, const int16_t *lut_b, const int64_t *table, int n_b,
                   int64_t gap, int nthreads, int64_t *score, int32_t *err_code, int64_t *err_pos) {
    if (nthreads < 1) nthreads = 1;
    uint64_t block = n / ((uint64_t)nthreads * 16);
    block = block < 1 ? 1 : block > 64 ? 64 : block;
    pair_job j = {global, a, b, off_a, off_b, pair_a, pair_b, n, lut_a, lut_b, table, n_b, gap, score, err_code, err_pos, 0, block, PO_OK};
    pthread_t *th = (pthread_t *)calloc((size_t)nthreads, sizeof(pthread_t));
    if (!th) return -100;
    int started = 0;
    for (int t = 1; t < nthreads; t++)
        if (pthread_create(&th[t], NULL, pair_worker, &j) == 0) started = t;
        else break;
    pair_worker(&j);
    for (int t = 1; t <= started; t++) pthread_join(th[t], NULL);
    free(th);
    return j.rc;
}
