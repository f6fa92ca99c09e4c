/*
 * oracle/parallel.h -- the worker pool of the dynamically scheduled batch drivers (seqhash, clone, fold,
 * fragment and the pair list).  Threads claim `block` items at a time from one shared counter, so a few
 * long items do not leave the others idle.  The calling thread works too.
 *
 * A static function in a header, not an export of liboracle.so, so that each driver's source still compiles
 * into a library that loads on its own, without the rest of the oracle.
 */
#ifndef PO_PARALLEL_H
#define PO_PARALLEL_H
#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>

#include "poly_oracle.h"

typedef struct {
    uint64_t n, block, next;
    void (*body)(void *ctx, uint64_t i);
    void *ctx;
} po_pool;

static void *po_pool_work(void *arg) {
    po_pool *p = arg;
    for (;;) {
        const uint64_t lo = __atomic_fetch_add(&p->next, p->block, __ATOMIC_RELAXED);
        if (lo >= p->n) return NULL;
        const uint64_t hi = p->n - lo < p->block ? p->n : lo + p->block;
        for (uint64_t i = lo; i < hi; i++) p->body(p->ctx, i);
    }
}

/* body(ctx, i) for every i < n on min(nthreads, n) threads, the caller included.  Stops starting threads at
 * the first pthread_create failure and joins only those it started.  Returns PO_OK or PO_NOMEM. */
static int po_parallel_for(uint64_t n, int nthreads, uint64_t block, void (*body)(void *ctx, uint64_t i), void *ctx) {
    if (nthreads < 1 || n < 2) nthreads = 1;
    else if ((uint64_t)nthreads > n) nthreads = (int)n;
    po_pool p = {n, block < 1 ? 1 : block, 0, body, ctx};
    pthread_t *th = malloc(sizeof *th * (size_t)nthreads);
    if (!th) return PO_NOMEM;
    int started = 1; /* th[0] is the calling thread */
    while (started < nthreads && pthread_create(&th[started], NULL, po_pool_work, &p) == 0) started++;
    po_pool_work(&p);
    for (int t = 1; t < started; t++) pthread_join(th[t], NULL);
    free(th);
    return PO_OK;
}
#endif
