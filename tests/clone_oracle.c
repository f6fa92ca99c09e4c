/* clone_oracle.c -- CPU restatement of poly's clone package (clone/clone.go:138-355), line by line.
 *
 * TEST INFRASTRUCTURE ONLY (tests/ and tools/bench_clone.py).  Compiled on first use by tests/clone_oracle.py
 * into a temporary directory and linked against oracle/libseqhash_oracle.so for po_seqhash.
 *
 * - regexp.FindAllStringIndex on a literal pattern: leftmost, non-overlapping matches (the next search starts
 *   at the end of the previous match).
 * - Go slice expressions that would be out of range are reported as a panic (return 1), never computed around.
 * - recurseLigate hashes every construct where the reference does (clone.go:275,305): eagerly, at the call site.
 *
 * Serialised string lists (inputs and outputs): for each string, a little-endian uint64 length then the bytes.
 * A fragment is three such strings: Sequence, ForwardOverhang, ReverseOverhang. */
#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

int po_seqhash(const uint8_t *seq, int64_t n, int seq_type, int circular, int double_stranded, uint8_t digest[32], int64_t *err_pos);

enum { CO_OK = 0, CO_PANIC = 1, CO_UNSUPPORTED = 2 };

/* ---- strings ---------------------------------------------------------------------------------------- */
typedef struct {
    uint8_t *p;
    int64_t n;
} str;

static str s_new(const uint8_t *p, int64_t n) {
    str s = {malloc(n > 0 ? (size_t)n : 1), n};
    if (n) memcpy(s.p, p, (size_t)n);
    return s;
}
static str s_cat(str a, str b) {
    str s = {malloc(a.n + b.n > 0 ? (size_t)(a.n + b.n) : 1), a.n + b.n};
    memcpy(s.p, a.p, (size_t)a.n);
    memcpy(s.p + a.n, b.p, (size_t)b.n);
    return s;
}
static int s_eq(str a, str b) { return a.n == b.n && memcmp(a.p, b.p, (size_t)a.n) == 0; }

/* transform.ReverseComplement: complementTable (transform.go:78-109), unlisted bytes are 0 */
static uint8_t comp(uint8_t c) {
    static const char from[] = "ABCDGHKMNRSTVWYabcdghkmnrstvwy", to[] = "TVGHCDMKNYSABWRtvghcdmknysabwr";
    for (int i = 0; from[i]; i++)
        if ((uint8_t)from[i] == c) return (uint8_t)to[i];
    return 0;
}
static str s_rc(str a) {
    str s = {malloc(a.n > 0 ? (size_t)a.n : 1), a.n};
    for (int64_t i = 0; i < a.n; i++) s.p[i] = comp(a.p[a.n - 1 - i]);
    return s;
}

typedef struct {
    str *v;
    int64_t n, cap;
} strlist;
static void sl_push(strlist *l, str s) {
    if (l->n == l->cap) {
        l->cap = l->cap ? 2 * l->cap : 16;
        l->v = realloc(l->v, sizeof(str) * (size_t)l->cap);
    }
    l->v[l->n++] = s;
}
static void sl_truncate(strlist *l, int64_t n) {
    while (l->n > n) free(l->v[--l->n].p);
}

/* serialised output: the strings of l, each as (uint64 length, bytes) */
static uint8_t *serialise(const strlist *l, uint64_t *bytes) {
    uint64_t n = 0;
    for (int64_t i = 0; i < l->n; i++) n += 8 + (uint64_t)l->v[i].n;
    uint8_t *out = malloc(n ? n : 1), *w = out;
    for (int64_t i = 0; i < l->n; i++) {
        uint64_t len = (uint64_t)l->v[i].n;
        memcpy(w, &len, 8);
        memcpy(w + 8, l->v[i].p, len);
        w += 8 + len;
    }
    *bytes = n;
    return out;
}

void co_free(void *p) { free(p); }

/* ---- CutWithEnzyme (clone.go:138-268) ------------------------------------------------------------------ */
typedef struct {
    int64_t position;
    int forward;
} overhang;

/* regexp.FindAllStringIndex of a literal: leftmost non-overlapping match starts */
static int64_t find_all(const uint8_t *s, int64_t n, const uint8_t *pat, int64_t m, int64_t *starts) {
    int64_t c = 0;
    for (int64_t i = 0; i + m <= n;) {
        if (memcmp(s + i, pat, (size_t)m) == 0) {
            starts[c++] = i;
            i += m;
        } else {
            i++;
        }
    }
    return c;
}

/* Go's s[lo:hi] on a string of length n is in range iff 0 <= lo <= hi <= n */
static int in_range(int64_t lo, int64_t hi, int64_t n) { return 0 <= lo && lo <= hi && hi <= n; }

typedef struct {
    const uint8_t *fsite, *rsite, *recog;
    int64_t fl, rl, recl, skip, ohl;
} enzyme;

/* Fragments of one part, appended to `out` as (Sequence, ForwardOverhang, ReverseOverhang) triples.
 * Returns CO_OK, CO_PANIC (a slice out of range) or CO_UNSUPPORTED (a byte >= 0x80: ToUpper re-encodes). */
static int cut(const uint8_t *part, int64_t L, int circular, int directional, const enzyme *e, strlist *out) {
    const int64_t N = circular ? 2 * L : L;
    for (int64_t i = 0; i < L; i++)
        if (part[i] >= 0x80) return CO_UNSUPPORTED;
    uint8_t *seq = malloc(N > 0 ? (size_t)N : 1);
    for (int64_t i = 0; i < N; i++) {
        uint8_t c = part[i % L];
        seq[i] = (c >= 'a' && c <= 'z') ? c - 32 : c; /* strings.ToUpper(part + part) */
    }
    /* checks.IsPalindromic(RecognitionSite) */
    int palindromic = 1;
    for (int64_t i = 0; i < e->recl; i++)
        if (e->recog[i] != comp(e->recog[e->recl - 1 - i])) palindromic = 0;

    int64_t *fs = malloc(sizeof(int64_t) * (size_t)(N + 1)), *rs = malloc(sizeof(int64_t) * (size_t)(N + 1));
    int64_t nf = find_all(seq, N, e->fsite, e->fl, fs), nr = 0;
    overhang *fo = malloc(sizeof(overhang) * (size_t)(nf + 1)), *ro = malloc(sizeof(overhang) * (size_t)(N + 1));
    for (int64_t i = 0; i < nf; i++) fo[i] = (overhang){fs[i] + e->fl + e->skip, 1};
    if (!palindromic) {
        nr = find_all(seq, N, e->rsite, e->rl, rs);
        for (int64_t i = 0; i < nr; i++) ro[i] = (overhang){rs[i] - e->skip, 0};
    }
    /* drop the last overhang of a set on a linear part (Skip counted twice, clone.go:166-174) */
    int64_t kf = nf, kr = nr;
    if (kf > 0 && !circular && fo[kf - 1].position + e->skip + e->ohl > N) kf--;
    if (kr > 0 && !circular && ro[kr - 1].position + e->skip + e->ohl > N) kr--;
    /* sort.SliceStable on forward ++ reverse */
    const int64_t n = kf + kr;
    overhang *ov = malloc(sizeof(overhang) * (size_t)(n + 1));
    for (int64_t i = 0, a = 0, b = 0; i < n; i++) ov[i] = (b >= kr || (a < kf && fo[a].position <= ro[b].position)) ? fo[a++] : ro[b++];

    int rc = CO_OK;
    const int64_t OH = e->ohl;
    str empty = {NULL, 0};
    if (n == 1 && !directional && !circular) {
        const int64_t P = ov[0].position;
        if (nf > 0) { /* len(forwardOverhangs): the set before the drop */
            if (!in_range(P + OH, N, N) || !in_range(0, P, N) || !in_range(P, P + OH, N)) { rc = CO_PANIC; goto done; }
            str f1 = s_new(seq + P + OH, N - P - OH), f2 = s_new(seq, P), o = s_new(seq + P, OH);
            sl_push(out, f1); sl_push(out, s_new(o.p, o.n)); sl_push(out, s_new(empty.p, 0));
            sl_push(out, f2); sl_push(out, s_new(empty.p, 0)); sl_push(out, o);
        } else {
            if (!in_range(P, N, N) || !in_range(0, P - OH, N) || !in_range(P - OH, P, N)) { rc = CO_PANIC; goto done; }
            str f1 = s_new(seq + P, N - P), f2 = s_new(seq, P - OH), o = s_new(seq + P - OH, OH);
            sl_push(out, f2); sl_push(out, s_new(empty.p, 0)); sl_push(out, s_new(o.p, o.n));
            sl_push(out, f1); sl_push(out, o); sl_push(out, s_new(empty.p, 0));
        }
        goto done;
    }
    if (n == 2 && !directional && circular) {
        const int64_t P = ov[0].position;
        if (!in_range(P + OH, L, N) || !in_range(0, P, N) || !in_range(P, P + OH, N)) { rc = CO_PANIC; goto done; }
        str s1 = s_new(seq + P + OH, L - P - OH), s2 = s_new(seq, P), o = s_new(seq + P, OH);
        sl_push(out, s_cat(s1, s2)); sl_push(out, s_new(o.p, o.n)); sl_push(out, o);
        free(s1.p); free(s2.p);
        goto done;
    }
    if (n > 1) {
        const int64_t rssl = e->recl + e->skip;
        strlist pieces = {0};
        for (int64_t i = 0; i < n - 1; i++) {
            overhang cur = ov[i], nxt = ov[i + 1];
            if (directional && !palindromic) {
                if (cur.forward && !nxt.forward) {
                    if (!in_range(cur.position, nxt.position, N)) { rc = CO_PANIC; break; }
                    sl_push(&pieces, s_new(seq + cur.position, nxt.position - cur.position));
                }
                if (nxt.position - rssl > L) break;
            } else {
                if (!in_range(cur.position, nxt.position, N)) { rc = CO_PANIC; break; }
                sl_push(&pieces, s_new(seq + cur.position, nxt.position - cur.position));
                if (nxt.position - rssl > L) break;
            }
        }
        for (int64_t i = 0; rc == CO_OK && i < pieces.n; i++) {
            str f = pieces.v[i];
            if (f.n > 8) {
                if (!in_range(OH, f.n - OH, f.n) || !in_range(0, OH, f.n) || !in_range(f.n - OH, f.n, f.n)) { rc = CO_PANIC; break; }
                sl_push(out, s_new(f.p + OH, f.n - 2 * OH));
                sl_push(out, s_new(f.p, OH));
                sl_push(out, s_new(f.p + f.n - OH, OH));
            }
        }
        sl_truncate(&pieces, 0);
        free(pieces.v);
    }
done:
    free(seq); free(fs); free(rs); free(fo); free(ro); free(ov);
    return rc;
}

/* CutWithEnzyme on one part.  *out: serialised fragments (3 strings each), freed with co_free. */
int co_cut(const uint8_t *part, int64_t L, int circular, int directional, const uint8_t *fsite, int64_t fl, const uint8_t *rsite,
           int64_t rl, const uint8_t *recog, int64_t recl, int64_t skip, int64_t ohl, uint8_t **out, uint64_t *out_bytes, int64_t *n_frag) {
    enzyme e = {fsite, rsite, recog, fl, rl, recl, skip, ohl};
    strlist l = {0};
    int rc = cut(part, L, circular, directional, &e, &l);
    if (rc != CO_OK) sl_truncate(&l, 0);
    *n_frag = l.n / 3;
    *out = serialise(&l, out_bytes);
    sl_truncate(&l, 0);
    free(l.v);
    return rc;
}

/* ---- timed CPU arm: CutWithEnzyme over (part, enzyme) items on nthreads threads ------------------------ */
typedef struct {
    const uint8_t *parts;
    const uint64_t *offsets;
    const uint8_t *circular;
    uint64_t n_parts, next;
    const enzyme *enz;
    int n_enz, directional;
    int64_t *n_frag;
    int32_t *status;
} cut_batch;

static void *cut_worker(void *arg) {
    cut_batch *b = arg;
    for (;;) {
        uint64_t i = __atomic_fetch_add(&b->next, 1, __ATOMIC_RELAXED);
        if (i >= b->n_parts * (uint64_t)b->n_enz) return NULL;
        const uint64_t p = i / (uint64_t)b->n_enz;
        strlist l = {0};
        b->status[i] = cut(b->parts + b->offsets[p], (int64_t)(b->offsets[p + 1] - b->offsets[p]), b->circular[p], b->directional,
                           &b->enz[i % (uint64_t)b->n_enz], &l);
        b->n_frag[i] = b->status[i] == CO_OK ? l.n / 3 : 0;
        sl_truncate(&l, 0);
        free(l.v);
    }
}

/* enzymes: n_enz records of (fsite, rsite, recog) as NUL-free byte strings with lengths, skip, ohl */
void co_cut_batch(const uint8_t *parts, const uint64_t *offsets, const uint8_t *circular, uint64_t n_parts, const uint8_t *const *sites,
                  const int64_t *site_lens, const int64_t *skip_ohl, int n_enz, int directional, int nthreads, int64_t *n_frag, int32_t *status) {
    enzyme *enz = malloc(sizeof(enzyme) * (size_t)n_enz);
    for (int k = 0; k < n_enz; k++)
        enz[k] = (enzyme){sites[3 * k], sites[3 * k + 1], sites[3 * k + 2], site_lens[3 * k], site_lens[3 * k + 1], site_lens[3 * k + 2],
                          skip_ohl[2 * k], skip_ohl[2 * k + 1]};
    cut_batch b = {parts, offsets, circular, n_parts, 0, enz, n_enz, directional, n_frag, status};
    if (nthreads < 1) nthreads = 1;
    pthread_t *th = malloc(sizeof(pthread_t) * (size_t)nthreads);
    for (int t = 1; t < nthreads; t++) pthread_create(&th[t], NULL, cut_worker, &b);
    cut_worker(&b);
    for (int t = 1; t < nthreads; t++) pthread_join(th[t], NULL);
    free(th);
    free(enz);
}

/* ---- recurseLigate / CircularLigate (clone.go:270-338) -------------------------------------------------- */
typedef struct {
    str seq, fwd, rev;
} fragment;

/* existingSeqhashes: a set of seqhash strings.  The key is the 4-byte metadata (C or L) and the digest; a
 * failed Hash gives "" in the reference (the error is dropped), which is its own key. */
typedef struct {
    uint8_t (*key)[34];
    uint8_t *used;
    uint64_t cap, n;
} hashset;

static uint64_t hs_hash(const uint8_t *k) {
    uint64_t h = 1469598103934665603ull;
    for (int i = 0; i < 34; i++) h = (h ^ k[i]) * 1099511628211ull;
    return h;
}
/* 1 if k was inserted (not present before) */
static int hs_insert(hashset *s, const uint8_t *k) {
    if (2 * (s->n + 1) > s->cap) {
        hashset t = {NULL, NULL, s->cap ? 2 * s->cap : 1024, 0};
        t.key = calloc(t.cap, 34);
        t.used = calloc(t.cap, 1);
        for (uint64_t i = 0; i < s->cap; i++)
            if (s->used[i]) hs_insert(&t, s->key[i]);
        free(s->key); free(s->used);
        *s = t;
    }
    for (uint64_t i = hs_hash(k) & (s->cap - 1);; i = (i + 1) & (s->cap - 1)) {
        if (!s->used[i]) {
            s->used[i] = 1;
            memcpy(s->key[i], k, 34);
            s->n++;
            return 1;
        }
        if (memcmp(s->key[i], k, 34) == 0) return 0;
    }
}

/* seqhash.Hash(construct, "DNA", circular, true) as a set key */
static void seqhash_key(str c, int circular, uint8_t key[34]) {
    int64_t pos;
    memset(key, 0, 34);
    if (po_seqhash(c.p, c.n, 0, circular, 1, key + 2, &pos) != 0) {
        memset(key, 0, 34); /* "" */
        return;
    }
    key[0] = 1;
    key[1] = circular ? 'C' : 'L';
}

typedef struct {
    const fragment *list;
    int64_t n;
    hashset seen;
    strlist open, infinite;
} ligation;

static void recurse_ligate(ligation *g, fragment seed, const fragment *used_in, int64_t n_used) {
    uint8_t key[34];
    if (s_eq(seed.fwd, seed.rev)) {
        str construct = s_cat(seed.fwd, seed.seq);
        seqhash_key(construct, 1, key);
        if (!hs_insert(&g->seen, key)) { free(construct.p); return; }
        sl_push(&g->open, construct);
        return;
    }
    /* usedFragments is this call's own slice: it grows across the loop's iterations */
    fragment *used = malloc(sizeof(fragment) * (size_t)(n_used + g->n + 1));
    memcpy(used, used_in, sizeof(fragment) * (size_t)n_used);
    const int64_t open0 = g->open.n, inf0 = g->infinite.n;
    str seed_rev_rc = s_rc(seed.rev);
    for (int64_t f = 0; f < g->n; f++) {
        const fragment nf = g->list[f];
        fragment ns = {{0}, {0}, {0}};
        str rev_owned = {NULL, 0}; /* ReverseComplement(newFragment.ForwardOverhang) of the second attach */
        int attached = 0;
        if (s_eq(seed.rev, nf.fwd)) {
            attached = 1;
            str t = s_cat(seed.seq, seed.rev);
            ns = (fragment){s_cat(t, nf.seq), seed.fwd, nf.rev};
            free(t.p);
        }
        str nf_rev_rc = s_rc(nf.rev);
        if (s_eq(seed.rev, nf_rev_rc) && !s_eq(seed.rev, seed_rev_rc)) {
            free(ns.seq.p);
            attached = 1;
            str t = s_cat(seed.seq, seed.rev), r = s_rc(nf.seq);
            rev_owned = s_rc(nf.fwd);
            ns = (fragment){s_cat(t, r), seed.fwd, rev_owned};
            free(t.p); free(r.p);
        }
        free(nf_rev_rc.p);
        if (!attached) continue;
        for (int64_t u = 0; u < n_used; u++) {
            if (s_eq(used[u].seq, nf.seq)) {
                str t = s_cat(used[u].fwd, used[u].seq), inf = s_cat(t, used[u].rev);
                free(t.p);
                free(rev_owned.p);
                free(ns.seq.p);
                free(seed_rev_rc.p);
                free(used);
                /* return nil, ...: whatever this call collected so far is dropped */
                sl_truncate(&g->open, open0);
                sl_truncate(&g->infinite, inf0);
                seqhash_key(inf, 0, key);
                if (!hs_insert(&g->seen, key)) { free(inf.p); return; }
                sl_push(&g->infinite, inf);
                return;
            }
        }
        used[n_used++] = nf;
        recurse_ligate(g, ns, used, n_used);
        free(rev_owned.p);
        free(ns.seq.p);
    }
    free(seed_rev_rc.p);
    free(used);
}

static fragment *parse_fragments(const uint8_t *buf, int64_t n) {
    fragment *f = malloc(sizeof(fragment) * (size_t)(n + 1));
    for (int64_t i = 0; i < n; i++) {
        str *parts[3] = {&f[i].seq, &f[i].fwd, &f[i].rev};
        for (int j = 0; j < 3; j++) {
            uint64_t len;
            memcpy(&len, buf, 8);
            parts[j]->p = (uint8_t *)buf + 8;
            parts[j]->n = (int64_t)len;
            buf += 8 + len;
        }
    }
    return f;
}

/* CircularLigate on n serialised fragments.  *clones and *loops: serialised strings (co_free). */
void co_circular_ligate(const uint8_t *frags, int64_t n, uint8_t **clones, uint64_t *clone_bytes, int64_t *n_clones, uint8_t **loops,
                        uint64_t *loop_bytes, int64_t *n_loops) {
    fragment *list = parse_fragments(frags, n);
    ligation g = {list, n, {0}, {0}, {0}};
    for (int64_t i = 0; i < n; i++) recurse_ligate(&g, list[i], NULL, 0);
    *n_clones = g.open.n;
    *n_loops = g.infinite.n;
    *clones = serialise(&g.open, clone_bytes);
    *loops = serialise(&g.infinite, loop_bytes);
    sl_truncate(&g.open, 0);
    sl_truncate(&g.infinite, 0);
    free(g.open.v); free(g.infinite.v);
    free(g.seen.key); free(g.seen.used);
    free(list);
}
