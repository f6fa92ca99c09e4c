/* CPU restatement of poly's synthesis/fragment (fragment.go), line for line: SetEfficiency with O(m^2)
 * table lookups per call, NextOverhangs over the A/T/G/C nesting, and optimizeOverhangIteration as the
 * reference's recursion (written as a loop: the call is in tail position), with the SetEfficiency of every
 * candidate recomputed from scratch.  The GPU's incremental formulation is checked against this file.
 *
 * TEST INFRASTRUCTURE ONLY.  The fidelity table is handed in by fragment_oracle.py, which reads
 * tests/golden/fragment/ligation_fidelity.json.  Statuses: 0 ok, 1 the reference panics, 2 unsupported
 * (a byte >= 0x80, which strings.ToUpper would re-encode), 3 "minFragmentSize (%d) larger than
 * maxFragmentSize (%d)", 4 "minFragmentSize must be equal to or greater than 12 . Got size of %d",
 * 5 "bestOverhangPosition failed by equaling zero". */
#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

enum { ST_OK, ST_PANIC, ST_UNSUPPORTED, ST_MIN_GT_MAX, ST_MIN_LT_12, ST_NO_POSITION };

typedef struct {
    const uint8_t *p;
    int64_t n;
} str;

static int32_t g_counts[120][120];
static int16_t g_key_of_code[256]; /* the map's hash: an A/C/G/T 4-mer's 2-bit code -> its key, or -1 */

static int base2(uint8_t b) { return b == 'A' ? 0 : b == 'C' ? 1 : b == 'G' ? 2 : b == 'T' ? 3 : -1; }

static int code_of(const uint8_t *p) {
    int c = 0;
    for (int i = 0; i < 4; ++i) {
        int b = base2(p[i]);
        if (b < 0) return -1;
        c = c << 2 | b;
    }
    return c;
}

void fr_set_table(const uint8_t *keys, const int32_t *counts) {
    memcpy(g_counts, counts, sizeof g_counts);
    for (int c = 0; c < 256; ++c) g_key_of_code[c] = -1;
    for (int k = 0; k < 120; ++k) g_key_of_code[code_of(keys + 4 * k)] = (int16_t)k;
}

/* transform.ReverseComplement's complementTable (transform.go:78-109); unlisted bytes are 0 */
static uint8_t comp(uint8_t b) {
    switch (b) {
    case 'A': return 'T'; case 'B': return 'V'; case 'C': return 'G'; case 'D': return 'H'; case 'G': return 'C';
    case 'H': return 'D'; case 'K': return 'M'; case 'M': return 'K'; case 'N': return 'N'; case 'R': return 'Y';
    case 'S': return 'S'; case 'T': return 'A'; case 'V': return 'B'; case 'W': return 'W'; case 'Y': return 'R';
    case 'a': return 't'; case 'b': return 'v'; case 'c': return 'g'; case 'd': return 'h'; case 'g': return 'c';
    case 'h': return 'd'; case 'k': return 'm'; case 'm': return 'k'; case 'n': return 'n'; case 'r': return 'y';
    case 's': return 's'; case 't': return 'a'; case 'v': return 'b'; case 'w': return 'w'; case 'y': return 'r';
    default: return 0;
    }
}

/* ReverseComplement(s) into a fresh buffer (the reference allocates one per call too) */
static str revcomp(str s) {
    uint8_t *o = malloc(s.n ? (size_t)s.n : 1);
    for (int64_t i = 0; i < s.n; ++i) o[i] = comp(s.p[s.n - i - 1]);
    return (str){o, s.n};
}

static int str_eq(str a, str b) { return a.n == b.n && (a.n == 0 || memcmp(a.p, b.p, (size_t)a.n) == 0); }

/* checks.IsPalindromic: sequence == ReverseComplement(sequence) */
static int is_palindromic(str s) {
    str r = revcomp(s);
    int eq = str_eq(s, r);
    free((void *)r.p);
    return eq;
}

/* the map's key lookup: a string is a key iff it equals one of the 120 (all of them A/C/G/T 4-mers) */
static int key_of(str s) {
    if (s.n != 4) return -1;
    int c = code_of(s.p);
    return c < 0 ? -1 : g_key_of_code[c];
}

/* mismatches[key{a, b}]: 0 for a missing key */
static int64_t mismatches(str a, str b) {
    int i = key_of(a), j = key_of(b);
    return i < 0 || j < 0 ? 0 : g_counts[i][j];
}

/* SetEfficiency (fragment.go:24-38) */
static double set_efficiency(const str *overhangs, int64_t m) {
    double efficiency = 1.0;
    for (int64_t a = 0; a < m; ++a) {
        int64_t nCorrect = mismatches(overhangs[a], overhangs[a]);
        int64_t nTotal = 0;
        for (int64_t b = 0; b < m; ++b) {
            nTotal = nTotal + mismatches(overhangs[a], overhangs[b]);
            str r = revcomp(overhangs[b]);
            nTotal = nTotal + mismatches(overhangs[a], r);
            free((void *)r.p);
        }
        if (nTotal != nCorrect) efficiency = efficiency * ((double)nCorrect / (double)nTotal);
    }
    return efficiency;
}

static str *set_from(const uint8_t *bytes, const uint64_t *off, uint64_t a, uint64_t b, int64_t extra) {
    str *s = malloc(sizeof(str) * (size_t)(b - a + (uint64_t)extra + 1));
    for (uint64_t i = a; i < b; ++i) s[i - a] = (str){bytes + off[i], (int64_t)(off[i + 1] - off[i])};
    return s;
}

double fr_set_efficiency(const uint8_t *bytes, const uint64_t *off, uint64_t n) {
    str *s = set_from(bytes, off, 0, n, 0);
    double e = set_efficiency(s, (int64_t)n);
    free(s);
    return e;
}

/* NextOverhangs (fragment.go:43-79): candidates (4 bytes each) and their efficiencies; returns the count */
int fr_next_overhangs(const uint8_t *bytes, const uint64_t *off, uint64_t n, uint8_t *cands, double *eff) {
    static const uint8_t bases[4] = {'A', 'T', 'G', 'C'};
    str *set = set_from(bytes, off, 0, n, 1);
    int count = 0;
    for (int b1 = 0; b1 < 4; ++b1)
        for (int b2 = 0; b2 < 4; ++b2)
            for (int b3 = 0; b3 < 4; ++b3)
                for (int b4 = 0; b4 < 4; ++b4) {
                    uint8_t x[4] = {bases[b1], bases[b2], bases[b3], bases[b4]};
                    str nx = {x, 4}, r = revcomp(nx);
                    int ok = 0, okReverse = 0;
                    for (uint64_t i = 0; i < n; ++i) {
                        ok |= str_eq(set[i], nx);
                        okReverse |= str_eq(set[i], r);
                    }
                    if (!ok && !okReverse && !is_palindromic(nx)) memcpy(cands + 4 * count++, x, 4);
                    free((void *)r.p);
                }
    for (int c = 0; c < count; ++c) {
        str x = {cands + 4 * c, 4}, r = revcomp(x);
        set[n] = x;
        double strand = set_efficiency(set, (int64_t)n + 1);
        set[n] = r;
        double complement = set_efficiency(set, (int64_t)n + 1);
        eff[c] = (strand + complement) / 2;
        free((void *)r.p);
    }
    free(set);
    return count;
}

/* Fragment / FragmentWithOverhangs (fragment.go:101-202).  n_inc == 0 is Fragment.  ends[k] is the end of
 * fragment k in the input's coordinates (fragment k starts at ends[k - 1] - 4, the first at 0);
 * *n_ends is 0 unless the status is ST_OK.  err_min / err_max are the values of the failing step. */
int fr_fragment(const uint8_t *seq_in, int64_t len_in, int64_t minFragmentSize, int64_t maxFragmentSize, const uint8_t *ex, const uint64_t *ex_off,
                uint64_t n_ex, const uint8_t *inc, const uint64_t *inc_off, uint64_t n_inc, double *eff, int64_t *err_min, int64_t *err_max,
                uint64_t *ends, uint64_t *n_ends) {
    *eff = 0;
    *err_min = *err_max = 0;
    *n_ends = 0;
    for (int64_t i = 0; i < len_in; ++i)
        if (seq_in[i] >= 0x80) return ST_UNSUPPORTED;
    /* sequence = strings.ToUpper(sequence) */
    uint8_t *up = malloc((size_t)(len_in > 0 ? len_in : 1));
    for (int64_t i = 0; i < len_in; ++i) up[i] = seq_in[i] >= 'a' && seq_in[i] <= 'z' ? seq_in[i] - 32 : seq_in[i];
    if (len_in < 4) { free(up); return ST_PANIC; } /* sequence[:4] */
    /* append([]string{sequence[:4], sequence[len(sequence)-4:]}, excludeOverhangs...) */
    int64_t cap = 2 + (int64_t)n_ex + len_in / 2 + 2, m = 0;
    str *excludeOverhangs = malloc(sizeof(str) * (size_t)cap);
    excludeOverhangs[m++] = (str){up, 4};
    excludeOverhangs[m++] = (str){up + len_in - 4, 4};
    for (uint64_t i = 0; i < n_ex; ++i) excludeOverhangs[m++] = (str){ex + ex_off[i], (int64_t)(ex_off[i + 1] - ex_off[i])};
    str *includeOverhangs = set_from(inc, inc_off, 0, n_inc, 0);
    str sequence = {up, len_in};
    uint64_t nfrag = 0;
    int st;
    for (;;) {
        if (sequence.n < maxFragmentSize) {
            ends[nfrag++] = (uint64_t)(sequence.p + sequence.n - up);
            *eff = set_efficiency(excludeOverhangs, m);
            st = ST_OK;
            break;
        }
        if (minFragmentSize > maxFragmentSize) { st = ST_MIN_GT_MAX; break; }
        if (minFragmentSize < 12) { st = ST_MIN_LT_12; break; }
        if (sequence.n < 2 * maxFragmentSize) {
            int64_t maxAndMinDifference = maxFragmentSize - minFragmentSize;
            int64_t maxFragmentSizeBuffer = (sequence.n + maxAndMinDifference) / 2;
            if (maxFragmentSizeBuffer > maxFragmentSize) maxFragmentSizeBuffer = maxFragmentSize;
            minFragmentSize = maxFragmentSizeBuffer - maxAndMinDifference;
            maxFragmentSize = maxFragmentSizeBuffer;
        }
        double bestOverhangEfficiency = 0;
        int64_t bestOverhangPosition = 0;
        for (int64_t overhangOffset = 0; overhangOffset <= maxFragmentSize - minFragmentSize; overhangOffset++) {
            int64_t overhangPosition = maxFragmentSize - overhangOffset;
            str overhangToTest = {sequence.p + overhangPosition - 4, 4};
            int alreadyExists = 0;
            for (int64_t i = 0; i < m; ++i) {
                str r = revcomp(excludeOverhangs[i]);
                if (str_eq(excludeOverhangs[i], overhangToTest) || str_eq(r, overhangToTest)) alreadyExists = 1;
                free((void *)r.p);
            }
            int buildAvailable = n_inc == 0;
            for (uint64_t i = 0; i < n_inc; ++i) {
                str r = revcomp(includeOverhangs[i]);
                if (str_eq(includeOverhangs[i], overhangToTest) || str_eq(r, overhangToTest)) buildAvailable = 1;
                free((void *)r.p);
            }
            if (!alreadyExists && buildAvailable && !is_palindromic(overhangToTest)) {
                excludeOverhangs[m] = overhangToTest; /* append(excludeOverhangs, overhangToTest) */
                double setEfficiency = set_efficiency(excludeOverhangs, m + 1);
                if (setEfficiency > bestOverhangEfficiency) {
                    bestOverhangEfficiency = setEfficiency;
                    bestOverhangPosition = overhangPosition;
                }
            }
        }
        if (bestOverhangPosition == 0) { st = ST_NO_POSITION; break; }
        ends[nfrag++] = (uint64_t)(sequence.p + bestOverhangPosition - up);
        excludeOverhangs[m++] = (str){sequence.p + bestOverhangPosition - 4, 4};
        sequence = (str){sequence.p + bestOverhangPosition - 4, sequence.n - (bestOverhangPosition - 4)};
    }
    if (st == ST_OK) *n_ends = nfrag;
    if (st == ST_MIN_GT_MAX || st == ST_MIN_LT_12) {
        *err_min = minFragmentSize;
        *err_max = maxFragmentSize;
    }
    free(excludeOverhangs);
    free(includeOverhangs);
    free(up);
    return st;
}

/* ---- threaded batch drivers (the CPU arm of tools/bench_fragment.py) ---- */
typedef struct {
    const uint8_t *seqs;
    const uint64_t *off;
    uint64_t n;
    int64_t min, max;
    const uint8_t *ex, *inc;
    const uint64_t *ex_off, *inc_off, *set_off, *ends_off;
    uint64_t n_ex, n_inc;
    int32_t *status;
    double *eff;
    int64_t *err_min, *err_max;
    uint64_t *ends, *n_ends;
    uint8_t *cands;
    uint32_t *n_cands;
    int kind; /* 0 fragment, 1 set efficiency, 2 next overhangs */
    uint64_t next;
    pthread_mutex_t mu;
} Batch;

static void *worker(void *arg) {
    Batch *b = arg;
    for (;;) {
        pthread_mutex_lock(&b->mu);
        uint64_t i = b->next++;
        pthread_mutex_unlock(&b->mu);
        if (i >= b->n) return NULL;
        if (b->kind == 0) {
            b->status[i] = fr_fragment(b->seqs + b->off[i], (int64_t)(b->off[i + 1] - b->off[i]), b->min, b->max, b->ex, b->ex_off, b->n_ex, b->inc,
                                       b->inc_off, b->n_inc, &b->eff[i], &b->err_min[i], &b->err_max[i], b->ends + b->ends_off[i], &b->n_ends[i]);
        } else if (b->kind == 1) {
            b->eff[i] = fr_set_efficiency(b->seqs, b->off + b->set_off[i], b->set_off[i + 1] - b->set_off[i]);
        } else {
            b->n_cands[i] = (uint32_t)fr_next_overhangs(b->seqs, b->off + b->set_off[i], b->set_off[i + 1] - b->set_off[i], b->cands + 1024 * i,
                                                        b->eff + 256 * i);
        }
    }
}

static void run(Batch *b, int threads) {
    pthread_mutex_init(&b->mu, NULL);
    if (threads < 1) threads = 1;
    pthread_t *t = malloc(sizeof(pthread_t) * (size_t)threads);
    for (int k = 0; k < threads; ++k) pthread_create(&t[k], NULL, worker, b);
    for (int k = 0; k < threads; ++k) pthread_join(t[k], NULL);
    free(t);
    pthread_mutex_destroy(&b->mu);
}

/* item i's ends go to ends[ends_off[i] ..], which must have room for (L - 12) / 2 + 2 of them */
void fr_fragment_batch(const uint8_t *seqs, const uint64_t *off, uint64_t n, int64_t min, int64_t max, const uint8_t *ex, const uint64_t *ex_off,
                       uint64_t n_ex, const uint8_t *inc, const uint64_t *inc_off, uint64_t n_inc, int32_t *status, double *eff, int64_t *err_min,
                       int64_t *err_max, uint64_t *ends, const uint64_t *ends_off, uint64_t *n_ends, int threads) {
    Batch b = {.seqs = seqs, .off = off, .n = n, .min = min, .max = max, .ex = ex, .ex_off = ex_off, .n_ex = n_ex, .inc = inc, .inc_off = inc_off,
               .n_inc = n_inc, .status = status, .eff = eff, .err_min = err_min, .err_max = err_max, .ends = ends, .ends_off = ends_off,
               .n_ends = n_ends, .kind = 0};
    run(&b, threads);
}

/* set i is overhangs [set_off[i], set_off[i + 1]) of the ragged list (bytes, off) */
void fr_set_efficiency_batch(const uint8_t *bytes, const uint64_t *off, const uint64_t *set_off, uint64_t n_sets, double *eff, int threads) {
    Batch b = {.seqs = bytes, .off = off, .set_off = set_off, .n = n_sets, .eff = eff, .kind = 1};
    run(&b, threads);
}

/* cands: n_sets x 256 x 4 bytes, eff: n_sets x 256 */
void fr_next_overhangs_batch(const uint8_t *bytes, const uint64_t *off, const uint64_t *set_off, uint64_t n_sets, uint8_t *cands, uint32_t *n_cands,
                             double *eff, int threads) {
    Batch b = {.seqs = bytes, .off = off, .set_off = set_off, .n = n_sets, .cands = cands, .n_cands = n_cands, .eff = eff, .kind = 2};
    run(&b, threads);
}
