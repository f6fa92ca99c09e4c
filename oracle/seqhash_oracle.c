/*
 * oracle/seqhash_oracle.c -- CPU restatement of seqhash (seqhash/seqhash.go:78-223) and of BLAKE3
 * (hash mode, 32-byte output, written from the BLAKE3 specification).
 *
 * TEST INFRASTRUCTURE ONLY (as everything under oracle/): the checker of the CUDA seqhash path and the
 * timed CPU arm of tools/bench_seqhash.py ("C restatement, not Go").  Loaded by tests/seqhash_oracle.py.
 *
 * Non-ASCII input: the first byte that is >= 0x80 or outside the alphabet decides, as the library
 * does (DESIGN.md §7): a byte >= 0x80 there is reported as unsupported (3), not hashed.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "parallel.h"
#include "poly_oracle.h"

/* ---- BLAKE3 ------------------------------------------------------------------------------------ */
#define B3_CHUNK_START 1u
#define B3_CHUNK_END 2u
#define B3_PARENT 4u
#define B3_ROOT 8u

static const uint32_t B3_IV[8] = {0x6A09E667u, 0xBB67AE85u, 0x3C6EF372u, 0xA54FF53Au,
                                  0x510E527Fu, 0x9B05688Cu, 0x1F83D9ABu, 0x5BE0CD19u};
static const int B3_PERM[16] = {2, 6, 3, 10, 7, 0, 4, 13, 1, 11, 12, 5, 9, 14, 15, 8};

static uint32_t rotr32(uint32_t x, int r) { return (x >> r) | (x << (32 - r)); }

static void b3_g(uint32_t *v, int a, int b, int c, int d, uint32_t x, uint32_t y) {
    v[a] = v[a] + v[b] + x; v[d] = rotr32(v[d] ^ v[a], 16);
    v[c] = v[c] + v[d];     v[b] = rotr32(v[b] ^ v[c], 12);
    v[a] = v[a] + v[b] + y; v[d] = rotr32(v[d] ^ v[a], 8);
    v[c] = v[c] + v[d];     v[b] = rotr32(v[b] ^ v[c], 7);
}

/* out[0..7] = the chaining value of compressing the 16-word block under cv */
static void b3_compress(const uint32_t cv[8], const uint32_t block[16], uint64_t counter, uint32_t block_len, uint32_t flags,
                        uint32_t out[8]) {
    uint32_t v[16], m[16], t[16];
    for (int i = 0; i < 8; i++) v[i] = cv[i];
    for (int i = 0; i < 4; i++) v[8 + i] = B3_IV[i];
    v[12] = (uint32_t)counter; v[13] = (uint32_t)(counter >> 32); v[14] = block_len; v[15] = flags;
    memcpy(m, block, sizeof m);
    for (int r = 0; r < 7; r++) {
        b3_g(v, 0, 4, 8, 12, m[0], m[1]);   b3_g(v, 1, 5, 9, 13, m[2], m[3]);
        b3_g(v, 2, 6, 10, 14, m[4], m[5]);  b3_g(v, 3, 7, 11, 15, m[6], m[7]);
        b3_g(v, 0, 5, 10, 15, m[8], m[9]);  b3_g(v, 1, 6, 11, 12, m[10], m[11]);
        b3_g(v, 2, 7, 8, 13, m[12], m[13]); b3_g(v, 3, 4, 9, 14, m[14], m[15]);
        for (int i = 0; i < 16; i++) t[i] = m[B3_PERM[i]];
        memcpy(m, t, sizeof m);
    }
    for (int i = 0; i < 8; i++) out[i] = v[i] ^ v[i + 8];
}

static void b3_words(const uint8_t *p, size_t len, uint32_t w[16]) { /* little-endian, zero padded */
    uint8_t b[64] = {0};
    memcpy(b, p, len);
    for (int i = 0; i < 16; i++) w[i] = (uint32_t)b[4 * i] | (uint32_t)b[4 * i + 1] << 8 | (uint32_t)b[4 * i + 2] << 16 | (uint32_t)b[4 * i + 3] << 24;
}

/* The final compression of one chunk, held back until the caller knows whether it is the root. */
typedef struct {
    uint32_t cv[8], block[16], block_len, flags;
    uint64_t counter;
} b3_output;

static b3_output b3_chunk(const uint8_t *p, size_t len, uint64_t counter) {
    b3_output o;
    memcpy(o.cv, B3_IV, sizeof o.cv);
    size_t nblocks = len ? (len + 63) / 64 : 1;
    for (size_t b = 0; b + 1 < nblocks; b++) {
        uint32_t w[16];
        b3_words(p + 64 * b, 64, w);
        b3_compress(o.cv, w, counter, 64, b == 0 ? B3_CHUNK_START : 0, o.cv);
    }
    size_t last = len - 64 * (nblocks - 1);
    b3_words(p + 64 * (nblocks - 1), last, o.block);
    o.block_len = (uint32_t)last;
    o.flags = B3_CHUNK_END | (nblocks == 1 ? B3_CHUNK_START : 0);
    o.counter = counter;
    return o;
}

static b3_output b3_parent(const uint32_t left[8], const uint32_t right[8]) {
    b3_output o;
    memcpy(o.cv, B3_IV, sizeof o.cv);
    memcpy(o.block, left, 32);
    memcpy(o.block + 8, right, 32);
    o.block_len = 64;
    o.flags = B3_PARENT;
    o.counter = 0;
    return o;
}

static void b3_cv(const b3_output *o, uint32_t flags, uint32_t out[8]) {
    b3_compress(o->cv, o->block, o->counter, o->block_len, o->flags | flags, out);
}

/* The incremental hasher of the specification: a stack of subtree chaining values, merged whenever
 * the number of completed chunks has a trailing zero bit. */
void po_blake3(const uint8_t *in, uint64_t len, uint8_t out[32]) {
    uint32_t stack[64][8];
    int depth = 0;
    uint64_t chunk = 0, pos = 0;
    while (len - pos > 1024) {
        b3_output o = b3_chunk(in + pos, 1024, chunk);
        uint32_t cv[8];
        b3_cv(&o, 0, cv);
        uint64_t total = ++chunk;
        while ((total & 1) == 0) {
            b3_output p = b3_parent(stack[--depth], cv);
            b3_cv(&p, 0, cv);
            total >>= 1;
        }
        memcpy(stack[depth++], cv, 32);
        pos += 1024;
    }
    b3_output o = b3_chunk(in + pos, (size_t)(len - pos), chunk);
    while (depth > 0) {
        uint32_t cv[8];
        b3_cv(&o, 0, cv);
        o = b3_parent(stack[--depth], cv);
    }
    uint32_t h[8];
    b3_cv(&o, B3_ROOT, h);
    for (int i = 0; i < 8; i++)
        for (int k = 0; k < 4; k++) out[4 * i + k] = (uint8_t)(h[i] >> (8 * k));
}

/* ---- seqhash.go ---------------------------------------------------------------------------------- */
/* transform.complementTable (transform/transform.go:78-109): unlisted bytes are 0 */
static uint8_t sh_complement(uint8_t c) {
    static const char from[] = "ABCDGHKMNRSTVWYabcdghkmnrstvwy", to[] = "TVGHCDMKNYSABWRtvghcdmknysabwr";
    for (int i = 0; from[i]; i++)
        if ((uint8_t)from[i] == c) return (uint8_t)to[i];
    return 0;
}

/* boothLeastRotation (seqhash.go:78-124), literally: the doubled string and the failure slice */
int64_t po_booth_least_rotation(const uint8_t *seq, int64_t n) {
    if (n <= 0) return 0;
    int64_t m = 2 * n, k = 0;
    uint8_t *s = malloc((size_t)m);
    int64_t *f = malloc((size_t)m * sizeof *f);
    memcpy(s, seq, (size_t)n);
    memcpy(s + n, seq, (size_t)n);
    for (int64_t i = 0; i < m; i++) f[i] = -1;
    for (int64_t j = 1; j < m; j++) {
        uint8_t c = s[j];
        int64_t i = f[j - k - 1];
        while (i != -1 && c != s[k + i + 1]) {
            if (c < s[k + i + 1]) k = j - i - 1;
            i = f[i];
        }
        if (c != s[k + i + 1]) {
            if (c < s[k]) k = j;
            f[j - k] = -1;
        } else {
            f[j - k] = i + 1;
        }
    }
    free(s);
    free(f);
    return k;
}

/* RotateSequence (seqhash.go:127-138) */
void po_rotate_sequence(const uint8_t *seq, int64_t n, uint8_t *out) {
    int64_t r = po_booth_least_rotation(seq, n);
    memcpy(out, seq + r, (size_t)(n - r));
    memcpy(out + (n - r), seq, (size_t)r);
}

/* Hash (seqhash.go:141-223) for seq_type 0 DNA, 1 RNA, 2 PROTEIN.  Returns 0 and the BLAKE3 digest of the
 * deterministic sequence; 1 letter outside the alphabet (*err_pos = its byte index); 2 double-stranded
 * protein; 3 a byte >= 0x80 first (*err_pos = its byte index). */
int po_seqhash(const uint8_t *seq, int64_t n, int seq_type, int circular, int double_stranded, uint8_t digest[32], int64_t *err_pos) {
    static const char nucleic[] = "ATUGCYRSWKMBDHVNZ", protein[] = "ACDEFGHIKLMNPQRSTVWYUO*BXZ";
    const char *alphabet = seq_type == 2 ? protein : nucleic;
    uint8_t *s = malloc(n ? (size_t)n : 1);
    *err_pos = 0;
    for (int64_t i = 0; i < n; i++) {
        uint8_t c = seq[i];
        if (c >= 0x80) { *err_pos = i; free(s); return 3; }
        if (c >= 'a' && c <= 'z') c -= 32;             /* strings.ToUpper */
        if (seq_type == 1 && c == 'U') c = 'T';        /* strings.ReplaceAll(sequence, "U", "T") */
        if (c == 0 || !strchr(alphabet, c)) { *err_pos = i; free(s); return 1; }
        s[i] = c;
    }
    if (seq_type == 2 && double_stranded) { free(s); return 2; }
    uint8_t *a = malloc(n ? (size_t)n : 1), *rc = malloc(n ? (size_t)n : 1), *b = malloc(n ? (size_t)n : 1);
    for (int64_t i = 0; i < n; i++) rc[i] = sh_complement(s[n - 1 - i]); /* transform.ReverseComplement */
    const uint8_t *det = s;
    if (circular && double_stranded) {
        po_rotate_sequence(s, n, a);
        po_rotate_sequence(rc, n, b);
        det = memcmp(a, b, (size_t)n) <= 0 ? a : b;    /* sort.Strings, first element */
    } else if (circular) {
        po_rotate_sequence(s, n, a);
        det = a;
    } else if (double_stranded) {
        det = memcmp(s, rc, (size_t)n) <= 0 ? s : rc;
    }
    po_blake3(det, (uint64_t)n, digest);
    free(s); free(a); free(b); free(rc);
    return 0;
}

/* ---- batch driver (timed CPU arm): sequences handed out one at a time to nthreads threads ---------- */
typedef struct {
    const uint8_t *seqs;
    const uint64_t *offsets;
    int seq_type, circular, ds;
    uint8_t *digest;
    int32_t *err_code;
    int64_t *err_pos;
} sh_batch;

static void sh_one(void *arg, uint64_t i) {
    sh_batch *b = arg;
    int64_t pos = 0;
    int code = po_seqhash(b->seqs + b->offsets[i], (int64_t)(b->offsets[i + 1] - b->offsets[i]), b->seq_type, b->circular, b->ds,
                          b->digest + 32 * i, &pos);
    if (code) memset(b->digest + 32 * i, 0, 32);
    b->err_code[i] = code;
    b->err_pos[i] = pos;
}

int po_seqhash_batch(const uint8_t *seqs, const uint64_t *offsets, uint64_t n, int seq_type, int circular, int double_stranded,
                     int nthreads, uint8_t *digest, int32_t *err_code, int64_t *err_pos) {
    sh_batch b = {seqs, offsets, seq_type, circular, double_stranded, digest, err_code, err_pos};
    return po_parallel_for(n, nthreads, 1, sh_one, &b);
}
