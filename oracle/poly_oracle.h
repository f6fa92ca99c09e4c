/*
 * oracle/poly_oracle.h -- CPU restatement of the bebop/poly hot path: every function liboracle.so exports.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under oracle/ is part of the product: it
 * may be imported/linked/executed only by tests/, __graft_entry__.smoke() and
 * bench.py's cpu_baseline / --impl reference legs, and only as the checker (or
 * the timed CPU baseline) -- never as a fallback for the CUDA path.
 *
 * Parity pinning: the Go reference cannot be executed in this image (no Go
 * toolchain).  The restatement is pinned by (1) MurmurHash3_x86_32 known-answer
 * vectors (the algorithm lives in github.com/spaolacci/murmur3 v1.1.0, go.mod:12,
 * which is not vendored under /root/reference), (2) a replay of every assertion
 * in the reference's own tests for this path (search/mash/mash_test.go:9-62,
 * search/align/align_test.go:139-292, search/align/example_test.go:82,110,
 * primers/primers_test.go:29-84, primers/pcr/example_test.go:36,46,54) and
 * (3) the golden checksums of SURVEY.md section 8c/8d.  See tests/test_oracle_*.py.
 *
 * All citations are file:line under /root/reference.
 */
#ifndef POLY_ORACLE_H
#define POLY_ORACLE_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define PO_OK 0
#define PO_PANIC (-1)       /* the Go reference would panic on this input        */
#define PO_UNSUPPORTED (-2) /* outside the restated domain (non-ASCII ToUpper)   */
#define PO_NOMEM (-100)     /* a batch driver could not allocate its worker pool */

/* github.com/spaolacci/murmur3 v1.1.0 Sum32WithSeed == MurmurHash3_x86_32. */
uint32_t po_murmur3_32(const uint8_t *data, size_t len, uint32_t seed);

/* search/mash/mash.go:68-104, literally (full re-sort on every qualifying insert).
 * `sketches` has length s and is updated in place exactly as the receiver is. */
int po_mash_sketch_faithful(const uint8_t *seq, int64_t len, int k, int s, uint32_t *sketches);
/* Closed form of the same function (SURVEY 8a row a3): identical results. */
int po_mash_sketch_closed(const uint8_t *seq, int64_t len, int k, int s, uint32_t *sketches);

/* search/mash/mash.go:107-135.  `a` is the receiver.  Writes the matching count. */
int po_mash_similarity(const uint32_t *a, int sa, const uint32_t *b, int sb,
                       int64_t *same, double *similarity);
/* search/mash/mash.go:138-140. */
int po_mash_distance(const uint32_t *a, int sa, const uint32_t *b, int sb, double *distance);

/* Batch driver used for CPU-baseline timing: one fresh zeroed 4*s-byte sketch per
 * read (as mash.New does, mash.go:59-65), reads in [offsets[i], offsets[i+1]).
 * variant 0 = faithful, 1 = closed form.  out is n*s words (padded layout).
 * If out == NULL the sketches are allocated, computed and freed per read (pure
 * timing mode; a digest of the per-read word sums is returned through checksum). */
int po_mash_sketch_batch(const uint8_t *bases, const uint64_t *offsets, uint64_t n, int k, int s,
                         int variant, int nthreads, uint32_t *out, uint64_t *checksum);

/* search/align/align.go:171-203 (score + first-max position; traceback is out of
 * scope).  lut_a / lut_b map a byte to its index in the first / second alphabet
 * (-1 = "Symbol not in alphabet", alphabet/alphabet.go:35-41); table is
 * n_a x n_b row-major (search/align/matrix/matrix.go:28-38).
 * err_code: 0 none, 1 symbol of a not in first alphabet, 2 symbol of b not in
 * second alphabet; err_pos = index of the offending byte in that string. */
int po_sw_score(const uint8_t *a, int64_t la, const uint8_t *b, int64_t lb,
                const int16_t *lut_a, const int16_t *lut_b, const int64_t *table, int n_b,
                int64_t gap, int64_t *score, int64_t *max_row, int64_t *max_col,
                int32_t *err_code, int64_t *err_pos);

/* search/align/align.go:171-232 in full (score + the two aligned strings). */
int po_sw_align(const uint8_t *a, int64_t la, const uint8_t *b, int64_t lb, const int16_t *lut_a,
                const int16_t *lut_b, const int64_t *table, int n_b, int64_t gap, int64_t *score,
                uint8_t *out_a, uint8_t *out_b, int64_t cap, int64_t *out_len, int32_t *err_code,
                int64_t *err_pos);

/* search/align/align.go:100-166 in full (score + the two aligned strings). */
int po_nw_align(const uint8_t *a, int64_t la, const uint8_t *b, int64_t lb, const int16_t *lut_a,
                const int16_t *lut_b, const int64_t *table, int n_b, int64_t gap, int64_t *score,
                uint8_t *out_a, uint8_t *out_b, int64_t cap, int64_t *out_len, int32_t *err_code,
                int64_t *err_pos);

/* search/align/align.go:100-166, score only. */
int po_nw_score(const uint8_t *a, int64_t la, const uint8_t *b, int64_t lb,
                const int16_t *lut_a, const int16_t *lut_b, const int64_t *table, int n_b,
                int64_t gap, int64_t *score, int32_t *err_code, int64_t *err_pos);

/* io/fastq/fastq.go:88-99,117-214 over a whole buffer (see the definition for the error codes). */
int po_fastq_parse(const uint8_t *text, uint64_t n, uint64_t *seq_start, uint64_t *seq_len, uint64_t cap,
                   uint64_t *n_records, int32_t *err_code, uint64_t *err_line);

/* io/fasta/fasta.go:72-77,96-118,149-243 (fasta.Parse) over a whole buffer, with the bufio.Reader
 * underneath modelled literally; alias=1 keeps the reference's use of `line` after Peek(1)
 * (fasta.go:192), alias=0 copies the line first.  See fasta_oracle.c for the error codes. */
int po_fasta_parse(const uint8_t *text, uint64_t n, uint32_t max_line_size, int alias, uint8_t *seq,
                   uint64_t seq_cap, uint64_t *seq_off, uint8_t *name, uint64_t name_cap,
                   uint64_t *name_off, uint64_t rec_cap, uint64_t *n_records, int32_t *err_code,
                   uint64_t *err_line);

/* transform/transform.go:15-23,78-109. out has room for len bytes. */
void po_reverse_complement(const uint8_t *seq, int64_t len, uint8_t *out);

/* primers/primers.go:70-105.  Returns PO_PANIC for the empty string
 * (primers.go:89 indexes sequence[len-1]) and PO_UNSUPPORTED if a byte >= 0x80
 * is present (strings.ToUpper would re-encode it). */
int po_santalucia(const uint8_t *seq, int64_t len, double cp, double na, double mg,
                  double *tm, double *dh, double *ds);
/* primers/primers.go:121-128. */
int po_melting_temp(const uint8_t *seq, int64_t len, double *tm);

/* ---- batch drivers (batch_drivers.c): a static parallel-for of per-item calls, for bench.py's
 * CPU legs only.  checksum (may be NULL) receives a digest so that the work cannot be elided. */
int po_sw_score_batch(const uint8_t *queries, const uint64_t *offsets, uint64_t n, const uint8_t *templ, int64_t templ_len,
                      const int16_t *lut_a, const int16_t *lut_b, const int64_t *table, int n_b, int64_t gap, int nthreads,
                      int64_t *score, uint64_t *checksum);
int po_melting_temp_batch(const uint8_t *bases, const uint64_t *offsets, uint64_t n, int nthreads, double *tm, uint64_t *checksum);
int po_mash_similarity_block(const uint32_t *sk, uint64_t n, int s, uint64_t row_lo, uint64_t row_hi, uint64_t col_lo,
                             uint64_t col_hi, int nthreads, uint32_t *same, uint64_t *checksum);

/* ---- seqhash_oracle.c: seqhash/seqhash.go:78-223 and BLAKE3 (hash mode, 32-byte output) */
void po_blake3(const uint8_t *in, uint64_t len, uint8_t out[32]);
int64_t po_booth_least_rotation(const uint8_t *seq, int64_t n);
void po_rotate_sequence(const uint8_t *seq, int64_t n, uint8_t *out);
int po_seqhash(const uint8_t *seq, int64_t n, int seq_type, int circular, int double_stranded, uint8_t digest[32], int64_t *err_pos);
int po_seqhash_batch(const uint8_t *seqs, const uint64_t *offsets, uint64_t n, int seq_type, int circular, int double_stranded,
                     int nthreads, uint8_t *digest, int32_t *err_code, int64_t *err_pos);

/* ---- pair_oracle.c: po_sw_score / po_nw_score over a list of (a, b) index pairs */
int po_pair_scores(int global, const uint8_t *a, const uint64_t *off_a, const uint8_t *b, const uint64_t *off_b, const uint32_t *pair_a,
                   const uint32_t *pair_b, uint64_t n, const int16_t *lut_a, const int16_t *lut_b, const int64_t *table, int n_b,
                   int64_t gap, int nthreads, int64_t *score, int32_t *err_code, int64_t *err_pos);

/* ---- clone_oracle.c: clone/clone.go:138-355 (CutWithEnzyme, CircularLigate) */
void co_free(void *p);
int co_cut(const uint8_t *part, int64_t L, int circular, int directional, const uint8_t *fsite, int64_t fl, const uint8_t *rsite,
           int64_t rl, const uint8_t *recog, int64_t recl, int64_t skip, int64_t ohl, uint8_t **out, uint64_t *out_bytes, int64_t *n_frag);
int co_cut_batch(const uint8_t *parts, const uint64_t *offsets, const uint8_t *circular, uint64_t n_parts, const uint8_t *const *sites,
                 const int64_t *site_lens, const int64_t *skip_ohl, int n_enz, int directional, int nthreads, int64_t *n_frag, int32_t *status);
void co_circular_ligate(const uint8_t *frags, int64_t n, uint8_t **clones, uint64_t *clone_bytes, int64_t *n_clones, uint8_t **loops,
                        uint64_t *loop_bytes, int64_t *n_loops);

/* ---- fold_oracle.c: fold.go and seqfold.go (Zuker) */
void fo_set_table(int kind, int t, int count, const char *keys, const double *h, const double *s);
void fo_set_multibranch(int kind, const double *mb);
int fo_fold(const char *raw, int64_t n, double temp, double *mfe, char *db, int64_t *db_len, char **structs);
int fo_probe(const char *raw, int64_t n, double temp, int which, int a, int b, int cc, int d, double *out);
void fo_pair(const char *s, int a, int b, int c, int d, char *out);
void fo_free(void *p);
int fo_fold_batch(const uint8_t *seqs, const uint64_t *off, uint64_t n, double temp, double *mfe, uint8_t *db, uint64_t *db_len,
                  int32_t *status, int threads);

/* ---- fragment_oracle.c: synthesis/fragment/fragment.go */
void fr_set_table(const uint8_t *keys, const int32_t *counts);
double fr_set_efficiency(const uint8_t *bytes, const uint64_t *off, uint64_t n);
int fr_next_overhangs(const uint8_t *bytes, const uint64_t *off, uint64_t n, uint8_t *cands, double *eff);
int fr_fragment(const uint8_t *seq_in, int64_t len_in, int64_t minFragmentSize, int64_t maxFragmentSize, const uint8_t *ex,
                const uint64_t *ex_off, uint64_t n_ex, const uint8_t *inc, const uint64_t *inc_off, uint64_t n_inc, double *eff,
                int64_t *err_min, int64_t *err_max, uint64_t *ends, uint64_t *n_ends);
int fr_fragment_batch(const uint8_t *seqs, const uint64_t *off, uint64_t n, int64_t min, int64_t max, const uint8_t *ex,
                      const uint64_t *ex_off, uint64_t n_ex, const uint8_t *inc, const uint64_t *inc_off, uint64_t n_inc, int32_t *status,
                      double *eff, int64_t *err_min, int64_t *err_max, uint64_t *ends, const uint64_t *ends_off, uint64_t *n_ends,
                      int threads);
int fr_set_efficiency_batch(const uint8_t *bytes, const uint64_t *off, const uint64_t *set_off, uint64_t n_sets, double *eff, int threads);
int fr_next_overhangs_batch(const uint8_t *bytes, const uint64_t *off, const uint64_t *set_off, uint64_t n_sets, uint8_t *cands,
                            uint32_t *n_cands, double *eff, int threads);

#ifdef __cplusplus
}
#endif
#endif
