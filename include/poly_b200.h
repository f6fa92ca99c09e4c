/*
 * poly_b200.h -- C ABI of libpolyb200.so: the H100 (sm_90a) implementation of
 * bebop/poly's search/mash sketching hot path plus the two secondary batched
 * kernels (search/align.SmithWaterman score, primers.SantaLucia).
 *
 * The reference is pure Go and has NO FFI/plugin interface (SURVEY.md 8b); the
 * drop-in boundary is the exported Go API of three leaf packages.  Each entry
 * point below names the reference function it replaces (file:line in
 * bebop/poly); INTEGRATION.md shows the cgo binding for each.
 *
 * Conventions
 *   - plain C: pointers + sizes, no C++/torch types, no exceptions across the ABI;
 *   - every function returns PG_OK (0) or a PG_ERR_* code; pg_last_error() gives a
 *     thread-local message;
 *   - the caller owns every buffer; the library never retains a caller pointer
 *     after return (cgo pointer rule) and never frees caller memory;
 *   - functions without the _dev suffix take HOST pointers (pageable or pinned) and
 *     perform the host<->device copies themselves; *_dev functions take DEVICE
 *     pointers on the calling thread's device (pg_thread_device / pg_init) plus a
 *     CUDA stream (cudaStream_t cast to void*, NULL = the legacy default stream) and
 *     only enqueue work: the sketch, Smith-Waterman / Needleman-Wunsch score, Tm and
 *     synth *_dev entry points never wait for the device.  Exceptions, which
 *     synchronise the given stream before returning because a host decision depends
 *     on a device result: pg_mash_distance_block_dev / pg_mash_distance_sparse_dev /
 *     pg_mash_cluster_dev / pg_mash_dereplicate_dev (sortedness and bucket sizes choose the
 *     algorithm), pg_fastq_ingest_dev /
 *     pg_fasta_ingest_dev (they return counts and the error position by value),
 *     pg_seqhash_batch_dev (waits for earlier work on the stream to read the total length, but not
 *     for its own kernels), and
 *     pg_mash_sketch_batch_dev for ragged batches the threshold path does not take
 *     (s < 2, or more than 4 Mi row x item slots) when they hold few long sequences, and
 *     pg_mash_sketch_groups_dev and pg_mash_sketcher_add_dev (they size and decide their passes over hash ranges on
 *     the host);
 *   - a ragged batch of n items passes n + 1 offsets, item i being [offsets[i], offsets[i+1]).
 *     Offsets must not decrease: the host-pointer entry points return PG_ERR_ARG if they do,
 *     without launching anything;
 *   - there is NO CPU fallback: without a usable sm_90 device every compute entry
 *     point fails with PG_ERR_NO_DEVICE.
 */
#ifndef POLY_B200_H
#define POLY_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PG_OK 0
#define PG_ERR_CUDA 1        /* a CUDA runtime call failed (see pg_last_error)          */
#define PG_ERR_ARG 2         /* invalid argument                                         */
#define PG_ERR_NO_DEVICE 3   /* no CUDA device / not an sm_90 part                       */
#define PG_ERR_PANIC 4       /* >= 1 item hits an input on which the Go reference panics */
#define PG_ERR_UNSUPPORTED 5 /* >= 1 item is outside the supported domain                */
#define PG_ERR_NOMEM 6

/* per-item status codes (status arrays) */
#define PG_ITEM_OK 0
#define PG_ITEM_PANIC 1       /* reference panics (index out of range) on this item     */
#define PG_ITEM_UNSUPPORTED 2 /* e.g. byte >= 0x80 passed to SantaLucia (ToUpper)       */
#define PG_ITEM_FOLD_NOT_NUCLEIC 3 /* fold: "the sequence %s is not RNA or DNA"           */
#define PG_ITEM_FOLD_INTERNAL 4    /* fold: one of the reference's internal errors fired  */
#define PG_ITEM_FRAGMENT_MIN_GT_MAX 5  /* fragment: "minFragmentSize (%d) larger than maxFragmentSize (%d)" */
#define PG_ITEM_FRAGMENT_MIN_LT_12 6   /* fragment: "minFragmentSize must be equal to or greater than 12 . Got size of %d" */
#define PG_ITEM_FRAGMENT_NO_POSITION 7 /* fragment: "bestOverhangPosition failed by equaling zero" */

/* ---- library / device management -------------------------------------------- */
int pg_version(void);
/* Choose the process-default CUDA device (one process per GPU layout).  Optional: the first
 * compute call initialises the current CUDA device (device 0 unless the caller changed it).
 * The library keeps one context per device and serves any number of devices from one process:
 *   - pg_thread_device(d) binds the CALLING THREAD's later calls to device d (-1: back to the
 *     process default) -- for hosts that drive several GPUs themselves (Go: after
 *     runtime.LockOSThread());
 *   - the *_multi entry points shard one batch over several devices on their own.
 * Entry points are safe to call concurrently from many threads: host-pointer entry points are
 * serialised per device, *_dev entry points only enqueue work on the caller's stream. */
int pg_init(int device);
int pg_thread_device(int device);
/* Move the calling thread to the CPUs of the NUMA node the device is attached to and prefer that
 * node for memory it allocates afterwards (call before pg_host_alloc).  Best effort; *node (may be
 * NULL) receives the node or -1 when nothing was done. */
int pg_numa_bind_thread(int device, int *node);
int pg_shutdown(void);
const char *pg_last_error(void);
int pg_device_count(int *count);
int pg_device_sm_count(int *sms);
/* Pinned host memory for callers that want full PCIe bandwidth (optional). */
int pg_host_alloc(void **ptr, size_t bytes);
int pg_host_free(void *ptr);
/* Device memory helpers for C/Go callers of the *_dev entry points. */
int pg_dev_alloc(void **dptr, size_t bytes);
int pg_dev_free(void *dptr);
int pg_memcpy_h2d(void *dst_dev, const void *src_host, size_t bytes, void *stream);
int pg_memcpy_d2h(void *dst_host, const void *src_dev, size_t bytes, void *stream);
int pg_stream_sync(void *stream);

/* ---- mash.Sketch -- replaces (*Mash).Sketch on a fresh mash.New(k, s) -----------
 * search/mash/mash.go:59-65 (New) and :68-104 (Sketch), one sketch per read.
 *
 * Read i is bases[offsets[i] .. offsets[i+1]) (raw bytes, any value; the hash is
 * MurmurHash3_x86_32(seed 0) of the k raw bytes, mash.go:74-76).  With
 * n_i = max(len_i - k, 0) hashes (mash.go:73 visits L-k windows, not L-k+1):
 *   n_i <  s : out row i = the n_i hashes in positional order   (mash.go:81-84)
 *   n_i >= s : out row i = ascending bottom-s multiset          (mash.go:87-102)
 * count[i] = min(n_i, s) informative words; row i starts at out + i*row_stride.
 * row_stride must be >= the largest count of the batch (>= s with PG_SKETCH_PAD_ZERO; the host
 * entry points check this for the whole batch before launching anything); words
 * [count[i], row_stride) of a row are written as zeros -- the zero tail a fresh Mash holds,
 * as far as the row reaches.  With PG_SKETCH_PAD_ZERO every row is a full Go array of s words.
 * status[i] (may be NULL) reports per-read PG_ITEM_PANIC for s in {0,1} inputs on
 * which mash.go:96-98 indexes Sketches[-1]; k < 0 or s < 0 is PG_ERR_ARG.
 * Reads may be of any length (a batch of few long sequences is cut into slices that are sketched
 * in parallel and merged) and k and s of any size: in the n_i >= s regime, sketches above 16384 words
 * or k above 1024 take a slower global-memory path instead of the shared-memory kernels.
 */
#define PG_SKETCH_PAD_ZERO 1u
/* Host-buffer entry points only: write nothing but the count[i] informative words of a row -- the literal
 * behaviour of (*Mash).Sketch, which never touches Sketches[n:s] in the n < s regime (mash.go:73-80).  A Go
 * caller that hands in a fresh make([]uint32, n*s) slab (zeroed by the runtime) gets full Sketches arrays
 * without the library writing 4*s bytes per read; a reused array keeps its old tail, as in the reference. */
#define PG_SKETCH_TAIL_KEEP 2u

int pg_mash_sketch_batch(const uint8_t *bases, const uint64_t *offsets, uint64_t n_reads, int32_t k,
                         int32_t s, uint32_t flags, uint32_t *out, uint64_t row_stride,
                         uint32_t *count, int32_t *status);
/* Same, for fixed-length reads stored back to back (read i at bases + i*read_len):
 * no offsets array, count is min(max(read_len-k,0), s) for every read. */
int pg_mash_sketch_uniform(const uint8_t *bases, uint64_t n_reads, uint32_t read_len, int32_t k,
                           int32_t s, uint32_t flags, uint32_t *out, uint64_t row_stride,
                           int32_t *status);
/* Device-resident variants (inputs already in HBM, outputs stay in HBM). */
int pg_mash_sketch_batch_dev(const uint8_t *d_bases, const uint64_t *d_offsets, uint64_t n_reads,
                             uint64_t max_read_len, int32_t k, int32_t s, uint32_t flags,
                             uint32_t *d_out, uint64_t row_stride, uint32_t *d_count,
                             int32_t *d_status, void *stream);
int pg_mash_sketch_uniform_dev(const uint8_t *d_bases, uint64_t n_reads, uint32_t read_len,
                               int32_t k, int32_t s, uint32_t flags, uint32_t *d_out,
                               uint64_t row_stride, int32_t *d_status, void *stream);
/* Fused sketch + all-gather over NVLink peer memory (one process per GPU).  Every rank owns a
 * "gathered" buffer of world*n_local rows; gathered_ptrs[p] is that buffer on rank p as seen from
 * THIS process (own pointer for p == rank, pg_ipc_import()ed peer mappings otherwise).  The
 * sketch kernel stores each finished tile / row straight into all of them at row offset
 * rank*n_local (TMA bulk stores to peer addresses in the fill regime), so the transfer overlaps
 * the hashing tile by tile and no separate collective pass runs.  Rows are compact
 * (row stride = min(max(read_len-k,0), s) words).  The caller must synchronise the stream and
 * barrier across ranks before reading its gathered buffer.  n_local MUST be the same on all
 * ranks (the row offset is rank*n_local; use the _scatter_dev variant for unequal shards); world <= 8. */
#define PG_MAX_PEERS 8
#define PG_IPC_HANDLE_BYTES 64
int pg_ipc_export(void *dptr, uint8_t handle[PG_IPC_HANDLE_BYTES]);
int pg_ipc_import(const uint8_t handle[PG_IPC_HANDLE_BYTES], void **dptr);
int pg_ipc_close(void *dptr);
int pg_mash_sketch_uniform_gather_dev(const uint8_t *d_bases, uint64_t n_local, uint32_t read_len,
                                      int32_t k, int32_t s, void *const *gathered_ptrs,
                                      int32_t world, int32_t rank, void *stream);
/* The same with an explicit row offset: the n_local sketches go to rows [row_offset, row_offset +
 * n_local) of each of the n_dst buffers (dst_ptrs[self] is the local one).  Shards may then differ
 * in size; any k, any n_local (rows the TMA path does not take are stored by the generic kernels). */
int pg_mash_sketch_uniform_scatter_dev(const uint8_t *d_bases, uint64_t n_local, uint32_t read_len,
                                       int32_t k, int32_t s, void *const *dst_ptrs, int32_t n_dst,
                                       int32_t self, uint64_t row_offset, void *stream);

/* ---- canonical k-mers: PG_KMER_CANONICAL, a flag of the grouped sketch, the sketcher and the screen ----
 * Mash hashes canonical k-mers: a k-mer and its reverse complement are one k-mer, so contigs of either orientation and
 * reads of either strand meet.  With the flag (pg_mash_sketch_groups_flags, pg_mash_sketcher_create_flags,
 * pg_mash_screen_create_flags and their _dev forms) the windows of a record of length L >= k >= 1 are:
 *   - Windows: positions 0 .. L - k, so L - k + 1 of them and none when L < k.  This is Mash's k-mer set, one more than
 *     the forward mode's L - k: the forward mode skips the last window (mash.go:73), which would break strand
 *     symmetry.  No window crosses a record.
 *   - Canonical form: for w = bases[p .. p+k), rc(w)[i] = complement(w[k-1-i]), complement being
 *     transform.complementTable (upper- and lower-case IUPAC letters; every unlisted byte maps to 0).
 *     canon(w) = w if w <= rc(w) in unsigned byte order (memcmp), else rc(w).
 *   - Hash: murmur3.Sum32(canon(w)), the same MurmurHash3_x86_32 with seed 0 over k raw bytes as the forward mode.
 *     Case is not folded and no byte is skipped.
 *   - Strand symmetry: a record whose bytes all lie in ABCDGHKMNRSTVWY and their lower case may be replaced by its
 *     reverse complement without changing any row, count or screen result.
 *   - Counting: min_copies and the screen's pool counts count a k-mer and its reverse complement together.
 *   - Mash's choice: on upper-case ACGT the canonical strand is Mash's (memcmp(kmer_fwd, kmer_rev) <= 0); only the
 *     hash function differs from Mash.
 * Everything else (rows, min_copies, the sketcher's caps, budget and completeness, the screen's results, winners and
 * samples) is as documented for each call, over this window multiset instead of the forward one.  Errors, added right
 * after each call's k < 0 rule: a flag bit other than PG_KMER_CANONICAL, and k == 0 with PG_KMER_CANONICAL (no strand to
 * choose), both PG_ERR_ARG before any device work.  flags == 0 is the call without the flag, byte for byte. */
#define PG_KMER_CANONICAL 1u

/* ---- grouped sketch: one sketch per group of records (`mash sketch genome.fa`, `mash sketch -r -m M reads.fq`) ----
 * A draft assembly is many contigs and a read set many reads; Mash sketches each as one set.  Records are ragged
 * as in pg_mash_sketch_batch (record i = bases[offsets[i] .. offsets[i+1])); group g is records
 * [group_offsets[g], group_offsets[g+1]).  The groups partition the records: group_offsets[0] == 0,
 * group_offsets[n_groups] == n_records, never decreasing; empty groups are allowed.
 *   - Windows: a record of length L contributes the windows (*Mash).Sketch hashes, positions 0 .. L - k - 1
 *     (mash.go:73; none when L <= k), each murmur3.Sum32 over its raw bytes: forward strand, case-sensitive, any
 *     byte value, as the screen counts them.  No window crosses a record.  pg_mash_sketch_groups_flags (+ _dev) with
 *     PG_KMER_CANONICAL takes the canonical windows instead (above).
 *   - c_g(v) = the windows of group g's records whose hash is v.  Row g = the distinct values v with
 *     c_g(v) >= min_copies in ascending order, the smallest count[g] = min(q_g, s) of them (q_g: how many qualify),
 *     then zeros up to row_stride.  The row is a set (no value twice) and always ascending, also when q_g < s; a
 *     real hash can be 0, so count[g] tells the tail apart.  A group of one record with L - k >= s, min_copies 1 and
 *     no repeated value in its bottom-s multiset gives pg_mash_sketch_batch's row of that record, word for word.
 *   - Row g depends only on the multiset of group g's windows: not on the order of its records, the order of the
 *     groups, the other groups of the call or how a batch of groups is split over calls.  Rows are exact: whatever
 *     passes the device takes, every count is exact.
 *   - Errors, checked in this order before any device work: a null out or count with n_groups > 0; k < 0 (as for
 *     the sketch calls); s < 1; min_copies < 1; row_stride < s; a null buffer with work to do (group_offsets and
 *     offsets when n_groups > 0; bases when the records hold a byte, or in _dev when n_records > 0); in the host call, group offsets that do not partition
 *     the records or record offsets that decrease: all PG_ERR_ARG.  The _flags forms check their flags right after
 *     k < 0 (above).  PG_ERR_NOMEM when device memory runs out.
 *     n_groups == 0 is valid and needs no buffers.  _dev trusts its offsets as pg_mash_sketch_batch_dev does.
 *   - Passes: pass t counts, for every group still open, the windows whose hash lies in the group's next range of
 *     values into an open-addressing table; values with count >= min_copies are appended to the row.  The first
 *     range admits about s + 6 sqrt(s) + 48 windows, so a genome of distinct windows finishes in one pass; a read set
 *     filtered at min_copies >= 2 takes a few.  Later passes walk only the records of open groups.  _dev
 *     synchronises `stream` (the host decides the passes).
 *   - Device memory: 8 (n_records + 1) x 2 + 16 (n_groups + 1) + 32 n_groups bytes besides the caller's buffers,
 *     and per pass 32 bytes per table slot, at most 2^26 slots (2 GiB); a table holds twice the distinct values its
 *     range is expected to admit.  The host call also stages the bases, offsets, rows and counts. */
int pg_mash_sketch_groups(const uint8_t *bases, const uint64_t *offsets, uint64_t n_records, const uint64_t *group_offsets,
                          uint64_t n_groups, int32_t k, int32_t s, uint32_t min_copies, uint32_t *out, uint64_t row_stride,
                          uint32_t *count);
int pg_mash_sketch_groups_dev(const uint8_t *d_bases, const uint64_t *d_offsets, uint64_t n_records, const uint64_t *d_group_offsets,
                              uint64_t n_groups, int32_t k, int32_t s, uint32_t min_copies, uint32_t *d_out, uint64_t row_stride,
                              uint32_t *d_count, void *stream);
/* the same with flags (0 or PG_KMER_CANONICAL) after min_copies; flags == 0 is the call above */
int pg_mash_sketch_groups_flags(const uint8_t *bases, const uint64_t *offsets, uint64_t n_records, const uint64_t *group_offsets,
                                uint64_t n_groups, int32_t k, int32_t s, uint32_t min_copies, uint32_t flags, uint32_t *out,
                                uint64_t row_stride, uint32_t *count);
int pg_mash_sketch_groups_flags_dev(const uint8_t *d_bases, const uint64_t *d_offsets, uint64_t n_records, const uint64_t *d_group_offsets,
                                    uint64_t n_groups, int32_t k, int32_t s, uint32_t min_copies, uint32_t flags, uint32_t *d_out,
                                    uint64_t row_stride, uint32_t *d_count, void *stream);

/* ---- grouped sketch grown in place: read sets larger than device memory, added batch by batch ----
 * A sketcher holds G groups (fixed at create), k, s, m = min_copies and a budget B = max_values: the most distinct
 * values one group keeps between adds.  Windows are exactly those of pg_mash_sketch_groups: positions 0 .. L - k - 1
 * of each record, murmur3 over the raw bytes, forward strand, never crossing a record; a sketcher made by
 * pg_mash_sketcher_create_flags with PG_KMER_CANONICAL takes the canonical windows (above) in every add, and the
 * one-shot call it equals is then pg_mash_sketch_groups_flags with the same flag.  c_g(v) = the windows of every
 * record added to group g so far whose hash is v.
 *   - Per group the sketcher keeps a cap C_g, which starts at 2^32 and never grows, and a state: every value v < C_g
 *     with c_g(v) >= 1, and beside each one min(c_g(v), m).  Invariant: every count below C_g is exact.  An add of
 *     records to group g:
 *       1. V = the distinct values below the old C_g, with counts over the old state plus this batch's windows;
 *          Q = {v in V : c >= m}.
 *       2. t_s = (s-th smallest value of Q) + 1, or 2^32 if |Q| < s.  Lossless: counts only grow, so no value at or
 *          above t_s can ever enter the row.
 *       3. t_B = the (B+1)-th smallest value of V, or 2^32 if |V| <= B.  This is the budget.
 *       4. C_g = min(C_g, t_s, t_B); the state keeps V below it.
 *     Batch windows at or above the old C_g are discarded.  Groups that get no records in an add are unchanged.
 *   - Rows, readable at any time, changing nothing: row g holds the values of Q below C_g, ascending: n_values[g] =
 *     min(|Q below C_g|, s) of them, then zeros up to row_stride.  complete[g] = (n_values[g] == s) || (C_g == 2^32).
 *     held[g] = the number of values in the state.
 *   - Properties:
 *       complete => equal: if complete[g], row g and n_values[g] equal pg_mash_sketch_groups over the concatenation
 *         of every record added to g, byte for byte, whatever the split (empty adds, one-record adds, a group spread
 *         over many adds, adds that start or end inside a group);
 *       always a prefix: row g is always the first n_values[g] words of that one-shot row (the values below C_g are
 *         the smallest qualifying values overall, and their counts are exact);
 *       with m = 1 every group is always complete and held[g] <= s after every add.
 *     held shows how close a group is to its budget; an incomplete group asks for a larger max_values.
 *   - Batch layout: records [group_offsets[i], group_offsets[i+1]) of the batch belong to group first_group + i, with
 *     group_offsets[0] == 0 and group_offsets[n_batch_groups] == n_records (the one-shot layout with a group base).
 *   - Errors, checked in this order before any device work (PG_ERR_ARG):
 *       create: a null out; n_groups == 0 or n_groups > 2^32 - 1; k < 0; (create_flags: an unknown flag bit; k == 0
 *         with PG_KMER_CANONICAL); s < 1; min_copies < 1; max_values < s.
 *       add: a null sketcher (no device needed); n_records == 0 with n_batch_groups == 0 is a valid no-op;
 *         first_group + n_batch_groups > G; n_records == 0 is then a valid no-op; a null offsets or group_offsets, or a
 *         null bases (in the host add only when the records hold a byte); in the host add, group offsets that do not
 *         partition the records, or record offsets that decrease.  add_dev trusts its offsets.
 *       rows: a null sketcher; first + count > G; row_stride < s; a null out or n_values with count > 0.  complete and
 *         held may be NULL.
 *     PG_ERR_NOMEM when memory runs out.  After any error the sketcher holds exactly what it held before: an add builds
 *     the new state in new buffers and swaps it in at the end.
 *   - Synchronisation: add_dev synchronises its stream (the host plans the passes); rows_dev only enqueues, and a later
 *     add waits for it on the device before it releases the state rows_dev reads.
 *   - Threads: one lock per sketcher; adds are serialised and rows waits for a running add.  The sketcher lives on the
 *     device current at create.
 *   - Device memory: the state takes 8 bytes per held value (uint32 value, uint32 saturated count), plus 8 (G + 1)
 *     bytes of segment offsets and 8 G of caps.  During an add: the old and the new state together, the add's list of
 *     kept values (12 bytes each, twice while it is sorted), and per pass 44 bytes per table slot, at most 2^26 slots;
 *     a table holds twice the distinct values its range is expected to admit.  The host add also stages the batch. */
typedef struct pg_mash_sketcher pg_mash_sketcher;
int pg_mash_sketcher_create(uint64_t n_groups, int32_t k, int32_t s, uint32_t min_copies, uint64_t max_values, pg_mash_sketcher **out);
/* the same with flags (0 or PG_KMER_CANONICAL): the mode belongs to the sketcher, add and rows are unchanged */
int pg_mash_sketcher_create_flags(uint64_t n_groups, int32_t k, int32_t s, uint32_t min_copies, uint64_t max_values, uint32_t flags,
                                  pg_mash_sketcher **out);
int pg_mash_sketcher_add(pg_mash_sketcher *sk, const uint8_t *bases, const uint64_t *offsets, uint64_t n_records, const uint64_t *group_offsets,
                         uint64_t first_group, uint64_t n_batch_groups);
int pg_mash_sketcher_add_dev(pg_mash_sketcher *sk, const uint8_t *d_bases, const uint64_t *d_offsets, uint64_t n_records,
                             const uint64_t *d_group_offsets, uint64_t first_group, uint64_t n_batch_groups, void *stream);
int pg_mash_sketcher_rows(const pg_mash_sketcher *sk, uint64_t first, uint64_t count, uint32_t *out, uint64_t row_stride, uint32_t *n_values,
                          uint8_t *complete, uint64_t *held);
int pg_mash_sketcher_rows_dev(const pg_mash_sketcher *sk, uint64_t first, uint64_t count, uint32_t *d_out, uint64_t row_stride,
                              uint32_t *d_n_values, uint8_t *d_complete, uint64_t *d_held, void *stream);
int pg_mash_sketcher_free(pg_mash_sketcher *sk);

/* ---- Mash distance between grouped sketches (`mash dist`, `mash dist -d D -v P`, `mash triangle`) ----
 * Inputs are rows as pg_mash_sketch_groups and pg_mash_sketcher_rows write them: rows is n x row_stride uint32 and row
 * i holds count[i] <= s strictly ascending values (unsigned order) in its first words; one s and one k for the call.
 * For query row A (a values) and reference row B (b values), Mash's compareSketches loop:
 *     i = j = common = denom = 0
 *     while denom < s and i < a and j < b:
 *         if A[i] < B[j]: i++   elif B[j] < A[i]: j++   else: i++; j++; common++
 *         denom++
 *     if denom < s: denom += min(a - i, s - denom); denom += min(b - j, s - denom)
 * That is, denom = min(s, |A u B|) and common = the shared values among the denom smallest values of A u B.
 *   - distance: +0.0 if common == denom (two empty rows included); 1.0 if common == 0; else -log(2J / (1 + J)) / k with
 *     J = (double)common / denom, clamped to 1.0 when larger.  Mash's estimate of the per-base mutation rate (1 - ANI).
 *   - p-value (Mash's pValue): 1.0 if common == 0.  Else pQ = 1 / (1 + 4^k / len_q), pR likewise with len_r, 4^k being the
 *     double ldexp(1, 2k); r = pQ pR / (pQ + pR - pQ pR), taken as 0 when that denominator is 0; p = P[Binomial(denom, r)
 *     >= common] (GSL's gsl_cdf_binomial_Q(common - 1, r, denom)), 0 when r == 0.  Computed on the device in double from
 *     the incomplete beta function: its prefactor as a binomial density in Loader's saddle-point form (no log-gamma
 *     differences), then the continued fraction.  Tested against an exact tail for denom up to 2^24: where the exact
 *     p >= 1e-300 the relative error is at most tol(denom) = 4e-12 max(1, sqrt(denom / 10^4)), plus 4 eps |d ln p /
 *     d ln r| for one ulp of r; below 1e-300 the value is in [0, 2e-300].  Never NaN or -0.0.
 *     len is the number of bases Mash records for a sketch (an assembly: the sum of its record lengths), >= 1.
 *   - Properties: swapping the query and reference sets together with their lengths transposes all four outputs bit
 *     for bit (every formula is symmetric); a row against itself gives common = denom = count and distance 0.  The call
 *     cannot tell an incomplete sketcher row (complete[g] == 0) from a small group: passing complete rows is the
 *     caller's job, as k and the canonical mode are.
 *   - Unlike (*Mash).Distance (pg_mash_distance_block), a row with fewer than s values compares as the set it is: the
 *     reference's range early-out makes such a row, whose tail is zeros, distance 1 from everything, itself included.
 * pg_mash_dist (dense, `mash dist`): common, denom, distance and p_value are nq x nr, row-major, query = row; any may be
 * NULL.  A row block is a slice of the queries.
 * pg_mash_dist_within (filtered, `mash dist -d -v`, `mash triangle`): the pairs (pair_q[t], pair_r[t]) with distance <=
 * max_distance and p <= max_p_value, in no particular order, with their common, denom, distance and p_value (each may
 * be NULL).  PG_PAIRS_UPPER keeps only r > q (a set against itself: needs nq == nr).  *n_pairs receives the number of
 * qualifying pairs; if it exceeds pairs_cap the first pairs_cap are stored and the call returns PG_ERR_ARG (as
 * pg_mash_distance_sparse).  The _dev form takes a DEVICE counter d_n_pairs (set on the stream, may exceed pairs_cap)
 * and does not block.
 *   - Lengths may be NULL only when p_value is NULL and, in the filtered form, max_p_value >= 1 (no p-value is computed).
 *   - Errors, checked in this order before any device work, all PG_ERR_ARG: nq or nr > 2^32 - 1; k < 1; s < 1;
 *     row_stride < s; a null rows or count on a non-empty side; null lengths on a non-empty side when a p-value is
 *     needed; in the filtered form a NaN limit, a flag bit other than PG_PAIRS_UPPER, PG_PAIRS_UPPER with nq != nr, a
 *     null pair_q, pair_r or n_pairs; in the host forms only, a count > s, a row that is not strictly ascending, or a
 *     length of 0 where lengths are read.  The _dev forms trust their rows (as _dev calls trust offsets) and read only the
 *     first count words of each.  nq == 0 or nr == 0 is valid.
 *   - Device: one warp merges a pair, over at most 2 s items of the merge.  Rows of s <= 3418 are staged in shared
 *     memory; larger s reads them from global memory.  Both forms only enqueue (_dev) or wait for their own stream.
 *   - Device memory: the _dev forms allocate nothing.  pg_mash_dist stages the references (4 nr (row_stride + 1) bytes,
 *     + 8 nr with lengths) and cuts the queries into blocks whose outputs (4 or 8 bytes per requested output per pair)
 *     stay under 1 GiB, with each block's query rows.  pg_mash_dist_within stages both sets and pairs_cap entries of
 *     every requested list (8 bytes of pair ids, 4 + 4 + 8 + 8 for the others). */
int pg_mash_dist(const uint32_t *q_rows, const uint32_t *q_count, uint64_t nq, const uint32_t *r_rows, const uint32_t *r_count, uint64_t nr,
                 uint64_t row_stride, int32_t s, int32_t k, const uint64_t *q_length, const uint64_t *r_length, uint32_t *common, uint32_t *denom,
                 double *distance, double *p_value);
int pg_mash_dist_dev(const uint32_t *d_q_rows, const uint32_t *d_q_count, uint64_t nq, const uint32_t *d_r_rows, const uint32_t *d_r_count, uint64_t nr,
                     uint64_t row_stride, int32_t s, int32_t k, const uint64_t *d_q_length, const uint64_t *d_r_length, uint32_t *d_common,
                     uint32_t *d_denom, double *d_distance, double *d_p_value, void *stream);
int pg_mash_dist_within(const uint32_t *q_rows, const uint32_t *q_count, uint64_t nq, const uint32_t *r_rows, const uint32_t *r_count, uint64_t nr,
                        uint64_t row_stride, int32_t s, int32_t k, const uint64_t *q_length, const uint64_t *r_length, double max_distance,
                        double max_p_value, uint32_t flags, uint32_t *pair_q, uint32_t *pair_r, uint32_t *common, uint32_t *denom, double *distance,
                        double *p_value, uint64_t pairs_cap, uint64_t *n_pairs);
int pg_mash_dist_within_dev(const uint32_t *d_q_rows, const uint32_t *d_q_count, uint64_t nq, const uint32_t *d_r_rows, const uint32_t *d_r_count,
                            uint64_t nr, uint64_t row_stride, int32_t s, int32_t k, const uint64_t *d_q_length, const uint64_t *d_r_length,
                            double max_distance, double max_p_value, uint32_t flags, uint32_t *d_pair_q, uint32_t *d_pair_r, uint32_t *d_common,
                            uint32_t *d_denom, double *d_distance, double *d_p_value, uint64_t pairs_cap, uint64_t *d_n_pairs, void *stream);

/* ---- single-process multi-GPU (SURVEY.md 8b "multi-GPU variants taking a device count", 8e) ----
 * What a Go host calls to reach all GPUs of the box with ONE call: reads are independent
 * (mash.go:68-104 touches only its receiver), so the batch is cut into contiguous shards, one per
 * device, each driven by its own host thread through the pipelined host path -- no data-path
 * collective.  devices == NULL: the first n_devices visible devices (n_devices <= 0: all of them);
 * otherwise the listed ordinals.  Arguments and results are exactly those of pg_mash_sketch_uniform /
 * pg_mash_sketch_batch; host buffers may be pageable or pinned (pg_host_alloc). */
int pg_mash_sketch_uniform_multi(const uint8_t *bases, uint64_t n_reads, uint32_t read_len, int32_t k,
                                 int32_t s, uint32_t flags, uint32_t *out, uint64_t row_stride,
                                 int32_t *status, const int32_t *devices, int32_t n_devices);
int pg_mash_sketch_batch_multi(const uint8_t *bases, const uint64_t *offsets, uint64_t n_reads,
                               int32_t k, int32_t s, uint32_t flags, uint32_t *out,
                               uint64_t row_stride, uint32_t *count, int32_t *status,
                               const int32_t *devices, int32_t n_devices);
/* mash.Sketch of every read followed by all-pairs Similarity/Distance (mash.go:68-104, 107-140) on
 * several devices: device r sketches its shard and the sketch kernel itself stores every finished
 * tile / row into the gathered buffer of EVERY device (in-process peer access over NVLink: the
 * all-gather is fused into the kernel), then computes row block r of the pair matrix.  Outputs (host,
 * each may be NULL): sketches n x s (full Go arrays, zero tail included), same n x n uint32,
 * distance n x n double; receiver = row.  Without peer access the exchange uses peer copies. */
int pg_mash_sketch_distance_multi(const uint8_t *bases, uint64_t n_reads, uint32_t read_len, int32_t k,
                                  int32_t s, const int32_t *devices, int32_t n_devices,
                                  uint32_t *sketches, uint32_t *same, double *distance);

/* Name of the kernel the last uniform call on this thread dispatched to and how many
 * kernels it launched (bench.py's gpu_launches evidence). */
const char *pg_last_kernel(void);
uint64_t pg_launch_count(void);

/* ---- (*Mash).Similarity / Distance -- search/mash/mash.go:107-140 ----------------
 * Sketch j is words sketches[sk_offsets[j] .. sk_offsets[j+1]) and its length is its
 * SketchSize (the full array a Go Mash holds, zero tail included).  For pair p the
 * receiver is pair_a[p], the argument pair_b[p].  Literal reference semantics:
 * larger/smaller by SketchSize with the receiver "larger" on ties (:109-115), the
 * range early-out (:117-119), the two-pointer walk (:121-132) -- exact also for
 * unsorted (n < s) sketches.  same[p] = matching count, similarity[p] =
 * same/smaller.SketchSize (:134), distance[p] = 1 - similarity (:139).  Any of
 * same/similarity/distance may be NULL.  A sketch of size 0 is PG_ITEM_PANIC.
 */
int pg_mash_similarity_pairs(const uint32_t *sketches, const uint64_t *sk_offsets,
                             uint64_t n_sketches, const uint32_t *pair_a, const uint32_t *pair_b,
                             uint64_t n_pairs, int64_t *same, double *similarity,
                             double *distance, int32_t *status);
int pg_mash_similarity_pairs_dev(const uint32_t *d_sketches, const uint64_t *d_sk_offsets,
                                 uint64_t n_sketches, const uint32_t *d_pair_a,
                                 const uint32_t *d_pair_b, uint64_t n_pairs, int64_t *d_same,
                                 double *d_similarity, double *d_distance, int32_t *d_status,
                                 void *stream);
/* All pairs of a row block against a set of equal-size sketches: rows
 * [row_begin, row_end) of the n x n matrix, receiver = row, argument = column.
 * sketches is n x s (full Go arrays).  same is (row_end-row_begin) x n uint32,
 * distance likewise double (either may be NULL).  Same literal semantics. */
int pg_mash_distance_block(const uint32_t *sketches, uint64_t n, int32_t s, uint64_t row_begin,
                           uint64_t row_end, uint32_t *same, double *distance);
int pg_mash_distance_block_dev(const uint32_t *d_sketches, uint64_t n, int32_t s,
                               uint64_t row_begin, uint64_t row_end, uint32_t *d_same,
                               double *d_distance, void *stream);

/* The same row block as (i, j, same) triples of the pairs that share at least one hash: every ordered
 * pair (i, j), row_begin <= i < row_end, j != i (with PG_PAIRS_UPPER: j > i only), whose matching count is
 * non-zero, in no particular order.  Pairs that are not listed have same == 0 (Similarity 0, Distance 1,
 * mash.go:134,139); the diagonal is never listed.  For n sketches this returns O(related pairs) instead of
 * the n x rows matrix (cfg3, j > i: 2.8e7 triples = 334 MB instead of 40 GB).  *n_pairs receives the number of
 * qualifying pairs; PG_ERR_ARG (with the first pairs_cap stored) if it exceeds pairs_cap.  The _dev variant
 * takes a DEVICE counter d_n_pairs (which may exceed pairs_cap) and never blocks on the result. */
#define PG_PAIRS_UPPER 1u
int pg_mash_distance_sparse(const uint32_t *sketches, uint64_t n, int32_t s, uint64_t row_begin,
                            uint64_t row_end, uint32_t flags, uint32_t *pair_i, uint32_t *pair_j,
                            uint32_t *pair_same, uint64_t pairs_cap, uint64_t *n_pairs);
int pg_mash_distance_sparse_dev(const uint32_t *d_sketches, uint64_t n, int32_t s, uint64_t row_begin,
                                uint64_t row_end, uint32_t flags, uint32_t *d_pair_i, uint32_t *d_pair_j,
                                uint32_t *d_pair_same, uint64_t pairs_cap, uint64_t *d_n_pairs,
                                void *stream);

/* ---- cluster: single-linkage groups of a sketch set at a matching-count threshold --------------------
 * sketches is n x s (full Go arrays, zero tail included, as pg_mash_distance_block takes them).
 *   - Link rule: sketches i < j are linked iff same(i, j) >= min_same, where same(i, j) is what
 *     sketches[i].Similarity(sketches[j]) counts with the LOWER index as the receiver (mash.go:107-135): the
 *     value pg_mash_distance_block writes at row i, column j, and pg_mash_distance_sparse lists under
 *     PG_PAIRS_UPPER.  Unsorted (L - k < s) sketches are counted by that literal walk, not as sets.  Between
 *     sketches of one size the walk advances whichever side holds the smaller value, so column i of row j holds
 *     the same count: the receiver is stated to name the entry that is read, not because the choice matters.
 *   - Groups are the connected components of the link graph (single linkage: members need not be linked
 *     directly).
 *   - Label rule: label[i] = the smallest sketch index in i's group, so label[i] == i marks one representative
 *     per group and the output depends on the input only.
 *   - *n_groups = number of i with label[i] == i; *n_links = number of linked pairs i < j (the count of
 *     PG_PAIRS_UPPER triples with same >= min_same).  Either may be NULL.
 *   - Errors, checked in this order: n > 2^32 - 1 is PG_ERR_ARG; n == 0 is valid (nothing is read or written
 *     but the two counts, which are 0); s <= 0 is PG_ERR_PANIC as in the distance calls (Sketches[-1]);
 *     min_same == 0 (every pair would link) or min_same > s (none could) is PG_ERR_ARG.  PG_ERR_UNSUPPORTED
 *     as pg_mash_distance_block when unsorted sketches exceed the pairwise kernel's shared-memory tile.
 * A matching count for a Distance cut: the smallest c with 1 - (double)c / s <= max_distance.
 * The pairs are never materialised: dense row-block tiles are scanned on the device as they are produced.
 * Device memory beyond the sketches: one tile of <= 8 GiB, 4 n bytes and the distance plan.
 * The _dev variant synchronises `stream` in one place, while it builds the distance plan before the first tile
 * (sortedness and bucket sizes choose the algorithm, as in pg_mash_distance_block_dev); it then only enqueues,
 * and leaves d_label and the two DEVICE counters ordered on `stream` without waiting for them. */
int pg_mash_cluster(const uint32_t *sketches, uint64_t n, int32_t s, uint32_t min_same, uint32_t *label,
                    uint64_t *n_groups, uint64_t *n_links);
int pg_mash_cluster_dev(const uint32_t *d_sketches, uint64_t n, int32_t s, uint32_t min_same, uint32_t *d_label,
                        uint64_t *d_n_groups, uint64_t *d_n_links, void *stream);

/* ---- dereplicate: greedy representatives of a sketch set at a matching-count threshold ----------------
 * sketches is n x s (full Go arrays, zero tail included, as pg_mash_cluster takes them).
 *   - Link rule: that of pg_mash_cluster.  Sketches r < i are linked iff same(r, i) >= min_same, same(r, i)
 *     being what sketches[r].Similarity(sketches[i]) counts with the LOWER index as the receiver; unsorted
 *     (L - k < s) sketches are counted by that literal walk.
 *   - Representatives, in index order: i is a representative iff no representative r < i is linked to i (a
 *     caller's greedy loop over the set: every sketch within the cut of one kept so far joins the first such,
 *     any other is kept).  Callers who want another priority (length, quality) permute the set first.
 *   - Assignment: rep[i] = i for a representative.  Otherwise, by default, rep[i] = the smallest representative
 *     linked to i; with PG_DEREP_NEAREST, the linked earlier representative with the largest same (for one
 *     sketch size, the smallest Distance), ties to the smaller index.  Both modes pick the same representatives.
 *   - *n_reps = number of i with rep[i] == i.  It may be NULL.
 *   - The output depends on the input only: not on tile or sub-block size, grid or the order of atomics.
 *   - Errors, checked in this order: a flags bit other than PG_DEREP_NEAREST is PG_ERR_ARG; then the rules of
 *     pg_mash_cluster: n > 2^32 - 1 is PG_ERR_ARG; n == 0 is valid (nothing is read or written but *n_reps,
 *     which is 0); s <= 0 is PG_ERR_PANIC; min_same == 0 or min_same > s is PG_ERR_ARG.  PG_ERR_UNSUPPORTED as
 *     pg_mash_distance_block when unsorted sketches exceed the pairwise kernel's shared-memory tile.
 * A matching count for a Distance cut: the smallest c with 1 - (double)c / s <= max_distance.
 * The pairs are never materialised: dense row-block tiles are consumed on the device as they are produced, and
 * only the representatives' rows are read beyond the 1024-row diagonal blocks.
 * Device memory beyond the sketches: one tile of <= 8 GiB, the distance plan, the 4 n bytes of rep (the first
 * assignment is built there in place; PG_DEREP_NEAREST adds 8 n bytes, a 64-bit key per sketch), a 128 KiB link
 * bitmap and a 4 KiB list.
 * The _dev variant synchronises `stream` in one place, while it builds the distance plan before the first tile,
 * as pg_mash_cluster_dev does; it then only enqueues, with no host round trip per tile or sub-block, and leaves
 * d_rep and the DEVICE counter ordered on `stream` without waiting for them. */
#define PG_DEREP_NEAREST 1u
int pg_mash_dereplicate(const uint32_t *sketches, uint64_t n, int32_t s, uint32_t min_same, uint32_t flags,
                        uint32_t *rep, uint64_t *n_reps);
int pg_mash_dereplicate_dev(const uint32_t *d_sketches, uint64_t n, int32_t s, uint32_t min_same, uint32_t flags,
                            uint32_t *d_rep, uint64_t *d_n_reps, void *stream);

/* ---- sketch index: top-k nearest references of query sketches -------------------------------------
 * A reference set of n sketches of size s (n x s full Go arrays, zero tail included, as
 * pg_mash_distance_block takes them) is copied to the device once and indexed there; batches of
 * query sketches are then ranked against it.  For query q and reference j, same[q][j] is what
 * queries[q].Similarity(refs[j]) counts -- the QUERY is the receiver (mash.go:107-135): larger/smaller
 * by SketchSize with the receiver winning ties, the range early-out, the two-pointer walk (exact also
 * for unsorted n < s sketches).  KmerSize is not compared, as in the reference.  distance =
 * 1 - same/min(sq, s) in double, bit-identical to (*Mash).Distance (mash.go:134,139).
 *
 * Result for query q (row q of the nq x top_k outputs): the references with same >= min_same, ordered
 * by same descending, then by reference index ascending (ties at the cut are broken the same way),
 * cut to the first top_k; n_hits[q] (<= top_k) of them are listed.  The denominator is the same for
 * every reference of a query, so this is also distance ascending.  Unused slots hold ref 0xFFFFFFFF,
 * same 0 and distance 1.0.  min_same = 0 also lists references that share nothing, in index order.
 * 1 <= top_k <= PG_INDEX_MAX_TOP_K, else PG_ERR_ARG.  Any of the four outputs may be NULL.  nq == 0
 * is valid.  A sketch of size 0 (s or sq) is PG_ERR_PANIC, as in the distance calls above.
 * PG_ERR_UNSUPPORTED when a query must be compared pairwise (an unsorted query or reference, or a set
 * too skewed for the inverted index) and 8 * (sq + s) words exceed the kernel's shared-memory tile.
 *
 * Ownership, device and threads:
 *   - create copies the reference sketches into device memory the index owns; no caller pointer is
 *     retained.  pg_mash_index_free releases it;
 *   - the index lives on the device current for the calling thread at creation (pg_thread_device /
 *     pg_init); queries run on that device whatever thread calls them (the calling thread's current
 *     CUDA device is set to it).  _dev queries take device pointers on that device;
 *   - the index changes only through pg_mash_index_add (below).  Each index has a reader-writer lock:
 *     every query call, host or _dev, holds it shared while it reads the index and enqueues, and an add
 *     holds it exclusively.  So any number of threads may query one index at once, and a query sees the
 *     index either wholly before or wholly after an add.  Freeing an index or adding to it while a _dev
 *     query on it is still enqueued on a stream that has not been synchronised is the caller's error (both
 *     release device buffers the query reads), as is freeing it while any call on it is running;
 *   - create, create_dev and both query calls synchronise (the host chooses the kernels from the data);
 *     query_dev leaves its outputs on the device, ordered on `stream`.
 */
#define PG_INDEX_MAX_TOP_K 1024u
typedef struct pg_mash_index pg_mash_index;
int pg_mash_index_create(const uint32_t *sketches, uint64_t n, int32_t s, pg_mash_index **out);
int pg_mash_index_create_dev(const uint32_t *d_sketches, uint64_t n, int32_t s, void *stream, pg_mash_index **out);
int pg_mash_index_query(const pg_mash_index *ix, const uint32_t *queries, uint64_t nq, int32_t sq, uint32_t top_k,
                        uint32_t min_same, uint32_t *hit_ref, uint32_t *hit_same, double *hit_distance, uint32_t *n_hits);
int pg_mash_index_query_dev(const pg_mash_index *ix, const uint32_t *d_queries, uint64_t nq, int32_t sq, uint32_t top_k,
                            uint32_t min_same, uint32_t *d_hit_ref, uint32_t *d_hit_same, double *d_hit_distance,
                            uint32_t *d_n_hits, void *stream);
int pg_mash_index_free(pg_mash_index *ix);

/* ---- sketch index: growing it ----------------------------------------------------------------------
 * pg_mash_index_add appends m sketches of size s (m x s full Go arrays, zero tail included, as create takes
 * them) as references n .. n + m - 1.  The batch is copied; no caller pointer is retained.
 *   - Invariant: for any split of a reference set R into R0, R1, ..., Rk, create(R0) followed by add(R1) ...
 *     add(Rk) answers every later pg_mash_index_query / pg_mash_index_query_within call (host or _dev) with
 *     the same hit_ref, hit_same, n_hits, hit_offsets and the same bytes of hit_distance as create(R).
 *   - Sketch size: an index that holds no reference (n == 0, whatever s it was created with) takes the s of
 *     the first non-empty batch; after that every batch must have the index's s.
 *   - Errors, checked in this order: a null index is PG_ERR_ARG (no device is needed); m == 0 is valid and
 *     changes nothing; s <= 0 is PG_ERR_PANIC, as in create; an s other than a non-empty index's s is
 *     PG_ERR_ARG; n + m > 2^32 - 1 is PG_ERR_ARG (the join keys hold 32-bit ids), checked before any buffer
 *     is read; a null buffer is PG_ERR_ARG.  PG_ERR_NOMEM when device memory runs out.  After any error
 *     the index holds exactly what it held before and still answers queries.
 *   - The join index: when every reference so far is ascending and the index has its (value, id) join, an
 *     ascending batch is merged into it on the device, with no rebuild.  A batch with an unsorted sketch
 *     drops the join, and from then on every query row is compared pairwise, as create does for a set with
 *     an unsorted sketch.  An index without a join (unsorted references, values too skewed for the join, or
 *     PG_K3_PAIRWISE at creation) stays without one; an empty index is indexed as create would index the
 *     batch.  Answers are the same either way; only the speed differs.
 *   - Device memory: the old and the new index are both held until the add completes.  With T old join
 *     entries and M = m x s new ones the peak of a merge is the sum of the old sketches (4 n s bytes), the
 *     new copy (4 (n + m) s bytes), the old entries (8 T bytes), the batch's keys and their sort (16 M bytes
 *     plus CUB's temporary storage), the merged entries (8 (T + M) bytes) and the index's flags (n + m bytes);
 *     the host call adds 4 m s bytes, the batch staged on the device.
 *   - Synchronisation: both calls synchronise; the host must read how many batch sketches are unsorted to
 *     choose the join update, as create does.  The _dev call reads d_sketches on `stream` and does its work
 *     there.
 *   - Threads: see the index block above; an add excludes every query and every other add on the index.
 *     The lock prefers readers: an add waits until no query holds it, so a steady stream of overlapping
 *     queries from many threads can delay an add for as long as the stream lasts. */
int pg_mash_index_add(pg_mash_index *ix, const uint32_t *sketches, uint64_t m, int32_t s);
int pg_mash_index_add_dev(pg_mash_index *ix, const uint32_t *d_sketches, uint64_t m, int32_t s, void *stream);

/* ---- sketch index: every reference within a matching-count cut (radius query) ----------------------
 * The question "which references lie within Distance <= d of each query, however many there are", answered
 * against a pg_mash_index without the top-k cap.
 *   - Lists: query q's hits are the references j with same[q][j] >= min_same, in ascending reference index,
 *     stored at positions [hit_offsets[q], hit_offsets[q+1]) of hit_ref / hit_same / hit_distance.  same[q][j]
 *     is what queries[q].Similarity(refs[j]) counts, the QUERY being the receiver, exactly as in
 *     pg_mash_index_query; hit_distance = 1 - same/min(sq, s) in double, bit-identical to (*Mash).Distance.
 *     hit_offsets has nq + 1 entries; hit_offsets[nq] is the total.
 *   - The output depends on the input alone: not on the row-block size, the grid or the order of atomics.
 *   - Any of hit_ref / hit_same / hit_distance may be NULL.  With all three NULL (and hits_cap = 0) the call
 *     only counts: it fills the offsets and the total and does not report an overflow.  n_hits (d_n_hits) may
 *     be NULL too: the total is also hit_offsets[nq].
 *   - A Distance cut becomes a count as for pg_mash_cluster: the smallest c with 1 - (double)c / min(sq, s) <=
 *     max_distance.
 *   - Errors, checked in this order: a null index is PG_ERR_ARG; min_same == 0 is PG_ERR_ARG (it would list all
 *     nq x n pairs); nq == 0 is valid and writes hit_offsets[0] = 0 and a total of 0; sq <= 0 is PG_ERR_PANIC;
 *     a null hit_offsets (or, for the host call, null queries) is PG_ERR_ARG; PG_ERR_UNSUPPORTED when a query
 *     must be compared pairwise and the tile does not fit, as pg_mash_index_query reports it.
 *   - min_same > min(sq, s) is valid and gives empty lists, as does an index of n == 0 references.
 *   - Overflow: a total above hits_cap in a host call that asks for a list is PG_ERR_ARG; the offsets are then complete, the first
 *     hits_cap hits are stored and *n_hits holds the total (as pg_mash_distance_sparse does).  The _dev call does
 *     not fail on overflow: it never writes a list past hits_cap and leaves the total in d_n_hits.
 *   - Each row block's dense counts are read twice, once to count and once to fill, so unlike the top-k query
 *     there is no 2^24 limit on the sketch size.
 * Synchronisation: the _dev call synchronises `stream` only where pg_mash_index_query_dev does, while it reads
 * how many queries are unsorted; it then only enqueues (the offsets are scanned on the device, block after block)
 * and leaves every output ordered on `stream` without waiting for it.  The host call synchronises.
 * Threads and ownership: those of the index block above; any number of threads may mix pg_mash_index_query and
 * pg_mash_index_query_within calls on one index. */
int pg_mash_index_query_within(const pg_mash_index *ix, const uint32_t *queries, uint64_t nq, int32_t sq,
                               uint32_t min_same, uint64_t *hit_offsets, uint32_t *hit_ref, uint32_t *hit_same,
                               double *hit_distance, uint64_t hits_cap, uint64_t *n_hits);
int pg_mash_index_query_within_dev(const pg_mash_index *ix, const uint32_t *d_queries, uint64_t nq, int32_t sq,
                                   uint32_t min_same, uint64_t *d_hit_offsets, uint32_t *d_hit_ref,
                                   uint32_t *d_hit_same, double *d_hit_distance, uint64_t hits_cap,
                                   uint64_t *d_n_hits, void *stream);

/* ---- dereplicate: growing a dereplication ------------------------------------------------------------
 * A dereplicator keeps the representatives of every sketch added so far and assigns each new batch against them
 * on the device, so a growing collection is never dereplicated from scratch.  Sketches are numbered in the order
 * they are added: the rows of a batch are ids first .. first + m - 1 (m x s full Go arrays, as pg_mash_dereplicate
 * takes them).  The batch is copied; no caller pointer is retained.
 *   - Invariant: split a set S of sketches of one size into B0, B1, ..., Bk and call add(B0) ... add(Bk).  The
 *     concatenated rep outputs equal pg_mash_dereplicate(S, min_same, flags) and the n_new_reps add up to its n_reps,
 *     in both modes and for any split, empty and one-row batches included.  rep values are global ids.
 *   - Why it is exact: under the greedy rule a sketch's flag and assignment depend only on the representatives
 *     before it.  So no earlier row ever changes, and a batch row is decided by the kept representatives linked to
 *     it and by the batch's own representatives before it.  The first are found by a query of the batch against
 *     the representative index (the query is the receiver; for one sketch size the count is symmetric, so it is the
 *     dereplicate count, unsorted sketches included), the second by the dereplicate pass over the batch alone.
 *   - Link rule, count and cut: those of pg_mash_dereplicate.  PG_DEREP_NEAREST is the only flag.
 *   - Errors.  create checks, in this order: a flags bit other than PG_DEREP_NEAREST is PG_ERR_ARG; s <= 0 is
 *     PG_ERR_PANIC (the rule dereplicate applies to a non-empty set); min_same == 0 or min_same > s is PG_ERR_ARG.
 *     add (host and _dev) checks, in this order: a null dereplicator is PG_ERR_ARG (no device is needed); m == 0 is
 *     valid and changes nothing (*first = n, *n_new_reps = 0); s <= 0 is PG_ERR_PANIC; an s other than the
 *     dereplicator's is PG_ERR_ARG; n + m > 2^32 - 1 is PG_ERR_ARG, checked before any buffer is read; a null
 *     buffer (sketches or rep) is PG_ERR_ARG.  PG_ERR_UNSUPPORTED and PG_ERR_NOMEM arise where the index query,
 *     the dereplicate pass or the index add raise them.  After any error the dereplicator holds exactly what it
 *     held before; only the caller's rep contents are then unspecified.  first and n_new_reps may be NULL.
 *   - Representative index: pg_mash_dereplicator_index returns a borrowed, read-only pg_mash_index whose reference
 *     p is the p-th representative in ascending id order, so the existing top-k and radius queries answer "which
 *     kept sketch is this one closest to".  pg_mash_dereplicator_reps maps positions to ids: the first min(cap,
 *     n_reps) ids into `ids` and their number into *n_reps; more than cap is PG_ERR_ARG after the first cap are
 *     stored.  Ids are append-only, so a reps read made after a query covers every position that query returned.
 *     The handle is valid until pg_mash_dereplicator_free and must not be passed to pg_mash_index_add or
 *     pg_mash_index_free.  pg_mash_dereplicator_index(NULL) is NULL; pg_mash_dereplicator_free(NULL) is PG_OK.
 *   - Synchronisation: an add synchronises, once each to read the batch's sortedness for the query, to plan the
 *     batch's pass, to read how many new representatives there are, and in the index add; so first and n_new_reps
 *     are host pointers in _dev too.  _dev reads d_sketches and writes d_rep on `stream`, where it does its work.
 *   - Threads: adds on one dereplicator are serialised by its own lock, and reps waits for a running add.  An add
 *     holds the representative index's reader-writer lock exclusively from start to end, so a query on the
 *     borrowed index sees it wholly before or wholly after an add.  The dereplicator lives on the device current
 *     at creation.
 *   - Device memory of an add, with R kept representatives and R' new ones: the m x R counts of the query (in row
 *     blocks of at most 2 GiB), the batch's distance plan and its tile of <= 8 GiB, 4 m bytes of rep (PG_DEREP_NEAREST
 *     adds 8 m bytes of keys), the gathered new rows (4 R' s bytes) and ids (4 (R + R') bytes), and the peak of
 *     pg_mash_index_add for R' rows; the host call adds 4 m s bytes, the batch staged on the device. */
typedef struct pg_mash_dereplicator pg_mash_dereplicator;
int pg_mash_dereplicator_create(int32_t s, uint32_t min_same, uint32_t flags, pg_mash_dereplicator **out);
int pg_mash_dereplicator_add(pg_mash_dereplicator *d, const uint32_t *sketches, uint64_t m, int32_t s,
                             uint32_t *rep, uint64_t *first, uint64_t *n_new_reps);
int pg_mash_dereplicator_add_dev(pg_mash_dereplicator *d, const uint32_t *d_sketches, uint64_t m, int32_t s,
                                 uint32_t *d_rep, uint64_t *first, uint64_t *n_new_reps, void *stream);
int pg_mash_dereplicator_reps(const pg_mash_dereplicator *d, uint32_t *ids, uint64_t cap, uint64_t *n_reps);
const pg_mash_index *pg_mash_dereplicator_index(const pg_mash_dereplicator *d);
int pg_mash_dereplicator_free(pg_mash_dereplicator *d);

/* ---- cluster: growing a clustering -------------------------------------------------------------------
 * A clusterer keeps an index over every sketch added so far and their single-linkage labels, and merges each new
 * batch into the groups on the device, so a growing collection is never clustered from scratch.  Sketches are
 * numbered in the order they are added: the rows of a batch are ids first .. first + m - 1 (m x s full Go arrays,
 * as pg_mash_cluster takes them).  The batch is copied; no caller pointer is retained.
 *   - Invariant: split a set S of sketches of one size into B0, B1, ..., Bk and call add(B0) ... add(Bk).  After
 *     the add of Bj, labels(0, n) equals the labels of pg_mash_cluster(B0 .. Bj, min_same) and *n_groups its
 *     group count; the add's label output is the slice [first, first + m) of those labels, and the *n_links of
 *     the adds sum to its n_links.  This holds for any split, empty and one-row batches included.  Labels are
 *     global ids.
 *   - Why it is exact: single linkage is union-find over the links, so the components of B0 .. Bj are those of
 *     B0 .. Bj-1 united with every link between a row of Bj and any earlier sketch and every link inside Bj.  The
 *     first come from a query of Bj against the index of all earlier sketches (the batch row is the receiver;
 *     for one sketch size the count is symmetric, so it is the cluster count, unsorted sketches included), the
 *     second from the cluster pass over Bj alone (the lower row is the receiver).  Labels are the smallest id of
 *     each group, which the input alone decides.
 *   - Earlier labels can change: a batch row that links two earlier groups joins them, and the larger label is
 *     retired.  *n_merged is the number of earlier groups absorbed into another by this add (roots r < first
 *     whose label changed); 0 says no earlier label changed.  *n_links counts this add's links, cross and inner.
 *   - Link rule, count and cut: those of pg_mash_cluster.
 *   - Errors.  create checks, in this order: a null out is PG_ERR_ARG; s <= 0 is PG_ERR_PANIC (the rule cluster
 *     applies to a non-empty set); min_same == 0 or min_same > s is PG_ERR_ARG.  add (host and _dev) checks, in
 *     this order: a null clusterer is PG_ERR_ARG (no device is needed); m == 0 is valid and changes nothing
 *     (*first = n, *n_groups = the current count, *n_links = *n_merged = 0); s <= 0 is PG_ERR_PANIC; an s other
 *     than the clusterer's is PG_ERR_ARG; n + m > 2^32 - 1 is PG_ERR_ARG, checked before any buffer is read; a
 *     null sketches buffer is PG_ERR_ARG.  PG_ERR_UNSUPPORTED and PG_ERR_NOMEM arise where the index query, the
 *     cluster pass over the batch or the index add raise them.  After any error the clusterer's labels, index
 *     and counts are exactly what they were; only the caller's label contents are then unspecified.  label and
 *     every count pointer may be NULL.  labels: begin > end, end > n, or a null buffer with end > begin is
 *     PG_ERR_ARG.
 *   - The index: pg_mash_clusterer_index returns a borrowed, read-only pg_mash_index whose reference p is sketch
 *     p, so "which group would this new sketch join" is a top-k or radius query followed by a labels read.  The
 *     handle is valid until pg_mash_clusterer_free and must not be passed to pg_mash_index_add or
 *     pg_mash_index_free.  pg_mash_clusterer_index(NULL) is NULL; pg_mash_clusterer_free(NULL) is PG_OK.
 *   - Synchronisation: an add synchronises, to read the batch's sortedness for the query, to plan the batch's
 *     pass, to read the counts, and in the index add; so the counts are host pointers in _dev too.  _dev reads
 *     d_sketches and writes d_label on `stream`, where it does its work.  labels_dev copies on `stream` and does
 *     not wait.  Enqueuing labels_dev or a _dev query on the borrowed index and then adding or freeing before
 *     that stream is synchronised is the caller's error, as for the index.
 *   - Threads: adds on one clusterer are serialised by its own lock, and label reads wait for a running add.  An
 *     add holds the index's reader-writer lock exclusively from start to end (taken before the device lock), so
 *     a query on the borrowed index sees it wholly before or wholly after an add.  The clusterer lives on the
 *     device current at creation.
 *   - Device memory of an add, with n sketches held: the m x n counts of the query (in row blocks of at most
 *     2 GiB), the batch's distance plan and its tile of <= 8 GiB, the forest of the n + m sketches and their new
 *     labels (4 (n + m) bytes each) while the old 4 n bytes of labels are held, and the peak of pg_mash_index_add
 *     for m rows; the host call adds 4 m s bytes, the batch staged on the device.  The index holds 4 n s bytes of
 *     sketches and its join at 8 bytes per entry: at 100 000 sketches of s = 2000, 0.8 GB and about 1.6 GB. */
typedef struct pg_mash_clusterer pg_mash_clusterer;
int pg_mash_clusterer_create(int32_t s, uint32_t min_same, pg_mash_clusterer **out);
int pg_mash_clusterer_add(pg_mash_clusterer *c, const uint32_t *sketches, uint64_t m, int32_t s, uint32_t *label, uint64_t *first,
                          uint64_t *n_groups, uint64_t *n_links, uint64_t *n_merged);
int pg_mash_clusterer_add_dev(pg_mash_clusterer *c, const uint32_t *d_sketches, uint64_t m, int32_t s, uint32_t *d_label,
                              uint64_t *first, uint64_t *n_groups, uint64_t *n_links, uint64_t *n_merged, void *stream);
int pg_mash_clusterer_labels(const pg_mash_clusterer *c, uint64_t begin, uint64_t end, uint32_t *label);
int pg_mash_clusterer_labels_dev(const pg_mash_clusterer *c, uint64_t begin, uint64_t end, uint32_t *d_label, void *stream);
const pg_mash_index *pg_mash_clusterer_index(const pg_mash_clusterer *c);
int pg_mash_clusterer_free(pg_mash_clusterer *c);

/* ---- screen: which references of a sketch set a pool of reads contains --------------------------------
 * Mash Screen (Ondov et al., Genome Biol 20:232, 2019): every k-mer window of a pool of reads is hashed, and each
 * reference sketch is asked how many of its hashes the pool holds and how often.  A screen holds n reference
 * sketches of size s (n x s full Go arrays, zero tail included, as pg_mash_index_create takes them), a k-mer size k
 * and a running pool, which adds grow and reset empties.
 *   - Windows: a pool read of length L contributes the windows (*Mash).Sketch hashes, positions 0 .. L - k - 1
 *     (the last k-mer is never hashed, mash.go:73; L <= k gives none), each hashed by murmur3.Sum32 over its raw
 *     bytes: forward strand, case-sensitive, any byte value.  k is not checked against the references, as in the
 *     reference; pass the k the sketches were made with.  A screen made by create_flags (+ _dev) with
 *     PG_KMER_CANONICAL counts the canonical windows (above) in every add; like k, the mode is not checked against
 *     the sketches' (pass sketches made in the same mode, e.g. by pg_mash_sketch_groups_flags).
 *   - Counts: c_pool(v) = the windows of every read of every add since creation or the last reset whose hash is v;
 *     c_r(v) = the words of reference r equal to v, taken as given (zero-tail words are the value 0; unsorted
 *     fill-regime sketches are allowed).
 *   - Results for reference r: shared[r] = sum over v of min(c_r(v), c_pool(v)), the multiset count Similarity
 *     uses; containment[r] = (double)shared[r] / (double)s; multiplicity[r] = the lower median (element
 *     floor((m - 1) / 2) of m in ascending order) of the multiset in which each v with c_pool(v) >= 1 contributes
 *     the value c_pool(v) min(c_r(v), c_pool(v)) times; 0 when shared[r] == 0.  Mash Screen's identity,
 *     containment^(1/k), is left to the caller.
 *   - Winners (winners, winners_dev), Mash Screen's winner-take-all (mash screen -w): each value v with
 *     c_pool(v) >= 1 is given to one of its contenders, the references r with c_r(v) >= 1: the one with the largest
 *     shared[r] of results (the first pass), a tie to the smallest reference index.  All references of a screen have
 *     one s, so this is Mash's order by identity (shared / s)^(1/k), exact for every k (0 included); Mash breaks its
 *     ties by genome length, which a screen does not hold, so the tie rule is this library's own.  The reallocation
 *     is done once, from the first-pass scores, as in Mash.  winners then returns the three arrays of results over
 *     the values each reference won: shared_w[r] = sum over v won by r of min(c_r(v), c_pool(v)) (<= shared[r]),
 *     containment_w[r] = shared_w[r] / s, multiplicity_w[r] = the lower median of c_pool(v) over the won values,
 *     each counted min(c_r(v), c_pool(v)) times, 0 when r won nothing.  Zero-tail words take part as any other word
 *     (the value 0 has every zero-tailed reference as a contender).  A reference that shares no pool value with
 *     another reference keeps its results, and with n == 1 winners equals results.  The output does not depend on
 *     the order of the device's atomics, and winners leaves the screen as it was.
 *   - Split invariance: for any split of a pool into adds (empty and one-read adds included) the results and the
 *     winners equal those of one add of the concatenation; after a reset the screen answers as a freshly created one.
 *   - Errors, checked in this order: a null screen or out is PG_ERR_ARG (no device is needed); k < 0 is
 *     PG_ERR_ARG, as for the sketch calls; (create_flags: an unknown flag bit, then k == 0 with PG_KMER_CANONICAL,
 *     PG_ERR_ARG); s <= 0 with n > 0 is PG_ERR_PANIC, as for index create; n > 2^32 - 1 is
 *     PG_ERR_ARG (the keys hold 32-bit ids); a null buffer is PG_ERR_ARG.  n == 0 and n_reads == 0 are valid (an
 *     add of no read changes nothing and needs no buffer).  Offsets that decrease in a host add are PG_ERR_ARG.
 *     Any output of results or winners may be NULL.  PG_ERR_NOMEM when device memory runs out.  After any error the screen
 *     holds what it held before.
 *   - _dev offsets: add_dev trusts d_offsets as pg_mash_sketch_batch_dev does.  With non-decreasing offsets it
 *     counts exactly the windows above.  Offsets that decrease give unspecified counts, but no byte outside
 *     [d_offsets[0], d_offsets[n_reads]) is read and no memory outside the screen is written.
 *   - Ownership, device and threads, as for pg_mash_index: create copies everything (no caller pointer is kept)
 *     and the screen lives on the device current at creation.  Each screen has a reader-writer lock: add, add_dev
 *     and reset hold it exclusively, results, winners and their _dev forms shared, while they enqueue.  The host
 *     calls synchronise (create also to size its buffers).  add_dev, results_dev and winners_dev only enqueue on
 *     `stream`; add_dev
 *     makes no host decision that depends on the data.  Work enqueued by _dev calls on different streams is ordered
 *     by the caller: results see an add_dev only once its stream is ordered before them (a host call runs on the
 *     library's own stream), and freeing or resetting a screen while a _dev call on it is still enqueued on an
 *     unsynchronised stream is the caller's error.
 *   - Counter width: pool counts are 64-bit, so a pool of more than 2^32 windows with one hash stays exact.
 *     multiplicity is uint64; shared <= s.
 *   - Device memory: with D distinct values among the n s words, a screen holds 8 n s bytes of sorted keys,
 *     4 D of values, 8 (D + 1) of counts and 8 (ceil(D / 4) + 1) of directory.  Create adds, while it runs, 8 n s bytes
 *     of unsorted keys, 8 n s of values and CUB's sort storage (the host call also stages 4 n s bytes of sketches);
 *     results add 16 n s bytes of multiplicity slots, 4 n of counts and CUB's segmented-sort storage; winners adds
 *     to those 8 D bytes of votes; the host add stages the pool's bytes and offsets.
 *   - Several samples (create_samples, add_samples, results_samples, winners_samples and their _dev forms): a screen
 *     holds S = n_samples >= 1 pools over one reference index, and each read of add_samples carries a sample id
 *     (one uint32 per read).  c_pool,q(v) = the windows (as above) with hash v of the reads tagged q, over every add
 *     since creation or the last reset.  Row q of results_samples is results with c_pool,q in place of c_pool; row q
 *     of winners_samples is the winner-take-all with sample q's own first-pass shared (samples never vote together:
 *     a value present in samples 1 and 2 is allocated in each apart).  Sample independence: row q equals, byte for
 *     byte, what a fresh pg_mash_screen_create screen answers after one add of only sample q's reads in the same
 *     order; a sample that received no reads has an all-zero row.  Split invariance holds per sample, for any mix
 *     of host and _dev adds; reset empties every sample.  results_samples and winners_samples write rows
 *     [first, first + count) of the [S][n] table, row-major: out[(q - first) * n + r]; any output may be NULL.
 *   - The single-sample calls on any screen: create and create_dev make S = 1; add and add_dev count every read into
 *     sample 0; results, results_dev, winners and winners_dev return row 0.
 *   - Errors of the sample calls, added to the order above: n_samples == 0 is PG_ERR_ARG, after the n > 2^32 - 1
 *     rule and before the null-buffer rule.  A null id array with n_reads > 0 is PG_ERR_ARG.  In a host add a sample
 *     id >= S is PG_ERR_ARG, checked on the host before anything is copied or launched (the screen keeps what it
 *     held).  first + count > S is PG_ERR_ARG.  add_samples_dev trusts d_sample_ids as it trusts d_offsets: a read
 *     whose id is >= S contributes nothing, and no memory outside the screen is written.
 *   - Device memory with S samples: the counters take 8 (S D + 1) bytes (one sink counter for reads whose id is not
 *     a sample); create returns PG_ERR_NOMEM when they do not fit.  results_samples and winners_samples tally the
 *     samples in groups of g = max(1, min(count, 2^28 / (n s))): their scratch is that of results (or winners) times
 *     g, at most 16 x 2^28 bytes of slots when n s <= 2^28, whatever S is. */
typedef struct pg_mash_screen pg_mash_screen;
int pg_mash_screen_create(const uint32_t *sketches, uint64_t n, int32_t s, int32_t k, pg_mash_screen **out);
int pg_mash_screen_create_dev(const uint32_t *d_sketches, uint64_t n, int32_t s, int32_t k, void *stream, pg_mash_screen **out);
int pg_mash_screen_add(pg_mash_screen *sc, const uint8_t *bases, const uint64_t *offsets, uint64_t n_reads);
int pg_mash_screen_add_dev(pg_mash_screen *sc, const uint8_t *d_bases, const uint64_t *d_offsets, uint64_t n_reads, void *stream);
int pg_mash_screen_reset(pg_mash_screen *sc);
int pg_mash_screen_results(const pg_mash_screen *sc, uint32_t *shared, double *containment, uint64_t *multiplicity);
int pg_mash_screen_results_dev(const pg_mash_screen *sc, uint32_t *d_shared, double *d_containment, uint64_t *d_multiplicity,
                               void *stream);
int pg_mash_screen_winners(const pg_mash_screen *sc, uint32_t *shared, double *containment, uint64_t *multiplicity);
int pg_mash_screen_winners_dev(const pg_mash_screen *sc, uint32_t *d_shared, double *d_containment, uint64_t *d_multiplicity,
                               void *stream);
int pg_mash_screen_create_samples(const uint32_t *sketches, uint64_t n, int32_t s, int32_t k, uint32_t n_samples, pg_mash_screen **out);
int pg_mash_screen_create_samples_dev(const uint32_t *d_sketches, uint64_t n, int32_t s, int32_t k, uint32_t n_samples, void *stream,
                                      pg_mash_screen **out);
/* create_samples with flags (0 or PG_KMER_CANONICAL): the mode belongs to the screen, like k; every add, results and
 * winners call is unchanged */
int pg_mash_screen_create_flags(const uint32_t *sketches, uint64_t n, int32_t s, int32_t k, uint32_t n_samples, uint32_t flags,
                                pg_mash_screen **out);
int pg_mash_screen_create_flags_dev(const uint32_t *d_sketches, uint64_t n, int32_t s, int32_t k, uint32_t n_samples, uint32_t flags,
                                    void *stream, pg_mash_screen **out);
int pg_mash_screen_add_samples(pg_mash_screen *sc, const uint8_t *bases, const uint64_t *offsets, const uint32_t *sample_ids, uint64_t n_reads);
int pg_mash_screen_add_samples_dev(pg_mash_screen *sc, const uint8_t *d_bases, const uint64_t *d_offsets, const uint32_t *d_sample_ids,
                                   uint64_t n_reads, void *stream);
/* rows [first, first + count) of the [S][n] table, row-major: out[(q - first) * n + r]; any output may be NULL */
int pg_mash_screen_results_samples(const pg_mash_screen *sc, uint32_t first, uint32_t count, uint32_t *shared, double *containment,
                                   uint64_t *multiplicity);
int pg_mash_screen_results_samples_dev(const pg_mash_screen *sc, uint32_t first, uint32_t count, uint32_t *d_shared, double *d_containment,
                                       uint64_t *d_multiplicity, void *stream);
int pg_mash_screen_winners_samples(const pg_mash_screen *sc, uint32_t first, uint32_t count, uint32_t *shared, double *containment,
                                   uint64_t *multiplicity);
int pg_mash_screen_winners_samples_dev(const pg_mash_screen *sc, uint32_t first, uint32_t count, uint32_t *d_shared, double *d_containment,
                                       uint64_t *d_multiplicity, void *stream);
int pg_mash_screen_free(pg_mash_screen *sc);

/* ---- align.SmithWaterman score -- search/align/align.go:171-203 -------------------
 * One template against n queries.  query_is_a != 0: stringA = query (outer loop),
 * stringB = template; else swapped.  lut_a/lut_b: byte -> index into the first /
 * second alphabet, -1 = not in alphabet (alphabet/alphabet.go:35-41); table is
 * n_a x n_b row-major (search/align/matrix/matrix.go:28-38); gap is ADDED
 * (align.go:193-194).  Per query: score (align.go:197-201 running max),
 * err_code 0 / 1 (symbol of stringA) / 2 (symbol of stringB) and err_pos (byte
 * index in that string) of the first failing cell in the reference's row-major
 * visiting order (align.go:188-191); on error score is 0.
 */
int pg_sw_score_batch(const uint8_t *queries, const uint64_t *q_offsets, uint64_t n_queries,
                      const uint8_t *templ, uint64_t templ_len, int32_t query_is_a,
                      const int16_t *lut_a, const int16_t *lut_b, const int64_t *table,
                      int32_t n_a, int32_t n_b, int64_t gap, int64_t *score, int32_t *err_code,
                      int64_t *err_pos);
int pg_sw_score_batch_dev(const uint8_t *d_queries, const uint64_t *d_q_offsets, uint64_t n_queries,
                          uint64_t max_query_len, const uint8_t *d_templ, uint64_t templ_len,
                          int32_t query_is_a, const int16_t *lut_a_host, const int16_t *lut_b_host,
                          const int64_t *table_host, int32_t n_a, int32_t n_b, int64_t gap,
                          int64_t *d_score, int32_t *d_err_code, int64_t *d_err_pos, void *stream);

/* ---- align.SmithWaterman with the aligned strings -- search/align/align.go:171-232 in full ----
 * (SURVEY.md 8f.1).  As pg_sw_score_batch, plus for every query the two aligned strings of the
 * reference's traceback (first maximum in row-major order, diagonal > up > left, align.go:205-229):
 * align_a / align_b hold n_queries rows of out_stride bytes, align_len[i] the common length.
 * status[i]: PG_ITEM_OK, or PG_ITEM_UNSUPPORTED if the alignment is longer than out_stride
 * (align_len[i] then reports the needed length).  Limits: queries of <= 64 symbols and scores
 * that fit 32 bits (PG_ERR_UNSUPPORTED otherwise). */
int pg_sw_align_batch(const uint8_t *queries, const uint64_t *q_offsets, uint64_t n_queries,
                      const uint8_t *templ, uint64_t templ_len, int32_t query_is_a,
                      const int16_t *lut_a, const int16_t *lut_b, const int64_t *table,
                      int32_t n_a, int32_t n_b, int64_t gap, int64_t *score, int32_t *err_code,
                      int64_t *err_pos, uint8_t *align_a, uint8_t *align_b, uint64_t out_stride,
                      uint32_t *align_len, int32_t *status);

/* align.NeedlemanWunsch in full (align.go:100-166): same interface; the traceback starts at
 * (len(a), len(b)) and runs while both indices are positive (align.go:141), so a leading rest of
 * one string is not emitted, exactly as in the reference. */
int pg_nw_align_batch(const uint8_t *queries, const uint64_t *q_offsets, uint64_t n_queries,
                      const uint8_t *templ, uint64_t templ_len, int32_t query_is_a,
                      const int16_t *lut_a, const int16_t *lut_b, const int64_t *table,
                      int32_t n_a, int32_t n_b, int64_t gap, int64_t *score, int32_t *err_code,
                      int64_t *err_pos, uint8_t *align_a, uint8_t *align_b, uint64_t out_stride,
                      uint32_t *align_len, int32_t *status);

/* ---- align.SmithWaterman / align.NeedlemanWunsch over a list of pairs ----------------------
 * Pair p aligns stringA = A[pair_a[p]] (the reference's outer loop, the rows) against
 * stringB = B[pair_b[p]], where A (seqs_a, offsets_a, n_seqs_a) and B are ragged sets as in the
 * one-template calls.  A and B may be the same buffers; a pair list never copies a sequence.  Per
 * pair, score / err_code / err_pos are bit-identical to pg_sw_score_batch (pg_nw_score_batch) on
 * that (a, b): the first failing cell in row-major order, score 0 on error.  Alphabet limits and
 * the int32 / int64 score-width rule are those of the one-template calls, with the longest a and
 * the longest b of the call.
 * Host entry points: both sets are checked as ragged batches and every pair index against
 * n_seqs_a / n_seqs_b before anything is launched (PG_ERR_ARG, no output written).  n_pairs == 0
 * is PG_OK.  Both sets are uploaded once; pairs, outputs and scratch go in groups sized from the
 * device memory left free by the sets (at most 1 GiB of pairs and outputs per group), and the
 * long-pair scratch shrinks to what fits; PG_ERR_NOMEM only when the two sets plus one pair's
 * scratch do not fit.  Score width and scratch follow the longest a and b the pairs reference.
 * _dev score variants take device sets, pairs and outputs and host max_len_a / max_len_b, LUTs and
 * table; they only enqueue work on `stream` and never wait for the device.  A pair whose index is
 * out of range, or whose sequence is longer than max_len_a / max_len_b, gets
 * err_code = PG_PAIR_OUT_OF_RANGE, score 0 and err_pos -1; nothing out of bounds is read.
 * pg_sw_align_pairs / pg_nw_align_pairs add the aligned strings exactly as pg_sw_align_batch /
 * pg_nw_align_batch (align_a / align_b rows of out_stride bytes, align_len, status, with
 * PG_ITEM_UNSUPPORTED and the needed length when out_stride is too short).  Every pair of a group
 * keeps a whole (la + 1) x (lb + 1) matrix of 32-bit cells, la / lb the group's longest referenced
 * a / b: scores must fit 32 bits over la + lb cells, and one pair's matrix is limited to 16 Gi cells
 * (PG_ERR_UNSUPPORTED otherwise). */
#define PG_PAIR_OUT_OF_RANGE 3
int pg_sw_score_pairs(const uint8_t *seqs_a, const uint64_t *offsets_a, uint64_t n_seqs_a,
                      const uint8_t *seqs_b, const uint64_t *offsets_b, uint64_t n_seqs_b,
                      const uint32_t *pair_a, const uint32_t *pair_b, uint64_t n_pairs,
                      const int16_t *lut_a, const int16_t *lut_b, const int64_t *table,
                      int32_t n_a, int32_t n_b, int64_t gap,
                      int64_t *score, int32_t *err_code, int64_t *err_pos);
int pg_nw_score_pairs(const uint8_t *seqs_a, const uint64_t *offsets_a, uint64_t n_seqs_a,
                      const uint8_t *seqs_b, const uint64_t *offsets_b, uint64_t n_seqs_b,
                      const uint32_t *pair_a, const uint32_t *pair_b, uint64_t n_pairs,
                      const int16_t *lut_a, const int16_t *lut_b, const int64_t *table,
                      int32_t n_a, int32_t n_b, int64_t gap,
                      int64_t *score, int32_t *err_code, int64_t *err_pos);
int pg_sw_score_pairs_dev(const uint8_t *d_seqs_a, const uint64_t *d_offsets_a, uint64_t n_seqs_a, uint64_t max_len_a,
                          const uint8_t *d_seqs_b, const uint64_t *d_offsets_b, uint64_t n_seqs_b, uint64_t max_len_b,
                          const uint32_t *d_pair_a, const uint32_t *d_pair_b, uint64_t n_pairs,
                          const int16_t *lut_a_host, const int16_t *lut_b_host, const int64_t *table_host,
                          int32_t n_a, int32_t n_b, int64_t gap,
                          int64_t *d_score, int32_t *d_err_code, int64_t *d_err_pos, void *stream);
int pg_nw_score_pairs_dev(const uint8_t *d_seqs_a, const uint64_t *d_offsets_a, uint64_t n_seqs_a, uint64_t max_len_a,
                          const uint8_t *d_seqs_b, const uint64_t *d_offsets_b, uint64_t n_seqs_b, uint64_t max_len_b,
                          const uint32_t *d_pair_a, const uint32_t *d_pair_b, uint64_t n_pairs,
                          const int16_t *lut_a_host, const int16_t *lut_b_host, const int64_t *table_host,
                          int32_t n_a, int32_t n_b, int64_t gap,
                          int64_t *d_score, int32_t *d_err_code, int64_t *d_err_pos, void *stream);
int pg_sw_align_pairs(const uint8_t *seqs_a, const uint64_t *offsets_a, uint64_t n_seqs_a,
                      const uint8_t *seqs_b, const uint64_t *offsets_b, uint64_t n_seqs_b,
                      const uint32_t *pair_a, const uint32_t *pair_b, uint64_t n_pairs,
                      const int16_t *lut_a, const int16_t *lut_b, const int64_t *table,
                      int32_t n_a, int32_t n_b, int64_t gap,
                      int64_t *score, int32_t *err_code, int64_t *err_pos,
                      uint8_t *align_a, uint8_t *align_b, uint64_t out_stride, uint32_t *align_len, int32_t *status);
int pg_nw_align_pairs(const uint8_t *seqs_a, const uint64_t *offsets_a, uint64_t n_seqs_a,
                      const uint8_t *seqs_b, const uint64_t *offsets_b, uint64_t n_seqs_b,
                      const uint32_t *pair_a, const uint32_t *pair_b, uint64_t n_pairs,
                      const int16_t *lut_a, const int16_t *lut_b, const int64_t *table,
                      int32_t n_a, int32_t n_b, int64_t gap,
                      int64_t *score, int32_t *err_code, int64_t *err_pos,
                      uint8_t *align_a, uint8_t *align_b, uint64_t out_stride, uint32_t *align_len, int32_t *status);

/* ---- align.NeedlemanWunsch score -- search/align/align.go:100-134 (fill) and :166 --------
 * (a "next" row of SURVEY.md 8f).  Same arguments and error semantics as the Smith-Waterman
 * entry points; score = matrix[len(a)][len(b)] of the global alignment (gap ramps on the first
 * row and column, no zero floor). */
int pg_nw_score_batch(const uint8_t *queries, const uint64_t *q_offsets, uint64_t n_queries,
                      const uint8_t *templ, uint64_t templ_len, int32_t query_is_a,
                      const int16_t *lut_a, const int16_t *lut_b, const int64_t *table,
                      int32_t n_a, int32_t n_b, int64_t gap, int64_t *score, int32_t *err_code,
                      int64_t *err_pos);
int pg_nw_score_batch_dev(const uint8_t *d_queries, const uint64_t *d_q_offsets, uint64_t n_queries,
                          uint64_t max_query_len, const uint8_t *d_templ, uint64_t templ_len,
                          int32_t query_is_a, const int16_t *lut_a_host, const int16_t *lut_b_host,
                          const int64_t *table_host, int32_t n_a, int32_t n_b, int64_t gap,
                          int64_t *d_score, int32_t *d_err_code, int64_t *d_err_pos, void *stream);

/* ---- primers.SantaLucia / MeltingTemp -- primers/primers.go:70-105,121-128 --------
 * tm/dh/ds may each be NULL.  status: PG_ITEM_PANIC for an empty primer
 * (primers.go:89), PG_ITEM_UNSUPPORTED for a byte >= 0x80 (strings.ToUpper would
 * re-encode it, primers.go:71).  MeltingTemp == cp 500e-9, na 50e-3, mg 0. */
int pg_tm_batch(const uint8_t *bases, const uint64_t *offsets, uint64_t n, double cp, double na,
                double mg, double *tm, double *dh, double *ds, int32_t *status);
int pg_tm_batch_dev(const uint8_t *d_bases, const uint64_t *d_offsets, uint64_t n, double cp,
                    double na, double mg, double *d_tm, double *d_dh, double *d_ds,
                    int32_t *d_status, void *stream);

/* ---- pcr.DesignPrimersWithOverhangs core -- primers/pcr/pcr.go:44-60 (SURVEY.md 8f.3) ---------
 * For each sequence: fwd_len = length of the forward primer (shortest prefix of >= 15 nt of the
 * upper-cased sequence with MeltingTemp >= target_tm, pcr.go:46-49), rev_len = length of the
 * reverse primer (reverse complement of the shortest such suffix, pcr.go:50-53).  Every candidate
 * is evaluated exactly as primers.MeltingTemp would.  status: PG_ITEM_PANIC where the reference
 * slices out of range (sequence shorter than 15 nt or exhausted before the target is reached),
 * PG_ITEM_UNSUPPORTED for bytes >= 0x80.  The primer strings themselves (overhang + primer,
 * pcr.go:55-59) are assembled by the caller from the lengths. */
int pg_design_primers_batch(const uint8_t *bases, const uint64_t *offsets, uint64_t n,
                            double target_tm, uint32_t *fwd_len, uint32_t *rev_len, int32_t *status);

/* ---- pcr.SimulateSimple building blocks -- primers/pcr/pcr.go:73-169 (SURVEY.md 8f.3) ---------
 * pg_pcr_minimal_primer_batch: the minimal-primer loop of pcr.go:93-100 for every primer:
 * min_len = the longest 3' suffix of >= 7 nt (minimalPrimerLength, pcr.go:35) whose MeltingTemp is still below target_tm (the
 * reference's loop keeps the last length that FAILED the test), 0 when the 7-mer already reaches
 * it, the primer's length when even the whole primer stays below (the reference then ignores the
 * primer, pcr.go:103).  status: PG_ITEM_PANIC for primers shorter than 7 nt, PG_ITEM_UNSUPPORTED
 * for bytes >= 0x80.
 * pg_find_sites_batch: every (possibly overlapping) exact occurrence of every pattern in every
 * sequence -- what suffixarray.Lookup(pattern, -1) returns at pcr.go:110,113; empty patterns have
 * none.  flags & PG_SITES_UPPER compares the ASCII-upper-cased sequence bytes (pcr.go:82).  Hits
 * come back unordered as (sequence index, position inside it, pattern index); *n_hits is the
 * number found, PG_ERR_ARG (with the first hits_cap stored) if it exceeds hits_cap. */
#define PG_SITES_UPPER 1u
int pg_pcr_minimal_primer_batch(const uint8_t *bases, const uint64_t *offsets, uint64_t n,
                                double target_tm, uint32_t *min_len, int32_t *status);
int pg_find_sites_batch(const uint8_t *seqs, const uint64_t *seq_offsets, uint64_t n_seq,
                        const uint8_t *patterns, const uint64_t *pat_offsets, uint32_t n_pat,
                        uint32_t flags, uint32_t *hit_seq, uint64_t *hit_pos, uint32_t *hit_pat,
                        uint64_t hits_cap, uint64_t *n_hits);

/* ---- FASTQ ingest -- io/fastq Parser.ParseNext / ParseN, io/fastq/fastq.go:88-99,117-214 -------
 * (SURVEY.md 8f.2: the step before the hot path.)  Parses a whole FASTQ text buffer on the GPU
 * into the dense bases + offsets layout the sketch entry points take.  Strict 4-line records;
 * parsing stops at the first record the reference rejects and the records before it are returned
 * together with the error, as ParseN does: *err_code 0 none, 1 a line of a record is not newline
 * terminated (EOF inside a record), 2 empty sequence, 3 empty quality, 4 no '@', 5 the reference
 * panics (empty identifier line, or an optional datum without '='), 6 line longer than the 64 KiB
 * reader of fastq.Parse; *err_line = 1-based number of the line the reference stops at.
 * Returns PG_ERR_ARG when a capacity is too small (*n_records / *total_bases hold the needs).
 * The _dev variant takes device buffers (text, bases, offsets) and host scalars. */
int pg_fastq_ingest(const uint8_t *text, uint64_t nbytes, uint8_t *bases, uint64_t bases_cap,
                    uint64_t *offsets, uint64_t records_cap, uint64_t *n_records,
                    uint64_t *total_bases, int32_t *err_code, uint64_t *err_line);
int pg_fastq_ingest_dev(const uint8_t *d_text, uint64_t nbytes, uint8_t *d_bases, uint64_t bases_cap,
                        uint64_t *d_offsets, uint64_t records_cap, uint64_t *n_records,
                        uint64_t *total_bases, int32_t *err_code, uint64_t *err_line, void *stream);

/* The same plus what fastq.Fastq holds besides the sequence (io/fastq/fastq.go:46-51): for record i
 * spans[4i .. 4i+3] = {begin, length of the identifier line (with its '@', without the newline),
 * begin, length of the quality line} as offsets into `text`.  The caller cuts Identifier
 * (strings.Split(line, " ")[0][1:], fastq.go:158), Optionals (the "key=value" tokens, fastq.go:159-165)
 * and Quality (fastq.go:199) out of the text it already holds: no second copy of the text is made. */
int pg_fastq_ingest_records(const uint8_t *text, uint64_t nbytes, uint8_t *bases, uint64_t bases_cap,
                            uint64_t *offsets, uint64_t *spans, uint64_t records_cap, uint64_t *n_records,
                            uint64_t *total_bases, int32_t *err_code, uint64_t *err_line);
int pg_fastq_ingest_records_dev(const uint8_t *d_text, uint64_t nbytes, uint8_t *d_bases, uint64_t bases_cap,
                                uint64_t *d_offsets, uint64_t *d_spans, uint64_t records_cap, uint64_t *n_records,
                                uint64_t *total_bases, int32_t *err_code, uint64_t *err_line, void *stream);

/* ---- FASTA ingest -- fasta.Parse = NewParser(r, maxLineSize).ParseAll(),
 * io/fasta/fasta.go:72-77,96-118,149-243 (SURVEY.md 8f.2) -----------------------------------------
 * Parses a whole FASTA text buffer on the GPU into dense sequences + offsets and (optionally:
 * pass names, name_offsets both non-NULL) dense names + name_offsets, n_records + 1 offsets each.
 * max_line_size as NewParser's (fasta.Parse uses 65536; values < 16 behave as 16 like
 * bufio.NewReaderSize).  Semantics are ParseNext's, quirks included: lines of length <= 1 and
 * ';' lines are skipped, a '>' line directly after a name line is sequence text, a record
 * without a trailing newline at the end of the text is dropped without an error, and parsing
 * stops at the first error with the records before it returned: *err_code 0 none,
 * 1 "did not find fasta start '>'", 2 "empty fasta sequence", 3 "line too large for buffer"
 * (>= max_line_size content bytes), 4 bufio.ErrBufferFull (over-long ';' line inside a record);
 * *err_line = the line number the reference's message prints.
 * flags & PG_FASTA_BUFIO_ALIAS: also reproduce the reference's use of the bufio line slice after
 * Peek(1) (fasta.go:192): a line whose newline is the last byte of a full reader buffer is seen
 * with its bytes replaced by the text one buffer further on, exactly as fasta.Parse over a
 * strings.Reader / bytes.Reader / *os.File yields.  Without the flag lines are taken as written.
 * Returns PG_ERR_ARG when a capacity is too small (*n_records, *total_bases, *total_name_bytes
 * then hold the needs; nbytes bounds both byte counts, the newline count + 1 the records). */
#define PG_FASTA_BUFIO_ALIAS 1u
int pg_fasta_ingest(const uint8_t *text, uint64_t nbytes, uint32_t max_line_size, uint32_t flags,
                    uint8_t *bases, uint64_t bases_cap, uint64_t *offsets, uint8_t *names,
                    uint64_t names_cap, uint64_t *name_offsets, uint64_t records_cap,
                    uint64_t *n_records, uint64_t *total_bases, uint64_t *total_name_bytes,
                    int32_t *err_code, uint64_t *err_line);
int pg_fasta_ingest_dev(const uint8_t *d_text, uint64_t nbytes, uint32_t max_line_size, uint32_t flags,
                        uint8_t *d_bases, uint64_t bases_cap, uint64_t *d_offsets, uint8_t *d_names,
                        uint64_t names_cap, uint64_t *d_name_offsets, uint64_t records_cap,
                        uint64_t *n_records, uint64_t *total_bases, uint64_t *total_name_bytes,
                        int32_t *err_code, uint64_t *err_line, void *stream);

/* ---- seqhash.Hash -- seqhash/seqhash.go:141-223 ----------------------------------------------------
 * One call hashes sequences [offsets[i], offsets[i+1]) of `seqs` (n + 1 offsets), all of one
 * seq_type (PG_SEQHASH_DNA / _RNA / _PROTEIN) and with one set of flags (PG_SEQHASH_CIRCULAR |
 * PG_SEQHASH_DOUBLE_STRANDED); another seq_type or flag bit is PG_ERR_ARG.  Per sequence, as Hash:
 * ASCII upper-case, U -> T for RNA, the alphabet check in order (DNA/RNA "ATUGCYRSWKMBDHVNZ", protein
 * "ACDEFGHIKLMNPQRSTVWYUO*BXZ"), then "Proteins cannot be double stranded"; the deterministic
 * sequence (least rotation when circular, the smaller of s and transform.ReverseComplement(s) -- or of
 * their least rotations -- when double-stranded; the complement of the DNA letters U and Z is the
 * byte 0x00, as in the reference) and digest[32 i .. 32 i + 31] = BLAKE3-256 of it.  The Seqhash
 * string is "v1_" + {D,R,P} + {C,L} + {D,S} + "_" + hex(digest).
 * err_code[i]: 0 ok; 1 a letter outside the alphabet, err_pos[i] = its byte index; 2 "Proteins cannot
 * be double stranded"; 3 a byte >= 0x80 comes before any letter outside the alphabet (strings.ToUpper
 * would re-encode it: unsupported, not hashed; err_pos[i] = its byte index).  Failed sequences get a
 * zero digest; err_code and err_pos may be NULL.  Sequences may be of any length: the host entry point
 * hashes them in groups under a device-memory budget (a single sequence needs about twice its length
 * of device memory; PG_ERR_NOMEM when that does not fit).
 * pg_seqhash_batch_dev: device pointers, max_len >= every sequence length, digest 4-byte aligned.  It
 * reads offsets[0] and offsets[n] back to the host to size its scratch (so it waits for earlier work on
 * the stream), then only enqueues: it returns before the hashes are computed. */
#define PG_SEQHASH_DNA 0
#define PG_SEQHASH_RNA 1
#define PG_SEQHASH_PROTEIN 2
#define PG_SEQHASH_CIRCULAR 1u
#define PG_SEQHASH_DOUBLE_STRANDED 2u
int pg_seqhash_batch(const uint8_t *seqs, const uint64_t *offsets, uint64_t n, int32_t seq_type,
                     uint32_t flags, uint8_t *digest, int32_t *err_code, uint64_t *err_pos);
int pg_seqhash_batch_dev(const uint8_t *d_seqs, const uint64_t *d_offsets, uint64_t n, int32_t seq_type,
                         uint32_t flags, uint8_t *d_digest, int32_t *d_err_code, uint64_t *d_err_pos,
                         uint64_t max_len, void *stream);
/* seqhash.RotateSequence / boothLeastRotation (seqhash.go:78-138) on the raw bytes (no case folding):
 * rotation[i] = the smallest start of the lexicographically least rotation of sequence i (0 when
 * empty); RotateSequence(s) = s[r:] + s[:r]. */
int pg_least_rotation_batch(const uint8_t *seqs, const uint64_t *offsets, uint64_t n, uint64_t *rotation);

/* ---- fold.Zuker -- fold/fold.go, fold/seqfold.go ----------------------------------------------------
 * Folds sequences [offsets[i], offsets[i+1]) of `seqs` (n + 1 offsets) at temp degrees Celsius, as
 * Zuker(seq, temp) followed by Result.MinimumFreeEnergy() and Result.DotBracket():
 * mfe[i] (float64, bit for bit the reference's sum), the dot-bracket at dot_bracket[offsets[i] -
 * offsets[0] ..] (laid out like seqs; it is never longer than the sequence) and its length db_len[i].
 * status[i] (may be NULL): PG_ITEM_OK; PG_ITEM_FOLD_NOT_NUCLEIC where the upper-cased sequence is
 * neither DNA (ACGT) nor RNA (ACGU), the reference's error "the sequence %s is not RNA or DNA";
 * PG_ITEM_PANIC where the reference panics (0 or 1 nt, or a traceback shift out of range);
 * PG_ITEM_UNSUPPORTED for a byte >= 0x80 (strings.ToUpper would re-encode it) or more than
 * PG_FOLD_MAX_LEN nt; PG_ITEM_FOLD_INTERNAL if one of the reference's internal errors fired.  Items
 * that are not OK get mfe 0, db_len 0 and '.' over their region of dot_bracket.  Returns PG_ERR_PANIC if any item panics, else
 * PG_ERR_UNSUPPORTED if any is unsupported, with every output written.  Items go to the device in
 * groups under a device-memory budget (about 34 n^2 + 0.13 n^3 bytes of scratch per n-nt item). */
#define PG_FOLD_MAX_LEN 1024
int pg_fold_zuker_batch(const uint8_t *seqs, const uint64_t *offsets, uint64_t n, double temp, double *mfe,
                        uint8_t *dot_bracket, uint64_t *db_len, int32_t *status);

/* ---- synthesis/fragment: Fragment, FragmentWithOverhangs, SetEfficiency, NextOverhangs ----------------
 * pg_fragment_batch: Fragment(seq, min_size, max_size, exclude) of every sequence [offsets[i], offsets[i+1])
 * of `seqs`, or FragmentWithOverhangs(..., exclude, include) when n_include > 0.  The exclude and include
 * lists (ragged, n_exclude + 1 and n_include + 1 offsets) are shared by the whole batch; overhangs are any
 * bytes of any length and are used exactly as given (only the sequence is upper-cased).  Per item:
 * status[i] (may be NULL) PG_ITEM_OK; PG_ITEM_FRAGMENT_MIN_GT_MAX / _MIN_LT_12 with the failing step's
 * values in err_min[i] / err_max[i] (after an end-game adjustment these are the adjusted values);
 * PG_ITEM_FRAGMENT_NO_POSITION; PG_ITEM_PANIC for fewer than 4 bytes; PG_ITEM_UNSUPPORTED for a byte >= 0x80.
 * efficiency[i] is the reference's float64, bit for bit (0 unless OK).  The fragments are given by their
 * ends: item i has frag_offsets[i+1] - frag_offsets[i] of them (0 unless OK) at ends[frag_offsets[i] ..];
 * fragment j is [start_j, end_j) of the item with start_0 = 0 and start_j = end_{j-1} - 4, and the last end
 * is the item's length.  *n_ends (the total) and frag_offsets (n + 1 entries) are always written; more ends
 * than ends_cap is PG_ERR_ARG with every other output written, and nothing written past ends[ends_cap]
 * (ends may hold the ends of the leading items, which went to the device first).  Otherwise returns
 * PG_ERR_PANIC if any item panics, else PG_ERR_UNSUPPORTED if any is unsupported, with every output
 * written.  Items go to the device in groups under a device-memory budget. */
int pg_fragment_batch(const uint8_t *seqs, const uint64_t *offsets, uint64_t n, int64_t min_size, int64_t max_size, const uint8_t *exclude,
                      const uint64_t *exclude_offsets, uint64_t n_exclude, const uint8_t *include, const uint64_t *include_offsets,
                      uint64_t n_include, int32_t *status, double *efficiency, int64_t *err_min, int64_t *err_max, uint64_t *frag_offsets,
                      uint64_t *ends, uint64_t ends_cap, uint64_t *n_ends);
/* Set i is the overhangs [set_offsets[i], set_offsets[i+1]) of the ragged list (overhangs, overhang_offsets),
 * in order (duplicates count).  pg_fragment_set_efficiency_batch: efficiency[i] = SetEfficiency(set i).
 * pg_fragment_next_overhangs_batch: NextOverhangs(set i): n_cands[i] candidates at cands[1024 i ..]
 * (4 bytes each, in the reference's order) and their efficiencies at efficiency[256 i ..]. */
int pg_fragment_set_efficiency_batch(const uint8_t *overhangs, const uint64_t *overhang_offsets, const uint64_t *set_offsets, uint64_t n_sets,
                                     double *efficiency);
int pg_fragment_next_overhangs_batch(const uint8_t *overhangs, const uint64_t *overhang_offsets, const uint64_t *set_offsets, uint64_t n_sets,
                                     uint8_t *cands, uint32_t *n_cands, double *efficiency);

/* ---- clone.CutWithEnzyme / CircularLigate / GoldenGate -- clone/clone.go:138-355 --------------------
 * An enzyme: RegexpFor and RegexpRev as literal sites (1..32 bytes of 0x01..0x7f; anything else is
 * PG_ERR_UNSUPPORTED: the library does not implement Go's regexp language), Skip, OverheadLength and
 * RecognitionSite.  Palindromic = RecognitionSite equals its reverse complement (checks.IsPalindromic).
 * Skip and OverheadLength are Go ints held here as int32: only -2^31 .. 2^31 - 1 is supported, and the
 * Python and Go bindings refuse a wider value as unsupported instead of narrowing it (a wrapped Skip cuts
 * somewhere else). */
typedef struct {
    const uint8_t *forward_site;
    uint32_t forward_len;
    const uint8_t *reverse_site;
    uint32_t reverse_len;
    const uint8_t *recognition_site;
    uint32_t recognition_len;
    int32_t skip;
    int32_t overhang_length;
} pg_clone_enzyme;
/* CutWithEnzyme(part p, directional, enzyme e) for every item i = p * n_enzymes + e, exactly as the
 * reference (quirks included): ToUpper(part) or ToUpper(part + part) when circular[p] != 0, leftmost
 * non-overlapping matches of each site, the linear drop of the last overhang of a set, the stable sort,
 * the four fragment branches and the len > 8 filter.  Per item: frag_count[i] and status[i] (may be
 * NULL): PG_ITEM_PANIC where a slice of the reference is out of range (no fragments; the call returns
 * PG_ERR_PANIC after writing everything else), PG_ITEM_UNSUPPORTED for a byte >= 0x80 (strings.ToUpper
 * would re-encode it).  Fragments in item order: Sequence f = seq_bytes[seq_offsets[f], seq_offsets[f+1]),
 * ForwardOverhang = oh_bytes[oh_offsets[2f], oh_offsets[2f+1]), ReverseOverhang = oh_bytes[oh_offsets[2f+1],
 * oh_offsets[2f+2]); seq_offsets has frag_cap + 1 entries, oh_offsets 2 * frag_cap + 1.  *n_frags,
 * *n_seq_bytes and *n_oh_bytes are always written; more than frag_cap, seq_cap or oh_cap is PG_ERR_ARG
 * (frag_count and status are written, the fragments are not).  A batch in which a part could hold 2^32 or
 * more matches of a site (2 L / site length for a circular part) is PG_ERR_ARG before any launch. */
int pg_clone_digest_batch(const uint8_t *parts, const uint64_t *part_offsets, const uint8_t *circular, uint64_t n_parts,
                          const pg_clone_enzyme *enzymes, uint32_t n_enzymes, int32_t directional, uint32_t *frag_count,
                          int32_t *status, uint8_t *seq_bytes, uint64_t seq_cap, uint64_t *seq_offsets, uint8_t *oh_bytes,
                          uint64_t oh_cap, uint64_t *oh_offsets, uint64_t frag_cap, uint64_t *n_frags, uint64_t *n_seq_bytes,
                          uint64_t *n_oh_bytes);
/* GoldenGate(parts of reaction r, enzyme) for n_reactions independent reactions: reaction r is parts
 * [reaction_offsets[r], reaction_offsets[r+1]) (reaction_offsets runs from 0 to n_parts).  All parts are
 * digested (directional) in one launch; recurseLigate runs on the host over fragment ids; every
 * construct it would hash is built and seqhashed on the device, in groups under a device-memory budget.
 * Per reaction the output keeps, in the reference's order, the first construct of each seqhash, as
 * CircularLigate's existingSeqhashes does.  Outputs: constructs of reaction 0, then 1, ..., each reaction's
 * in the reference's hashing order; construct k = out[construct_offsets[k], construct_offsets[k+1]),
 * kinds[k] 0 a clone (openConstructs) or 1 a looping construct (infiniteLoops), digests[32 k ..] its seqhash
 * digest (kinds and digests may be NULL); counts[2 r], counts[2 r + 1] = clones and loops of reaction r.
 * The work is bounded by the caller: *need_bytes and *need_constructs (always written) are the bytes and
 * the number of all constructs the ligations hash, duplicates included; more than bytes_cap or
 * constructs_cap is PG_ERR_ARG before anything is built.  Sized at the need, out holds bytes_cap bytes and
 * construct_offsets constructs_cap + 1 entries.  status[r] (may be NULL): PG_ITEM_PANIC / _UNSUPPORTED
 * when a part of the reaction cuts that way (the reaction has no constructs; the call returns
 * PG_ERR_PANIC / PG_ERR_UNSUPPORTED after writing everything else). */
int pg_clone_golden_gate_batch(const uint8_t *parts, const uint64_t *part_offsets, const uint8_t *circular, uint64_t n_parts,
                               const uint64_t *reaction_offsets, uint64_t n_reactions, const pg_clone_enzyme *enzyme,
                               uint64_t bytes_cap, uint64_t constructs_cap, uint8_t *out, uint64_t *construct_offsets,
                               uint8_t *kinds, uint8_t *digests, uint64_t *counts, int32_t *status, uint64_t *need_bytes,
                               uint64_t *need_constructs);
/* CircularLigate on caller-given fragments, in pg_clone_digest_batch's layout (n_frags fragments),
 * grouped into reactions by reaction_offsets (from 0 to n_frags); outputs as pg_clone_golden_gate_batch.
 * A fragment byte >= 0x80 is PG_ERR_UNSUPPORTED before anything is launched: seqhash.Hash's
 * strings.ToUpper would re-encode it (and maps some such letters into the alphabet). */
int pg_clone_circular_ligate_batch(const uint8_t *seq_bytes, const uint64_t *seq_offsets, const uint8_t *oh_bytes,
                                   const uint64_t *oh_offsets, uint64_t n_frags, const uint64_t *reaction_offsets,
                                   uint64_t n_reactions, uint64_t bytes_cap, uint64_t constructs_cap, uint8_t *out,
                                   uint64_t *construct_offsets, uint8_t *kinds, uint8_t *digests, uint64_t *counts,
                                   uint64_t *need_bytes, uint64_t *need_constructs);

/* ---- synthetic workloads (SURVEY.md 8d; bench/test tooling, not a reference API) ---
 * kind 0: independent reads  base(i,j) = code(seed, i*L + j)
 * kind 1: family reads       (family = reads per template, 1/64 substitutions)
 * Writes n_reads*read_len bytes for reads [first_read, first_read+n_reads). */
int pg_synth_reads_dev(uint8_t *d_bases, uint64_t first_read, uint64_t n_reads, uint32_t read_len,
                       uint64_t seed, int32_t kind, uint32_t family, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* POLY_B200_H */
