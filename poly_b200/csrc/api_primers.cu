// api_primers.cu -- the C ABI of poly's primers and pcr (SantaLucia Tm, DesignPrimers, the minimal primer)
// and of the site search.
#include <vector>

#include "runtime.cuh"

using namespace pg;

extern "C" {

// ---------------------------------------------------------------------------------
// SantaLucia Tm
// ---------------------------------------------------------------------------------
int pg_tm_batch_dev(const uint8_t *d_bases, const uint64_t *d_offsets, uint64_t n, double cp,
                    double na, double mg, double *d_tm, double *d_dh, double *d_ds, int32_t *d_status,
                    void *stream) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    return launch_tm(d_bases, d_offsets, n, cp, na, mg, d_tm, d_dh, d_ds, d_status, (cudaStream_t)stream);
}

int pg_tm_batch(const uint8_t *bases, const uint64_t *offsets, uint64_t n, double cp, double na,
                double mg, double *tm, double *dh, double *ds, int32_t *status) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if (n == 0) return PG_OK;
    if (!offsets) { set_error("null offsets"); return PG_ERR_ARG; }
    HostCall c;
    const Ragged<uint8_t> b = c.ragged(bases, offsets, n);
    double *d_tm = c.alloc<double>(n, true), *d_dh = c.alloc<double>(n, true), *d_ds = c.alloc<double>(n, true);
    int32_t *d_st = c.alloc<int32_t>(n);
    if ((rc = c.error()) || (rc = launch_tm(b.base, b.off, n, cp, na, mg, d_tm, d_dh, d_ds, d_st, c.st))) return rc;
    std::vector<int32_t> hst(n);
    c.download(tm, d_tm, n);
    c.download(dh, d_dh, n);
    c.download(ds, d_ds, n);
    c.download(hst.data(), d_st, n);
    if ((rc = c.finish())) return rc;
    return fold_item_status(hst, status, "at least one primer is empty: primers.SantaLucia panics (index out of range)",
                            "at least one primer holds a byte >= 0x80 (unsupported: strings.ToUpper would re-encode it)");
}

int pg_design_primers_batch(const uint8_t *bases, const uint64_t *offsets, uint64_t n,
                            double target_tm, uint32_t *fwd_len, uint32_t *rev_len, int32_t *status) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if (n == 0) return PG_OK;
    if (!offsets || !fwd_len || !rev_len) { set_error("null buffer"); return PG_ERR_ARG; }
    HostCall c;
    const Ragged<uint8_t> b = c.ragged(bases, offsets, n);
    uint32_t *d_f = c.alloc<uint32_t>(n), *d_r = c.alloc<uint32_t>(n);
    int32_t *d_st = c.alloc<int32_t>(n);
    if ((rc = c.error()) || (rc = launch_design_primers(b.base, b.off, n, target_tm, d_f, d_r, d_st, c.st))) return rc;
    std::vector<int32_t> hst(n);
    c.download(fwd_len, d_f, n);
    c.download(rev_len, d_r, n);
    c.download(hst.data(), d_st, n);
    if ((rc = c.finish())) return rc;
    return fold_item_status(hst, status, "at least one sequence is exhausted before the target Tm: pcr.DesignPrimers panics (slice bounds out of range)",
                            "at least one sequence holds a byte >= 0x80 (unsupported)");
}

int pg_pcr_minimal_primer_batch(const uint8_t *bases, const uint64_t *offsets, uint64_t n, double target_tm,
                                uint32_t *min_len, int32_t *status) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if (n == 0) return PG_OK;
    if (!offsets || !min_len) { set_error("null buffer"); return PG_ERR_ARG; }
    HostCall c;
    const Ragged<uint8_t> b = c.ragged(bases, offsets, n);
    uint32_t *d_m = c.alloc<uint32_t>(n);
    int32_t *d_st = c.alloc<int32_t>(n);
    if ((rc = c.error()) || (rc = launch_minimal_primer(b.base, b.off, n, target_tm, d_m, d_st, c.st))) return rc;
    std::vector<int32_t> hst(n);
    c.download(min_len, d_m, n);
    c.download(hst.data(), d_st, n);
    if ((rc = c.finish())) return rc;
    return fold_item_status(hst, status, "at least one primer is shorter than 7 nt: pcr.SimulateSimple panics (slice bounds out of range)",
                            "at least one primer holds a byte >= 0x80 (unsupported)");
}

int pg_find_sites_batch(const uint8_t *seqs, const uint64_t *seq_offsets, uint64_t n_seq, const uint8_t *patterns,
                        const uint64_t *pat_offsets, uint32_t n_pat, uint32_t flags, uint32_t *hit_seq, uint64_t *hit_pos,
                        uint32_t *hit_pat, uint64_t hits_cap, uint64_t *n_hits) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if (!n_hits) { set_error("null buffer"); return PG_ERR_ARG; }
    *n_hits = 0;
    if (n_seq == 0 || n_pat == 0) return PG_OK;
    if (!seq_offsets || !pat_offsets || (hits_cap && (!hit_seq || !hit_pos || !hit_pat))) { set_error("null buffer"); return PG_ERR_ARG; }
    HostCall c;
    const Ragged<uint8_t> sq = c.ragged(seqs, seq_offsets, n_seq);
    uint64_t max_pat_len;
    if ((rc = c.error()) || (rc = check_ragged(pat_offsets, n_pat, &max_pat_len))) return rc;
    const uint64_t sbytes = seq_offsets[n_seq] - seq_offsets[0], p0 = pat_offsets[0], pbytes = pat_offsets[n_pat] - p0;
    std::vector<uint64_t> poff(n_pat + 1);
    for (uint32_t q = 0; q <= n_pat; ++q) poff[q] = pat_offsets[q] - p0;  // the kernel stages patterns from offset 0
    const uint8_t *d_p = c.upload(patterns + p0, pbytes);
    const uint64_t *d_poff = c.upload(poff.data(), n_pat + 1);
    uint32_t *d_hs = c.alloc<uint32_t>(hits_cap), *d_hq = c.alloc<uint32_t>(hits_cap);
    uint64_t *d_hp = c.alloc<uint64_t>(hits_cap);
    unsigned long long *d_n = c.alloc<unsigned long long>(1, true);
    if ((rc = c.error()) || (rc = launch_find_sites(sq.base, sq.off, n_seq, sbytes, d_p, d_poff, n_pat, pbytes, flags, d_hs, d_hp, d_hq, hits_cap,
                                                    d_n, c.st)))
        return rc;
    return finish_capped(c, d_n, hits_cap, n_hits, {{hit_seq, d_hs, 4}, {hit_pos, d_hp, 8}, {hit_pat, d_hq, 4}}, "hits_cap", "occurrences");
}

}  // extern "C"
