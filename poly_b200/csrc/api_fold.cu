// api_fold.cu -- the C ABI of poly's fold: Zuker minimum free energy and dot-bracket structures.
#include <vector>

#include "runtime.cuh"

using namespace pg;

extern "C" {

// ---- fold.Zuker (fold.cu) -----------------------------------------------------------------------------
int pg_fold_zuker_batch(const uint8_t *seqs, const uint64_t *offsets, uint64_t n, double temp, double *mfe, uint8_t *dot_bracket,
                        uint64_t *db_len, int32_t *status) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if (n == 0) return PG_OK;
    if (!offsets) { set_error("null offsets"); return PG_ERR_ARG; }
    uint64_t max_len;  // the whole batch is checked before the first group is launched
    if ((rc = check_ragged(offsets, n, &max_len)) != PG_OK) return rc;
    if (!mfe || !dot_bracket || !db_len) { set_error("null mfe, dot_bracket or db_len"); return PG_ERR_ARG; }
    // An item's device memory: its scratch (V and W cells, branch lists), input and structure, and its words.
    const uint64_t budget = group_budget(8ull << 30);
    auto cost = [&](uint64_t i) { return fold_scratch_bytes(offsets[i + 1] - offsets[i]) + 2 * (offsets[i + 1] - offsets[i]) + 64; };
    const std::vector<uint8_t> tables = fold_tables(temp);
    std::vector<int32_t> hst(n);
    std::vector<uint64_t> scr;
    for (uint64_t g = 0; g < n;) {
        const uint64_t e = group_end(g, n, budget, cost), cnt = e - g, bytes = offsets[e] - offsets[g];
        scr.assign(1, 0);
        for (uint64_t i = g; i < e; ++i) scr.push_back(scr.back() + fold_scratch_bytes(offsets[i + 1] - offsets[i]));
        HostCall c;
        const Ragged<uint8_t> in = c.ragged(seqs, offsets + g, cnt);
        uint8_t *d_tab = c.upload(tables.data(), tables.size());
        uint64_t *d_scr_off = c.upload(scr.data(), cnt);
        uint8_t *d_scratch = c.alloc<uint8_t>(std::max<uint64_t>(scr.back(), 8));
        double *d_mfe = c.alloc<double>(cnt);
        uint8_t *d_db = c.alloc<uint8_t>(bytes);
        uint64_t *d_len = c.alloc<uint64_t>(cnt);
        int32_t *d_st = c.alloc<int32_t>(cnt);
        if ((rc = c.error()) || (rc = launch_fold_zuker(in.base, in.off, cnt, d_tab, d_scratch, d_scr_off, d_mfe, d_db, d_len, d_st, c.st))) return rc;
        c.download(mfe + g, d_mfe, cnt);
        c.download(dot_bracket + (offsets[g] - offsets[0]), d_db, bytes);
        c.download(db_len + g, d_len, cnt);
        c.download(hst.data() + g, d_st, cnt);
        if ((rc = c.finish()) != PG_OK) return rc;
        g = e;
    }
    return fold_item_status(hst, status, "at least one sequence makes fold.Zuker panic (empty, 1 nt, or a traceback index out of range)",
                            "at least one sequence holds a byte >= 0x80 or is longer than PG_FOLD_MAX_LEN (unsupported)");
}

}  // extern "C"
