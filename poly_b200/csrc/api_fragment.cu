// api_fragment.cu -- the C ABI of poly's synthesis/fragment: Fragment, SetEfficiency and NextOverhangs.
#include <algorithm>
#include <vector>

#include "runtime.cuh"

namespace pg {
namespace {

// SetEfficiency (next = 0) or NextOverhangs (next = 1) of every set, in groups of sets under the budget
static int overhang_sets(const uint8_t *overhangs, const uint64_t *overhang_offsets, const uint64_t *set_offsets, uint64_t n_sets, int next,
                         uint8_t *cands, uint32_t *n_cands, double *efficiency) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if (n_sets == 0) return PG_OK;
    if (!set_offsets || !efficiency || (next && (!cands || !n_cands))) { set_error("null buffer"); return PG_ERR_ARG; }
    uint64_t widest;
    if ((rc = check_ragged(set_offsets, n_sets, &widest))) return rc;
    const uint64_t n_ov = set_offsets[n_sets];
    if (n_ov && !overhang_offsets) { set_error("null overhang_offsets"); return PG_ERR_ARG; }
    if (n_ov && (rc = check_ragged(overhang_offsets, n_ov, &widest))) return rc;
    if (n_ov && overhang_offsets[n_ov] > overhang_offsets[0] && !overhangs) { set_error("null overhangs with non-empty entries"); return PG_ERR_ARG; }
    // the most keyed members of any set bounds the per-warp spill of its key list (every 4-byte member may be one)
    uint64_t max_keys = 0;
    for (uint64_t s = 0; s < n_sets; ++s) {
        uint64_t k = 0;
        for (uint64_t j = set_offsets[s]; j < set_offsets[s + 1]; ++j) k += overhang_offsets[j + 1] - overhang_offsets[j] == 4;
        max_keys = std::max(max_keys, k);
    }
    const FragmentHost h = fragment_host(nullptr, nullptr, 0, nullptr, nullptr, 0);
    const uint64_t budget = group_budget(4ull << 30), per_set = next ? 256 * (4 + 8) + 4 : 8;
    auto cost = [&](uint64_t) { return per_set; };
    HostCall c;
    const uint64_t zero = 0;
    const Ragged<uint8_t> in = n_ov ? c.ragged(overhangs, overhang_offsets, n_ov) : Ragged<uint8_t>{nullptr, c.upload(&zero, 1), 0};
    SetArgs a{};
    a.fid = c.upload(h.fid.data(), h.fid.size());
    a.ov = in.base;
    a.ov_off = in.off;
    a.set_off = c.upload(set_offsets, n_sets + 1);
    a.next = next;
    const uint64_t m0 = group_end(0, n_sets, budget, cost);  // no later group holds more sets
    a.eff = c.alloc<double>(next ? 256 * m0 : m0);
    if (next) {
        a.cands = c.alloc<uint8_t>(1024 * m0);
        a.n_cands = c.alloc<uint32_t>(m0);
    }
    if ((rc = c.error())) return rc;
    for (uint64_t g = 0; g < n_sets; g += a.n_sets) {
        a.first = g;
        a.n_sets = group_end(g, n_sets, budget, cost) - g;
        StreamScratch work(c.st);
        if ((rc = launch_overhang_sets(a, max_keys, budget, work, c.st))) return rc;
        c.download(efficiency + (next ? 256 * g : g), a.eff, next ? 256 * a.n_sets : a.n_sets);
        if (next) {
            c.download(cands + 1024 * g, a.cands, 1024 * a.n_sets);
            c.download(n_cands + g, a.n_cands, a.n_sets);
        }
        if ((rc = c.sync())) return rc;
    }
    return c.finish();
}

}  // namespace
}  // namespace pg

using namespace pg;

extern "C" {

// ---- synthesis/fragment (fragment.cu) -------------------------------------------------------------------
int pg_fragment_batch(const uint8_t *seqs, const uint64_t *offsets, uint64_t n, int64_t min_size, int64_t max_size, const uint8_t *exclude,
                      const uint64_t *exclude_offsets, uint64_t n_exclude, const uint8_t *include, const uint64_t *include_offsets,
                      uint64_t n_include, int32_t *status, double *efficiency, int64_t *err_min, int64_t *err_max, uint64_t *frag_offsets,
                      uint64_t *ends, uint64_t ends_cap, uint64_t *n_ends) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if (!n_ends || !frag_offsets) { set_error("null n_ends or frag_offsets"); return PG_ERR_ARG; }
    *n_ends = 0;
    frag_offsets[0] = 0;
    if (n == 0) return PG_OK;
    if (!offsets || !efficiency || !err_min || !err_max || (ends_cap && !ends) || (n_exclude && !exclude_offsets) || (n_include && !include_offsets)) {
        set_error("null buffer");
        return PG_ERR_ARG;
    }
    uint64_t max_len, widest;  // the whole batch and both lists are checked before the first group is launched
    if ((rc = check_ragged(offsets, n, &max_len)) || (n_exclude && (rc = check_ragged(exclude_offsets, n_exclude, &widest))) ||
        (n_include && (rc = check_ragged(include_offsets, n_include, &widest))))
        return rc;
    if ((offsets[n] > offsets[0] && !seqs) || (n_exclude && exclude_offsets[n_exclude] > exclude_offsets[0] && !exclude) ||
        (n_include && include_offsets[n_include] > include_offsets[0] && !include)) {
        set_error("null seqs, exclude or include with non-empty entries");
        return PG_ERR_ARG;
    }
    const FragmentHost h = fragment_host(exclude, exclude_offsets, n_exclude, include, include_offsets, n_include);
    // Items go to the device in groups whose input and worst-case ends region stay within the budget; a single
    // item over it is a group of its own.  The per-warp scratch gets another budget's worth at most.
    const uint64_t budget = group_budget(4ull << 30);
    auto item_bytes = [&](uint64_t i) { return (offsets[i + 1] - offsets[i]) + 8 * fragment_max_ends(offsets[i + 1] - offsets[i]) + 64; };
    std::vector<int32_t> hst(n);
    std::vector<uint64_t> region_off, cnt, out_off;
    uint64_t total = 0;
    for (uint64_t g = 0; g < n;) {
        const uint64_t e = group_end(g, n, budget, item_bytes), m = e - g;
        uint64_t group_max = 0;
        region_off.assign(1, 0);
        for (uint64_t i = g; i < e; ++i) {
            group_max = std::max(group_max, offsets[i + 1] - offsets[i]);
            region_off.push_back(region_off.back() + fragment_max_ends(offsets[i + 1] - offsets[i]));
        }
        HostCall c;
        const Ragged<uint8_t> in = c.ragged(seqs, offsets + g, m);
        FragmentArgs a{};
        a.seqs = in.base;
        a.off = in.off;
        a.n = m;
        a.min_size = min_size;
        a.max_size = max_size;
        a.fid = c.upload(h.fid.data(), h.fid.size());
        a.r_ex = c.upload(h.r_ex.data(), h.r_ex.size());
        a.ex_mask = c.upload(h.ex_mask.data(), 8);
        a.inc_mask = c.upload(h.inc_mask.data(), 8);
        a.ex_keys = c.upload(h.ex_keys.data(), h.ex_keys.size());
        a.n_ex_keys = h.ex_keys.size();
        a.ex_other = c.upload(h.ex_other.data(), h.ex_other.size());
        a.n_ex_other = h.ex_other.size();
        a.inc_other = c.upload(h.inc_other.data(), h.inc_other.size());
        a.n_inc_other = h.inc_other.size();
        a.has_include = n_include > 0;
        a.status = c.alloc<int32_t>(m);
        a.eff = c.alloc<double>(m);
        a.err_min = c.alloc<int64_t>(m);
        a.err_max = c.alloc<int64_t>(m);
        a.n_ends = c.alloc<uint64_t>(m);
        a.ends = c.alloc<uint64_t>(region_off.back());
        a.ends_off = c.upload(region_off.data(), m + 1);
        StreamScratch work(c.st);
        if ((rc = c.error()) || (rc = launch_fragment(a, group_max, budget, work, c.st))) return rc;
        cnt.resize(m);
        c.download(hst.data() + g, a.status, m);
        c.download(efficiency + g, a.eff, m);
        c.download(err_min + g, a.err_min, m);
        c.download(err_max + g, a.err_max, m);
        c.download(cnt.data(), a.n_ends, m);
        if ((rc = c.sync())) return rc;
        out_off.assign(1, 0);
        for (uint64_t i = 0; i < m; ++i) {
            out_off.push_back(out_off.back() + cnt[i]);
            frag_offsets[g + i + 1] = total + out_off.back();
        }
        if (total + out_off.back() <= ends_cap && out_off.back()) {
            const uint64_t *d_out_off = c.upload(out_off.data(), m + 1);
            uint64_t *d_out = c.alloc<uint64_t>(out_off.back());
            if ((rc = c.error()) || (rc = launch_fragment_compact(a.ends, a.ends_off, a.n_ends, d_out_off, m, d_out, c.st))) return rc;
            c.download(ends + total, d_out, out_off.back());
        }
        if ((rc = c.finish())) return rc;
        total += out_off.back();
        g = e;
    }
    *n_ends = total;
    if (total > ends_cap) {
        fold_item_status(hst, status, "", "");
        set_error("the batch has %llu fragment ends: ends_cap %llu", (unsigned long long)total, (unsigned long long)ends_cap);
        return PG_ERR_ARG;
    }
    return fold_item_status(hst, status, "at least one sequence is shorter than 4 bytes: fragment.Fragment panics (slice bounds out of range)",
                            "at least one sequence holds a byte >= 0x80 (unsupported)");
}

int pg_fragment_set_efficiency_batch(const uint8_t *overhangs, const uint64_t *overhang_offsets, const uint64_t *set_offsets, uint64_t n_sets,
                                     double *efficiency) {
    return overhang_sets(overhangs, overhang_offsets, set_offsets, n_sets, 0, nullptr, nullptr, efficiency);
}

int pg_fragment_next_overhangs_batch(const uint8_t *overhangs, const uint64_t *overhang_offsets, const uint64_t *set_offsets, uint64_t n_sets,
                                     uint8_t *cands, uint32_t *n_cands, double *efficiency) {
    return overhang_sets(overhangs, overhang_offsets, set_offsets, n_sets, 1, cands, n_cands, efficiency);
}

}  // extern "C"
