// api_clone.cu -- the C ABI of poly's clone: CutWithEnzyme, GoldenGate and CircularLigate.
#include <algorithm>
#include <cstring>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "clone.cuh"
#include "runtime.cuh"

namespace pg {
namespace {

// pg_clone_enzyme -> the kernels' form.  A site that is empty, longer than CLONE_MAX_SITE or holds a byte
// outside 0x01..0x7f is not a literal this library matches: PG_ERR_UNSUPPORTED.
int clone_enzyme(const pg_clone_enzyme &in, CloneEnzyme *out) {
    if (!in.forward_site || !in.reverse_site || (in.recognition_len && !in.recognition_site)) { set_error("null enzyme site"); return PG_ERR_ARG; }
    CloneEnzyme e{};
    for (int which = 0; which < 2; ++which) {
        const uint8_t *site = which ? in.reverse_site : in.forward_site;
        const uint32_t len = which ? in.reverse_len : in.forward_len;
        if (len == 0 || len > CLONE_MAX_SITE) { set_error("enzyme site of %u bytes: only literal sites of 1..%u bytes are supported", len, CLONE_MAX_SITE); return PG_ERR_UNSUPPORTED; }
        for (uint32_t j = 0; j < len; ++j) {
            if (site[j] == 0 || site[j] >= 0x80) { set_error("enzyme site byte 0x%02x is not supported", site[j]); return PG_ERR_UNSUPPORTED; }
            (which ? e.rsite : e.fsite)[j] = site[j];
        }
        (which ? e.rl : e.fl) = len;
    }
    e.recl = in.recognition_len;
    e.palindromic = 1;  // checks.IsPalindromic: RecognitionSite == transform.ReverseComplement(RecognitionSite)
    for (uint32_t j = 0; j < in.recognition_len; ++j)
        if (in.recognition_site[j] != complement(in.recognition_site[in.recognition_len - 1 - j])) e.palindromic = 0;
    e.skip = in.skip;
    e.ohl = in.overhang_length;
    *out = e;
    return PG_OK;
}

// The fragments of every reaction, on the host (for the enumeration) and in one device source buffer: the
// Sequence bytes at [0, seq_total), the overhang bytes after them.
struct LigationInput {
    const uint8_t *d_src;
    const uint8_t *seq, *oh;
    const uint64_t *seq_off, *oh_off;  // as pg_clone_digest_batch's outputs, from 0
    uint64_t seq_total;
    std::vector<uint64_t> reaction_frags;  // reaction r = fragments [reaction_frags[r], reaction_frags[r+1])
    std::vector<int32_t> status;           // per reaction: PG_ITEM_OK, or why it is not ligated
};

struct LigationOutput {
    uint64_t bytes_cap, constructs_cap;
    uint8_t *out, *kinds, *digests;
    uint64_t *construct_offsets, *counts, *need_bytes, *need_constructs;
    int32_t *status;
};

// Enumerate every reaction on the host, materialise and seqhash its emits on the device in groups under a
// memory budget, keep the first emit of each seqhash per reaction, and copy back the kept survivors.
int ligate_reactions(HostCall &c, const LigationInput &in, const LigationOutput &o) {
    const uint64_t R = in.reaction_frags.size() - 1;
    LigationPlan plan;
    std::vector<uint64_t> reaction_emits(R + 1, 0);
    std::unordered_map<std::string, uint64_t> interned;
    for (uint64_t r = 0; r < R; ++r) {
        reaction_emits[r] = plan.emits.size();
        if (in.status[r] != PG_ITEM_OK) continue;
        std::vector<LigFragment> frags;
        for (uint64_t f = in.reaction_frags[r]; f < in.reaction_frags[r + 1]; ++f) {
            const uint64_t s0 = in.seq_off[f], s1 = in.seq_off[f + 1], o0 = in.oh_off[2 * f], o1 = in.oh_off[2 * f + 1], o2 = in.oh_off[2 * f + 2];
            if (s1 - s0 > UINT32_MAX || o2 - o0 > UINT32_MAX) { set_error("fragment %llu is longer than 4 GiB", (unsigned long long)f); return PG_ERR_ARG; }
            const uint64_t id = interned.emplace(std::string((const char *)in.seq + s0, s1 - s0), interned.size()).first->second;
            frags.push_back(LigFragment{id, std::string((const char *)in.oh + o0, o1 - o0), std::string((const char *)in.oh + o1, o2 - o1), s0,
                                        in.seq_total + o0, in.seq_total + o1, (uint32_t)(s1 - s0)});
        }
        enumerate_ligation(frags, o.bytes_cap, o.constructs_cap, plan);
    }
    reaction_emits[R] = plan.emits.size();
    *o.need_bytes = plan.bytes;
    *o.need_constructs = plan.n_emits;
    if (plan.over) {
        set_error("the ligations emit %llu constructs of %llu bytes in all: constructs_cap %llu, bytes_cap %llu", (unsigned long long)plan.n_emits,
                  (unsigned long long)plan.bytes, (unsigned long long)o.constructs_cap, (unsigned long long)o.bytes_cap);
        return PG_ERR_ARG;
    }
    for (uint64_t r = 0; r < 2 * R; ++r) o.counts[r] = 0;
    o.construct_offsets[0] = 0;
    const uint64_t budget = group_budget(1ull << 30), n_emits = plan.emits.size();
    std::unordered_set<std::string> seen;  // existingSeqhashes of the current reaction
    uint64_t r = 0, n_out = 0, out_bytes = 0;
    for (uint64_t g = 0; g < n_emits;) {
        const uint64_t e = group_end(g, n_emits, budget, [&](uint64_t k) { return plan.emits[k].bytes; });
        // group layout: closed clones first, then looping constructs, so that each kind is one ragged batch
        std::vector<uint64_t> at(e - g), off_c{0}, off_l;
        uint64_t max_c = 0, max_l = 0;
        for (uint64_t k = g; k < e; ++k)
            if (plan.emits[k].kind == 0) {
                at[k - g] = off_c.back();
                off_c.push_back(off_c.back() + plan.emits[k].bytes);
                max_c = std::max(max_c, plan.emits[k].bytes);
            }
        off_l.push_back(off_c.back());
        for (uint64_t k = g; k < e; ++k)
            if (plan.emits[k].kind == 1) {
                at[k - g] = off_l.back();
                off_l.push_back(off_l.back() + plan.emits[k].bytes);
                max_l = std::max(max_l, plan.emits[k].bytes);
            }
        std::vector<Piece> pieces(plan.pieces.begin() + plan.emits[g].piece_begin, plan.pieces.begin() + plan.emits[e - 1].piece_end);
        for (uint64_t k = g; k < e; ++k)
            for (uint64_t i = plan.emits[k].piece_begin; i < plan.emits[k].piece_end; ++i) pieces[i - plan.emits[g].piece_begin].dst += at[k - g];
        const uint64_t nc = off_c.size() - 1, nl = off_l.size() - 1, n = e - g;
        StreamScratch gs(c.st);
        uint8_t *d_buf = nullptr, *d_dig = nullptr;
        Piece *d_pieces = nullptr;
        uint64_t *d_offc = nullptr, *d_offl = nullptr, *d_pos = nullptr;
        int32_t *d_err = nullptr;
        int rc;
        if ((rc = scratch_alloc(gs, &d_buf, off_l.back())) || (rc = scratch_alloc(gs, &d_pieces, pieces.size())) || (rc = scratch_alloc(gs, &d_offc, nc + 1)) ||
            (rc = scratch_alloc(gs, &d_offl, nl + 1)) || (rc = scratch_alloc(gs, &d_dig, 32 * n)) || (rc = scratch_alloc(gs, &d_err, n)) ||
            (rc = scratch_alloc(gs, &d_pos, n)))
            return rc;
        c.put(d_pieces, pieces.data(), pieces.size());
        c.put(d_offc, off_c.data(), nc + 1);
        c.put(d_offl, off_l.data(), nl + 1);
        if ((rc = c.error()) || (rc = launch_clone_pieces(in.d_src, d_pieces, pieces.size(), d_buf, c.st))) return rc;
        // seqhash.Hash(construct, "DNA", true, true) for clones (clone.go:275), (.., false, true) for loops (:305)
        if (nc && (rc = launch_seqhash(d_buf, d_offc, nc, max_c, off_c[nc], PG_SEQHASH_DNA, PG_SEQHASH_CIRCULAR | PG_SEQHASH_DOUBLE_STRANDED, d_dig,
                                       d_err, d_pos, c.st)))
            return rc;
        if (nl && (rc = launch_seqhash(d_buf, d_offl, nl, max_l, off_l[nl] - off_l[0], PG_SEQHASH_DNA, PG_SEQHASH_DOUBLE_STRANDED, d_dig + 32 * nc,
                                       d_err + nc, d_pos + nc, c.st)))
            return rc;
        std::vector<uint8_t> dig(32 * n);
        std::vector<int32_t> err(n);
        c.download(dig.data(), d_dig, 32 * n);
        c.download(err.data(), d_err, n);
        if ((rc = c.sync())) return rc;
        // dedup in emit order; the survivors are compacted on the device and come back in one copy
        std::vector<Piece> keep;
        uint64_t kept_bytes = 0, ic = 0, il = 0;
        for (uint64_t k = g; k < e; ++k) {
            while (k >= reaction_emits[r + 1]) {
                ++r;
                seen.clear();
            }
            const Emit &em = plan.emits[k];
            const uint64_t slot = em.kind == 0 ? ic++ : nc + il++;
            std::string key = err[slot] ? std::string() : std::string(1, (char)(em.kind + 1)) + std::string((const char *)&dig[32 * slot], 32);
            if (!seen.insert(std::move(key)).second || !em.kept) continue;
            keep.push_back(Piece{at[k - g], kept_bytes, (uint32_t)em.bytes, 0});
            kept_bytes += em.bytes;
            o.counts[2 * r + em.kind] += 1;
            if (o.kinds) o.kinds[n_out] = em.kind;
            if (o.digests) memcpy(o.digests + 32 * n_out, &dig[32 * slot], 32);
            o.construct_offsets[n_out + 1] = o.construct_offsets[n_out] + em.bytes;
            ++n_out;
        }
        if (!keep.empty()) {
            uint8_t *d_keep = nullptr;
            Piece *d_kp = nullptr;
            if ((rc = scratch_alloc(gs, &d_keep, kept_bytes)) || (rc = scratch_alloc(gs, &d_kp, keep.size()))) return rc;
            c.put(d_kp, keep.data(), keep.size());
            if ((rc = c.error()) || (rc = launch_clone_pieces(d_buf, d_kp, keep.size(), d_keep, c.st))) return rc;
            c.download(o.out + out_bytes, d_keep, kept_bytes);
            if ((rc = c.sync())) return rc;
        }
        out_bytes += kept_bytes;
        g = e;
    }
    return PG_OK;
}

// reaction statuses -> `status` and the call's code, as fold_item_status
int ligation_status(const std::vector<int32_t> &st, int32_t *status) {
    return fold_item_status(st, status, "at least one reaction cuts a part where clone.CutWithEnzyme panics (slice bounds out of range)",
                            "at least one reaction has a part with a byte >= 0x80 (unsupported)");
}

// Before anything is uploaded: the item count fits in 64 bits, and no item can hold 2^32 matches of a site
// (the walks count them in 32 bits; a part read doubled has at most 2 L / site length of them).
int clone_batch_check(const uint64_t *part_offsets, uint64_t n_parts, const std::vector<CloneEnzyme> &enz) {
    if (n_parts > UINT64_MAX / enz.size()) { set_error("n_parts x n_enzymes overflows"); return PG_ERR_ARG; }
    uint64_t max_len;
    int rc = check_ragged(part_offsets, n_parts, &max_len);
    if (rc != PG_OK) return rc;
    for (const CloneEnzyme &e : enz) {
        const uint64_t site = e.palindromic ? e.fl : std::min(e.fl, e.rl);
        if (max_len > UINT64_MAX / 2 || 2 * max_len / site > UINT32_MAX) {
            set_error("a part of %llu bytes could hold 2^32 or more matches of a %u-byte site", (unsigned long long)max_len, site);
            return PG_ERR_ARG;
        }
    }
    return PG_OK;
}

bool ligation_output_ok(const LigationOutput &o) {
    if (!o.construct_offsets || !o.counts || !o.need_bytes || !o.need_constructs || (o.bytes_cap && !o.out)) {
        set_error("null buffer");
        return false;
    }
    return true;
}
}  // namespace
}  // namespace pg

using namespace pg;

extern "C" {

int pg_clone_digest_batch(const uint8_t *parts, const uint64_t *part_offsets, const uint8_t *circular, uint64_t n_parts,
                          const pg_clone_enzyme *enzymes, uint32_t n_enzymes, int32_t directional, uint32_t *frag_count, int32_t *status,
                          uint8_t *seq_bytes, uint64_t seq_cap, uint64_t *seq_offsets, uint8_t *oh_bytes, uint64_t oh_cap,
                          uint64_t *oh_offsets, uint64_t frag_cap, uint64_t *n_frags, uint64_t *n_seq_bytes, uint64_t *n_oh_bytes) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if (!n_frags || !n_seq_bytes || !n_oh_bytes) { set_error("null buffer"); return PG_ERR_ARG; }
    *n_frags = *n_seq_bytes = *n_oh_bytes = 0;
    if (n_parts == 0 || n_enzymes == 0) return PG_OK;
    if (!part_offsets || !circular || !enzymes || !frag_count || !seq_offsets || !oh_offsets || (seq_cap && !seq_bytes) || (oh_cap && !oh_bytes)) {
        set_error("null buffer");
        return PG_ERR_ARG;
    }
    std::vector<CloneEnzyme> enz(n_enzymes);
    for (uint32_t k = 0; k < n_enzymes; ++k)
        if ((rc = clone_enzyme(enzymes[k], &enz[k])) != PG_OK) return rc;
    if ((rc = clone_batch_check(part_offsets, n_parts, enz)) != PG_OK) return rc;
    const uint64_t n_items = n_parts * n_enzymes;
    HostCall c;
    const Ragged<uint8_t> in = c.ragged(parts, part_offsets, n_parts);
    const uint8_t *d_circ = c.upload(circular, n_parts);
    const CloneEnzyme *d_enz = c.upload(enz.data(), n_enzymes);
    if ((rc = c.error())) return rc;
    StreamScratch work(c.st);
    DigestPlan d;
    if ((rc = clone_digest_plan(in.base, in.off, d_circ, n_parts, d_enz, n_enzymes, directional != 0, work, c.st, &d))) return rc;
    std::vector<int32_t> hst(n_items);
    std::vector<uint64_t> cnt(n_items);
    c.download(hst.data(), d.status, n_items);
    c.download(cnt.data(), d.n_frag, n_items);
    if ((rc = c.sync())) return rc;
    for (uint64_t i = 0; i < n_items; ++i) frag_count[i] = (uint32_t)cnt[i];
    *n_frags = d.frags;
    *n_seq_bytes = d.seq_total;
    *n_oh_bytes = d.oh_total;
    if (d.frags > frag_cap || d.seq_total > seq_cap || d.oh_total > oh_cap) {
        fold_item_status(hst, status, "", "");
        set_error("the digest gives %llu fragments, %llu sequence bytes and %llu overhang bytes: frag_cap %llu, seq_cap %llu, oh_cap %llu",
                  (unsigned long long)d.frags, (unsigned long long)d.seq_total, (unsigned long long)d.oh_total, (unsigned long long)frag_cap,
                  (unsigned long long)seq_cap, (unsigned long long)oh_cap);
        return PG_ERR_ARG;
    }
    uint64_t *d_soff = c.alloc<uint64_t>(d.frags + 1), *d_ooff = c.alloc<uint64_t>(2 * d.frags + 1);
    uint8_t *d_seq = c.alloc<uint8_t>(d.seq_total), *d_oh = c.alloc<uint8_t>(d.oh_total);
    if ((rc = c.error()) || (rc = clone_digest_write(d, d_soff, d_seq, d_ooff, d_oh, work, c.st))) return rc;
    c.download(seq_offsets, d_soff, d.frags + 1);
    c.download(oh_offsets, d_ooff, 2 * d.frags + 1);
    c.download(seq_bytes, d_seq, d.seq_total);
    c.download(oh_bytes, d_oh, d.oh_total);
    if ((rc = c.finish())) return rc;
    return fold_item_status(hst, status, "at least one item panics in clone.CutWithEnzyme (slice bounds out of range)",
                            "at least one part holds a byte >= 0x80 (unsupported)");
}

int pg_clone_golden_gate_batch(const uint8_t *parts, const uint64_t *part_offsets, const uint8_t *circular, uint64_t n_parts,
                               const uint64_t *reaction_offsets, uint64_t n_reactions, const pg_clone_enzyme *enzyme, uint64_t bytes_cap,
                               uint64_t constructs_cap, uint8_t *out, uint64_t *construct_offsets, uint8_t *kinds, uint8_t *digests,
                               uint64_t *counts, int32_t *status, uint64_t *need_bytes, uint64_t *need_constructs) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    const LigationOutput o{bytes_cap, constructs_cap, out, kinds, digests, construct_offsets, counts, need_bytes, need_constructs, status};
    if (!ligation_output_ok(o) || !reaction_offsets || !enzyme || (n_parts && (!part_offsets || !circular))) {
        set_error("null buffer");
        return PG_ERR_ARG;
    }
    *need_bytes = *need_constructs = 0;
    uint64_t widest;
    if ((rc = check_ragged(reaction_offsets, n_reactions, &widest))) return rc;
    if (reaction_offsets[0] != 0 || reaction_offsets[n_reactions] != n_parts) { set_error("reaction_offsets must run from 0 to n_parts"); return PG_ERR_ARG; }
    CloneEnzyme enz;
    if ((rc = clone_enzyme(*enzyme, &enz))) return rc;
    if (n_parts && (rc = clone_batch_check(part_offsets, n_parts, {enz}))) return rc;
    HostCall c;
    LigationInput in;
    in.status.assign(n_reactions, PG_ITEM_OK);
    in.reaction_frags.assign(n_reactions + 1, 0);
    std::vector<uint8_t> seq, oh;
    std::vector<uint64_t> soff{0}, ooff{0};
    StreamScratch work(c.st);
    uint8_t *d_src = nullptr;
    if (n_parts) {
        const Ragged<uint8_t> p = c.ragged(parts, part_offsets, n_parts);
        const uint8_t *d_circ = c.upload(circular, n_parts);
        const CloneEnzyme *d_enz = c.upload(&enz, 1);
        DigestPlan d;
        if ((rc = c.error()) || (rc = clone_digest_plan(p.base, p.off, d_circ, n_parts, d_enz, 1, 1, work, c.st, &d))) return rc;
        // the fragments stay on the device as the ligation's source: Sequence bytes, then overhang bytes
        uint64_t *d_soff = c.alloc<uint64_t>(d.frags + 1), *d_ooff = c.alloc<uint64_t>(2 * d.frags + 1);
        d_src = c.alloc<uint8_t>(d.seq_total + d.oh_total);
        if ((rc = c.error()) || (rc = clone_digest_write(d, d_soff, d_src, d_ooff, d_src + d.seq_total, work, c.st))) return rc;
        std::vector<int32_t> pst(n_parts);
        std::vector<uint64_t> cnt(n_parts);
        seq.resize(d.seq_total);
        oh.resize(d.oh_total);
        soff.resize(d.frags + 1);
        ooff.resize(2 * d.frags + 1);
        c.download(pst.data(), d.status, n_parts);
        c.download(cnt.data(), d.n_frag, n_parts);
        c.download(soff.data(), d_soff, d.frags + 1);
        c.download(ooff.data(), d_ooff, 2 * d.frags + 1);
        c.download(seq.data(), d_src, d.seq_total);
        c.download(oh.data(), d_src + d.seq_total, d.oh_total);
        if ((rc = c.sync())) return rc;
        for (uint64_t r = 0; r < n_reactions; ++r) {
            uint64_t nf = 0;
            for (uint64_t q = reaction_offsets[r]; q < reaction_offsets[r + 1]; ++q) {
                nf += cnt[q];
                if (pst[q] != PG_ITEM_OK && in.status[r] == PG_ITEM_OK) in.status[r] = pst[q];  // GoldenGate stops at the first
            }
            in.reaction_frags[r + 1] = in.reaction_frags[r] + nf;
        }
        in.seq_total = d.seq_total;
    } else {
        in.seq_total = 0;
    }
    in.d_src = d_src;
    in.seq = seq.data();
    in.oh = oh.data();
    in.seq_off = soff.data();
    in.oh_off = ooff.data();
    if ((rc = ligate_reactions(c, in, o))) return rc;
    if ((rc = c.finish())) return rc;
    return ligation_status(in.status, status);
}

int pg_clone_circular_ligate_batch(const uint8_t *seq_bytes, const uint64_t *seq_offsets, const uint8_t *oh_bytes, const uint64_t *oh_offsets,
                                   uint64_t n_frags, const uint64_t *reaction_offsets, uint64_t n_reactions, uint64_t bytes_cap,
                                   uint64_t constructs_cap, uint8_t *out, uint64_t *construct_offsets, uint8_t *kinds, uint8_t *digests,
                                   uint64_t *counts, uint64_t *need_bytes, uint64_t *need_constructs) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    const LigationOutput o{bytes_cap, constructs_cap, out, kinds, digests, construct_offsets, counts, need_bytes, need_constructs, nullptr};
    if (!ligation_output_ok(o) || !reaction_offsets || !seq_offsets || !oh_offsets) { set_error("null buffer"); return PG_ERR_ARG; }
    *need_bytes = *need_constructs = 0;
    uint64_t widest;
    if ((rc = check_ragged(reaction_offsets, n_reactions, &widest)) || (rc = check_ragged(seq_offsets, n_frags, &widest)) ||
        (rc = check_ragged(oh_offsets, 2 * n_frags, &widest)))
        return rc;
    if (reaction_offsets[0] != 0 || reaction_offsets[n_reactions] != n_frags) { set_error("reaction_offsets must run from 0 to n_frags"); return PG_ERR_ARG; }
    // offsets from 0, as the digest writes them
    const uint64_t s0 = seq_offsets[0], o0 = oh_offsets[0], S = seq_offsets[n_frags] - s0, O = oh_offsets[2 * n_frags] - o0;
    std::vector<uint64_t> soff(n_frags + 1), ooff(2 * n_frags + 1);
    for (uint64_t f = 0; f <= n_frags; ++f) soff[f] = seq_offsets[f] - s0;
    for (uint64_t f = 0; f <= 2 * n_frags; ++f) ooff[f] = oh_offsets[f] - o0;
    // seqhash.Hash upper-cases with strings.ToUpper, which maps some non-ASCII letters into the alphabet
    // (U+017F -> S, U+212A -> K): a byte >= 0x80 is not hashed here, so such fragments are refused
    for (uint64_t i = 0; i < S; ++i)
        if (seq_bytes[s0 + i] >= 0x80) { set_error("fragment sequence byte %llu is >= 0x80 (unsupported)", (unsigned long long)(s0 + i)); return PG_ERR_UNSUPPORTED; }
    for (uint64_t i = 0; i < O; ++i)
        if (oh_bytes[o0 + i] >= 0x80) { set_error("overhang byte %llu is >= 0x80 (unsupported)", (unsigned long long)(o0 + i)); return PG_ERR_UNSUPPORTED; }
    HostCall c;
    uint8_t *d_src = c.alloc<uint8_t>(S + O);
    if (d_src) {
        c.put(d_src, seq_bytes + s0, S);
        c.put(d_src + S, oh_bytes + o0, O);
    }
    if ((rc = c.error())) return rc;
    LigationInput in{d_src, seq_bytes + s0, oh_bytes + o0, soff.data(), ooff.data(), S,
                     std::vector<uint64_t>(reaction_offsets, reaction_offsets + n_reactions + 1), std::vector<int32_t>(n_reactions, PG_ITEM_OK)};
    if ((rc = ligate_reactions(c, in, o))) return rc;
    return c.finish();
}

}  // extern "C"
