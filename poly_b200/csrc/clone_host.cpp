// clone_host.cpp -- recurseLigate / CircularLigate (clone/clone.go:270-338) as a host enumeration over
// fragment ids, without hashing (DESIGN.md "Clone").
//
// Both seqhash branches of recurseLigate return at once whether or not the hash was new, so hashing never
// steers the recursion: it only decides which constructs reach the output.  The enumeration therefore
// records every construct the reference would hash (an emit) with its recipe, and the caller hashes them
// on the device and keeps, per reaction, the first emit of each seqhash that is also kept.
#include "clone.cuh"

namespace pg {

namespace {

std::string reverse_complement(const std::string &s) {
    std::string r(s.size(), '\0');
    for (size_t i = 0; i < s.size(); ++i) r[i] = (char)complement((uint8_t)s[s.size() - 1 - i]);
    return r;
}

struct Enumeration {
    const std::vector<LigFragment> &f;
    std::vector<std::string> fwd_rc, rev_rc;  // transform.ReverseComplement of each fragment's overhangs
    uint64_t bytes_cap, emits_cap;
    LigationPlan &plan;
    std::vector<Piece> seq;  // the seed's Sequence as pieces (dst unused until an emit)
    uint64_t seq_len = 0;

    void emit(uint8_t kind, std::initializer_list<Piece> head, bool with_seq) {
        uint64_t bytes = 0;
        for (const Piece &p : head) bytes += p.len;
        if (with_seq) bytes += seq_len;
        plan.bytes += bytes;
        plan.n_emits += 1;
        if (plan.over || plan.bytes > bytes_cap || plan.n_emits > emits_cap) {
            plan.over = true;
            return;
        }
        Emit e{plan.pieces.size(), 0, bytes, kind, 1};
        uint64_t dst = 0;
        auto add = [&](Piece p) {
            if (p.len == 0) return;
            p.dst = dst;
            dst += p.len;
            plan.pieces.push_back(p);
        };
        for (const Piece &p : head) add(p);
        if (with_seq)
            for (const Piece &p : seq) add(p);
        e.piece_end = plan.pieces.size();
        plan.emits.push_back(e);
    }

    // seed: its ForwardOverhang is that of the first fragment `first`; its ReverseOverhang the string
    // `rev` whose bytes are at (rev_src, rev_rc); its Sequence the pieces in `seq`.
    void recurse(uint64_t first, const std::string &rev, Piece rev_piece, const std::vector<uint64_t> &used_in) {
        const LigFragment &f0 = f[first];
        if (f0.fwd == rev) {  // construct = seed.ForwardOverhang + seed.Sequence
            emit(0, {Piece{f0.fwd_src, 0, (uint32_t)f0.fwd.size(), 0}}, true);
            return;
        }
        std::vector<uint64_t> used = used_in;  // usedFragments: grows across this call's iterations
        const uint64_t start = plan.emits.size();
        const bool rev_palindromic = rev == reverse_complement(rev);
        for (uint64_t k = 0; k < f.size(); ++k) {
            const LigFragment &nf = f[k];
            int attached = 0;  // 1 forwards, 2 reverse-complemented: the second test overrides the first
            if (rev == nf.fwd) attached = 1;
            if (rev == rev_rc[k] && !rev_palindromic) attached = 2;
            if (!attached) continue;
            for (uint64_t u : used) {
                if (f[u].seq_id != nf.seq_id) continue;
                // return nil, ...: the constructs this call collected are dropped (their hashes stay)
                if (!plan.over)
                    for (uint64_t i = start; i < plan.emits.size(); ++i) plan.emits[i].kept = 0;
                const LigFragment &uf = f[u];
                std::vector<Piece> saved;
                saved.swap(seq);
                const uint64_t saved_len = seq_len;
                seq_len = 0;
                emit(1, {Piece{uf.fwd_src, 0, (uint32_t)uf.fwd.size(), 0}, Piece{uf.seq_src, 0, uf.seq_len, 0},
                         Piece{uf.rev_src, 0, (uint32_t)uf.rev.size(), 0}},
                     false);
                seq.swap(saved);
                seq_len = saved_len;
                return;
            }
            used.push_back(k);
            // newSeed.Sequence = seed.Sequence + seed.ReverseOverhang + (newFragment.Sequence or its reverse complement)
            seq.push_back(rev_piece);
            seq.push_back(Piece{nf.seq_src, 0, nf.seq_len, attached == 2 ? 1u : 0u});
            seq_len += rev_piece.len + nf.seq_len;
            if (attached == 1)
                recurse(first, nf.rev, Piece{nf.rev_src, 0, (uint32_t)nf.rev.size(), 0}, used);
            else
                recurse(first, fwd_rc[k], Piece{nf.fwd_src, 0, (uint32_t)nf.fwd.size(), 1}, used);
            seq.pop_back();
            seq.pop_back();
            seq_len -= rev_piece.len + nf.seq_len;
        }
    }
};

}  // namespace

void enumerate_ligation(const std::vector<LigFragment> &frags, uint64_t bytes_cap, uint64_t emits_cap, LigationPlan &plan) {
    Enumeration g{frags, {}, {}, bytes_cap, emits_cap, plan, {}, 0};
    for (const LigFragment &x : frags) {
        g.fwd_rc.push_back(reverse_complement(x.fwd));
        g.rev_rc.push_back(reverse_complement(x.rev));
    }
    for (uint64_t i = 0; i < frags.size(); ++i) {
        g.seq.assign(1, Piece{frags[i].seq_src, 0, frags[i].seq_len, 0});
        g.seq_len = frags[i].seq_len;
        g.recurse(i, frags[i].rev, Piece{frags[i].rev_src, 0, (uint32_t)frags[i].rev.size(), 0}, {});
    }
}

}  // namespace pg
