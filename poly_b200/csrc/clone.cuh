// clone.cuh -- internal types of the clone digest and ligation (clone.cu, clone_host.cpp, api_clone.cu)
#pragma once
#include <string>
#include <vector>

#include "common.cuh"

namespace pg {

constexpr uint32_t CLONE_MAX_SITE = 32;  // longest literal site: one warp's 32-position window plus its halo

// An enzyme as the digest kernels read it: the two sites as literals, palindromic = the recognition site
// equals its reverse complement (checks.IsPalindromic), computed on the host.
struct CloneEnzyme {
    uint8_t fsite[CLONE_MAX_SITE], rsite[CLONE_MAX_SITE];
    uint32_t fl, rl, recl, palindromic;
    int32_t skip, ohl;
};

// A fragment as spans [x0, x1) of the virtual sequence ToUpper(part) or ToUpper(part + part): Sequence is
// a ++ b (b is empty except across the origin), then ForwardOverhang f and ReverseOverhang r.
struct FragRec {
    int64_t a0, a1, b0, b1, f0, f1, r0, r1;
    uint64_t part;
};

// Device state of one digest between its plan (counts and totals known) and its write.  All buffers belong
// to the StreamScratch passed to clone_digest_plan.
struct DigestPlan {
    uint64_t n_items = 0, frags = 0, seq_total = 0, oh_total = 0;
    const uint8_t *parts = nullptr;
    const uint64_t *off = nullptr;
    uint32_t *n_fwd = nullptr, *n_rev = nullptr;
    int32_t *status = nullptr;
    uint64_t *base = nullptr, *n_frag = nullptr, *seq_bytes = nullptr, *oh_bytes = nullptr;
    uint64_t *f_scan = nullptr, *s_scan = nullptr, *o_scan = nullptr;
    int64_t *starts = nullptr;
    FragRec *rec = nullptr;
};

// Digest of n_parts x n_enz items (item = part * n_enz + enzyme); parts[off[p], off[p+1]) on the device.
// The plan runs the site walks and the fragment kernel and reads back the totals (it synchronises st).
int clone_digest_plan(const uint8_t *d_parts, const uint64_t *d_off, const uint8_t *d_circ, uint64_t n_parts, const CloneEnzyme *d_enz,
                      uint32_t n_enz, int directional, StreamScratch &tmp, cudaStream_t st, DigestPlan *plan);
// Fragments in item order: Sequence f at d_seq[d_seq_off[f], d_seq_off[f+1]), ForwardOverhang at
// d_oh[d_oh_off[2f], d_oh_off[2f+1]), ReverseOverhang at d_oh[d_oh_off[2f+1], d_oh_off[2f+2]).
int clone_digest_write(const DigestPlan &d, uint64_t *d_seq_off, uint8_t *d_seq, uint64_t *d_oh_off, uint8_t *d_oh, StreamScratch &tmp,
                       cudaStream_t st);

// A piece of a construct: src[src, src + len), reverse-complemented when rc, written at dst
struct Piece {
    uint64_t src, dst;
    uint32_t len, rc;
};
int launch_clone_pieces(const uint8_t *d_src, const Piece *d_pieces, uint64_t n_pieces, uint8_t *d_dst, cudaStream_t st);

// ---- clone_host.cpp: recurseLigate without hashing --------------------------------------------------------
// A fragment of one reaction for the enumeration: its interned Sequence (equal ids <=> equal strings), the
// overhang strings, and where its bytes are in the ligation's source buffer.
struct LigFragment {
    uint64_t seq_id;
    std::string fwd, rev;
    uint64_t seq_src, fwd_src, rev_src;
    uint32_t seq_len;
};
// A construct the reference would hash: kind 0 a closed clone (clone.go:274), 1 a looping construct (:304);
// kept = 0 when an early return of an enclosing recurseLigate call drops it from the result.  Its recipe is
// pieces[piece_begin, piece_end) of the plan (dst relative to the construct's start).
struct Emit {
    uint64_t piece_begin, piece_end, bytes;
    uint8_t kind, kept;
};
struct LigationPlan {
    std::vector<Piece> pieces;
    std::vector<Emit> emits;
    uint64_t bytes = 0, n_emits = 0;  // totals, counted on past the caps
    bool over = false;                // a cap was passed: pieces and emits are incomplete
};
// Appends the emits of CircularLigate(frags) (clone.go:326-338), in the reference's hashing order, to plan.
// Recipes are stored while plan.bytes <= bytes_cap and plan.n_emits <= emits_cap; past that only counted.
void enumerate_ligation(const std::vector<LigFragment> &frags, uint64_t bytes_cap, uint64_t emits_cap, LigationPlan &plan);

}  // namespace pg
