// index_tests.cpp -- the sketch index through the C++ host mirror (poly::mash::Index).
// Usage: index_tests REFS.pgsketch QUERIES.pgsketch K MIN_SAME
// Prints one line per query, "q n_hits ref:same:distance_bits ...", with the distance's IEEE-754 bits in hex,
// then "ok: index tests pass" after its own checks.
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "poly_b200.hpp"

using namespace poly;

static int fail(const char *what) {
    std::printf("FAIL: %s\n", what);
    return 1;
}

int main(int argc, char **argv) {
    if (argc != 5) return fail("usage: index_tests REFS QUERIES K MIN_SAME");
    const auto refs = mash::MashesOf(mash::LoadSketchSet(argv[1]));
    const auto queries = mash::MashesOf(mash::LoadSketchSet(argv[2]));
    const uint32_t k = (uint32_t)std::strtoul(argv[3], nullptr, 10), minSame = (uint32_t)std::strtoul(argv[4], nullptr, 10);
    mash::Index ix(refs);
    const auto res = ix.Nearest(queries, k, minSame);
    for (size_t q = 0; q < res.size(); ++q) {
        std::printf("%zu %zu", q, res[q].size());
        for (auto &nb : res[q]) {
            uint64_t bits;
            std::memcpy(&bits, &nb.Distance, 8);
            std::printf(" %u:%u:%016llx", nb.Ref, nb.Same, (unsigned long long)bits);
        }
        std::printf("\n");
    }
    // each listed neighbour is what the single-pair Distance returns
    for (size_t q = 0; q < res.size(); q += 37)
        for (auto &nb : res[q])
            if (queries[q].Distance(refs[nb.Ref]) != nb.Distance) return fail("Nearest distance != Mash::Distance");
    // the top_k cap and empty sketches fail as documented
    try {
        ix.Nearest(queries, PG_INDEX_MAX_TOP_K + 1);
        return fail("top_k above the cap accepted");
    } catch (const Error &e) {
        if (e.code != PG_ERR_ARG) return fail("top_k above the cap: wrong code");
    }
    try {
        mash::Index bad({mash::New(21, 0)});
        return fail("size-0 reference accepted");
    } catch (const GoPanic &) {
    }
    std::printf("ok: index tests pass\n");
    return 0;
}
