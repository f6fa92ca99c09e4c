// within_tests.cpp -- radius queries of the sketch index through the C++ host mirror (poly::mash::Index::Within).
// Usage: within_tests REFS.pgsketch QUERIES.pgsketch MIN_SAME
// Prints one line per query, "q n_hits ref:same:distance_bits ...", with the distance's IEEE-754 bits in hex,
// then "ok: within tests pass" after its own checks.
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
    if (argc != 4) return fail("usage: within_tests REFS QUERIES MIN_SAME");
    const auto refs = mash::MashesOf(mash::LoadSketchSet(argv[1]));
    const auto queries = mash::MashesOf(mash::LoadSketchSet(argv[2]));
    const uint32_t minSame = (uint32_t)std::strtoul(argv[3], nullptr, 10);
    mash::Index ix(refs);
    const auto res = ix.Within(queries, minSame);
    for (size_t q = 0; q < res.size(); ++q) {
        std::printf("%zu %zu", q, res[q].size());
        for (auto &nb : res[q]) {
            uint64_t bits;
            std::memcpy(&bits, &nb.Distance, 8);
            std::printf(" %u:%u:%016llx", nb.Ref, nb.Same, (unsigned long long)bits);
        }
        std::printf("\n");
    }
    // each listed reference is what the single-pair Distance returns, and the lists run in reference order
    for (size_t q = 0; q < res.size(); q += 37)
        for (size_t t = 0; t < res[q].size(); ++t) {
            if (queries[q].Distance(refs[res[q][t].Ref]) != res[q][t].Distance) return fail("Within distance != Mash::Distance");
            if (t && res[q][t - 1].Ref >= res[q][t].Ref) return fail("Within list out of reference order");
        }
    // the first k of a list ranked by (Same desc, Ref asc) are what Nearest returns
    const auto top = ix.Nearest(queries, 10, minSame);
    for (size_t q = 0; q < res.size(); ++q) {
        auto ranked = res[q];
        std::stable_sort(ranked.begin(), ranked.end(), [](const mash::Neighbor &a, const mash::Neighbor &b) { return a.Same > b.Same; });
        if (ranked.size() > 10) ranked.resize(10);
        if (ranked.size() != top[q].size()) return fail("Within and Nearest disagree on a list's length");
        for (size_t t = 0; t < ranked.size(); ++t)
            if (ranked[t].Ref != top[q][t].Ref || ranked[t].Same != top[q][t].Same) return fail("Within and Nearest disagree");
    }
    // min_same 0 and empty query sketches fail as documented
    try {
        ix.Within(queries, 0);
        return fail("min_same 0 accepted");
    } catch (const Error &e) {
        if (e.code != PG_ERR_ARG) return fail("min_same 0: wrong code");
    }
    try {
        ix.Within({mash::New(21, 0)});
        return fail("size-0 query accepted");
    } catch (const GoPanic &) {
    }
    std::printf("ok: within tests pass\n");
    return 0;
}
