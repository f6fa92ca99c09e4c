// index_add_tests.cpp -- growing the sketch index through the C++ host mirror (poly::mash::Index::Add).
// Usage: index_add_tests REFS.pgsketch QUERIES.pgsketch MIN_SAME BATCHES
// Builds the index over the first reference, adds the rest in BATCHES batches of unequal size and prints one line
// per query of the grown index's Within, "q n_hits ref:same:distance_bits ...", then "ok: index add tests pass"
// after its own checks against an index built over the whole set.
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "poly_b200.hpp"

using namespace poly;

static int fail(const char *what) {
    std::printf("FAIL: %s\n", what);
    return 1;
}

static bool same_lists(const std::vector<std::vector<mash::Neighbor>> &a, const std::vector<std::vector<mash::Neighbor>> &b) {
    if (a.size() != b.size()) return false;
    for (size_t q = 0; q < a.size(); ++q) {
        if (a[q].size() != b[q].size()) return false;
        for (size_t t = 0; t < a[q].size(); ++t)
            if (a[q][t].Ref != b[q][t].Ref || a[q][t].Same != b[q][t].Same || std::memcmp(&a[q][t].Distance, &b[q][t].Distance, 8) != 0) return false;
    }
    return true;
}

int main(int argc, char **argv) {
    if (argc != 5) return fail("usage: index_add_tests REFS QUERIES MIN_SAME BATCHES");
    const auto refs = mash::MashesOf(mash::LoadSketchSet(argv[1]));
    const auto queries = mash::MashesOf(mash::LoadSketchSet(argv[2]));
    const uint32_t minSame = (uint32_t)std::strtoul(argv[3], nullptr, 10);
    const size_t batches = std::strtoul(argv[4], nullptr, 10);
    if (refs.size() < 2 || batches < 1) return fail("need two references and one batch");
    mash::Index ix({refs[0]});
    // batch b takes a share that grows with b, so the batches differ in size
    size_t at = 1;
    for (size_t b = 1; b <= batches && at < refs.size(); ++b) {
        const size_t end = b == batches ? refs.size() : std::min(refs.size(), at + (refs.size() - 1) * 2 * b / (batches * (batches + 1)) + 1);
        ix.Add(std::vector<mash::Mash>(refs.begin() + at, refs.begin() + end));
        at = end;
    }
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
    // the grown index answers as the index over the whole set
    mash::Index whole(refs);
    if (!same_lists(res, whole.Within(queries, minSame))) return fail("grown Within != whole Within");
    if (!same_lists(ix.Nearest(queries, 10, minSame), whole.Nearest(queries, 10, minSame))) return fail("grown Nearest != whole Nearest");
    // an empty batch changes nothing; another SketchSize and a size-0 batch fail as documented
    ix.Add({});
    if (!same_lists(ix.Within(queries, minSame), res)) return fail("empty Add changed the index");
    try {
        ix.Add({mash::New(21, refs[0].SketchSize + 1)});
        return fail("another SketchSize accepted");
    } catch (const Error &e) {
        if (e.code != PG_ERR_ARG) return fail("another SketchSize: wrong code");
    }
    try {
        ix.Add({mash::New(21, 0)});
        return fail("size-0 batch accepted");
    } catch (const GoPanic &) {
    }
    if (!same_lists(ix.Within(queries, minSame), res)) return fail("a rejected Add changed the index");
    std::printf("ok: index add tests pass\n");
    return 0;
}
