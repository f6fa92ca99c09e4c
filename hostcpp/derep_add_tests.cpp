// derep_add_tests.cpp -- a growing dereplication through the C++ host mirror (poly::mash::Dereplicator).
// Usage: derep_add_tests SET.pgsketch MIN_SAME first|nearest BATCHES
// Adds the set in BATCHES near-equal batches.  Prints the total of the new representatives, then the concatenated
// assignments on one line, then "ok: derep add tests pass" after its own checks.
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
    if (argc != 5 || (std::strcmp(argv[3], "first") && std::strcmp(argv[3], "nearest")))
        return fail("usage: derep_add_tests SET MIN_SAME first|nearest BATCHES");
    const auto set = mash::MashesOf(mash::LoadSketchSet(argv[1]));
    const uint32_t minSame = (uint32_t)std::strtoul(argv[2], nullptr, 10);
    const bool nearest = !std::strcmp(argv[3], "nearest");
    const size_t batches = std::max<size_t>(1, std::strtoul(argv[4], nullptr, 10));
    if (set.empty()) return fail("empty set");
    const int s = set[0].SketchSize;
    mash::Dereplicator d(s, minSame, nearest);
    std::vector<uint32_t> rep;
    uint64_t reps = 0;
    for (size_t b = 0; b < batches; ++b) {
        const size_t lo = set.size() * b / batches, hi = set.size() * (b + 1) / batches;
        const auto res = d.Add(std::vector<mash::Mash>(set.begin() + lo, set.begin() + hi));
        if (res.First != lo || res.Rep.size() != hi - lo) return fail("a batch is not numbered from the sketches before it");
        rep.insert(rep.end(), res.Rep.begin(), res.Rep.end());
        reps += res.NReps;
    }
    std::printf("%llu\n", (unsigned long long)reps);
    for (size_t i = 0; i < rep.size(); ++i) std::printf(i ? " %u" : "%u", rep[i]);
    std::printf("\n");
    // the one-shot call over the whole set agrees, and Reps lists the representatives
    const auto whole = mash::Dereplicate(set, minSame, nearest);
    if (whole.Rep != rep || whole.NReps != reps) return fail("the adds differ from Dereplicate of the whole set");
    std::vector<uint32_t> want;
    for (size_t i = 0; i < rep.size(); ++i)
        if (rep[i] == i) want.push_back((uint32_t)i);
    if (d.Reps() != want) return fail("Reps is not the list of representatives");
    // an empty batch changes nothing; another size and sizes <= 0 fail as documented
    if (d.Add({}).First != set.size()) return fail("empty batch");
    try {
        d.Add({mash::New(21, s + 1)});
        return fail("another sketch size accepted");
    } catch (const Error &e) {
        if (e.code != PG_ERR_ARG) return fail("another sketch size: wrong code");
    }
    try {
        mash::Dereplicator bad(0, 1, nearest);
        return fail("size-0 dereplicator accepted");
    } catch (const GoPanic &) {
    }
    for (uint32_t bad : {0u, (uint32_t)s + 1}) {
        try {
            mash::Dereplicator x(s, bad, nearest);
            return fail("min_same outside [1, s] accepted");
        } catch (const Error &e) {
            if (e.code != PG_ERR_ARG) return fail("min_same outside [1, s]: wrong code");
        }
    }
    if (d.Reps() != want) return fail("a rejected add changed the representatives");
    std::printf("ok: derep add tests pass\n");
    return 0;
}
