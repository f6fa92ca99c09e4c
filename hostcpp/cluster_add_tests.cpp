// cluster_add_tests.cpp -- a growing clustering through the C++ host mirror (poly::mash::Clusterer).
// Usage: cluster_add_tests SET.pgsketch MIN_SAME BATCHES
// Adds the set in BATCHES near-equal batches.  Prints the final group count and the summed link count, then the
// final labels on one line, then "ok: cluster add tests pass" after its own checks.
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
    if (argc != 4) return fail("usage: cluster_add_tests SET MIN_SAME BATCHES");
    const auto set = mash::MashesOf(mash::LoadSketchSet(argv[1]));
    const uint32_t minSame = (uint32_t)std::strtoul(argv[2], nullptr, 10);
    const size_t batches = std::max<size_t>(1, std::strtoul(argv[3], nullptr, 10));
    if (set.empty()) return fail("empty set");
    const int s = set[0].SketchSize;
    mash::Clusterer c(s, minSame);
    uint64_t links = 0, groups = 0;
    for (size_t b = 0; b < batches; ++b) {
        const size_t lo = set.size() * b / batches, hi = set.size() * (b + 1) / batches;
        const auto res = c.Add(std::vector<mash::Mash>(set.begin() + lo, set.begin() + hi));
        if (res.First != lo || res.Labels.size() != hi - lo) return fail("a batch is not numbered from the sketches before it");
        links += res.Links;
        groups = res.Groups;
        // after every add: the one-shot call over the prefix agrees
        const auto prefix = mash::Cluster(std::vector<mash::Mash>(set.begin(), set.begin() + hi), minSame);
        const auto got = c.Labels(0, hi);
        if (got != prefix.Labels || groups != prefix.Groups || links != prefix.Links) return fail("an add differs from Cluster of the prefix");
        if (std::vector<uint32_t>(got.begin() + lo, got.end()) != res.Labels) return fail("the batch labels are not the prefix's slice");
    }
    const auto all = c.Labels(0, set.size());
    std::printf("%llu %llu\n", (unsigned long long)groups, (unsigned long long)links);
    for (size_t i = 0; i < all.size(); ++i) std::printf(i ? " %u" : "%u", all[i]);
    std::printf("\n");
    // an empty batch changes nothing; another size and sizes <= 0 fail as documented
    const auto empty = c.Add({});
    if (empty.First != set.size() || empty.Groups != groups || empty.Links || empty.Merged) return fail("empty batch");
    try {
        c.Add({mash::New(21, s + 1)});
        return fail("another sketch size accepted");
    } catch (const Error &e) {
        if (e.code != PG_ERR_ARG) return fail("another sketch size: wrong code");
    }
    try {
        mash::Clusterer bad(0, 1);
        return fail("size-0 clusterer accepted");
    } catch (const GoPanic &) {
    }
    for (uint32_t bad : {0u, (uint32_t)s + 1}) {
        try {
            mash::Clusterer x(s, bad);
            return fail("min_same outside [1, s] accepted");
        } catch (const Error &e) {
            if (e.code != PG_ERR_ARG) return fail("min_same outside [1, s]: wrong code");
        }
    }
    try {
        c.Labels(0, set.size() + 1);
        return fail("labels past the sketches added accepted");
    } catch (const Error &e) {
        if (e.code != PG_ERR_ARG) return fail("labels past the end: wrong code");
    }
    if (c.Labels(0, set.size()) != all) return fail("a rejected add changed the labels");
    std::printf("ok: cluster add tests pass\n");
    return 0;
}
