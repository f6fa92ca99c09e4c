// cluster_tests.cpp -- single-linkage groups through the C++ host mirror (poly::mash::Cluster).
// Usage: cluster_tests SET.pgsketch MIN_SAME
// Prints "n_groups n_links", then the labels on one line, then "ok: cluster tests pass" after its own checks.
#include <cstdio>
#include <cstdlib>

#include "poly_b200.hpp"

using namespace poly;

static int fail(const char *what) {
    std::printf("FAIL: %s\n", what);
    return 1;
}

int main(int argc, char **argv) {
    if (argc != 3) return fail("usage: cluster_tests SET MIN_SAME");
    const auto set = mash::MashesOf(mash::LoadSketchSet(argv[1]));
    const uint32_t minSame = (uint32_t)std::strtoul(argv[2], nullptr, 10);
    const auto res = mash::Cluster(set, minSame);
    std::printf("%llu %llu\n", (unsigned long long)res.Groups, (unsigned long long)res.Links);
    for (size_t i = 0; i < res.Labels.size(); ++i) std::printf(i ? " %u" : "%u", res.Labels[i]);
    std::printf("\n");
    // a label is the smallest member of its group: never above its own index, and a representative labels itself
    uint64_t reps = 0;
    for (size_t i = 0; i < res.Labels.size(); ++i) {
        if (res.Labels[i] > i || res.Labels[res.Labels[i]] != res.Labels[i]) return fail("a label is not its group's smallest member");
        reps += res.Labels[i] == i;
    }
    if (reps != res.Groups) return fail("Groups != number of representatives");
    // the Distance of a pair with exactly minSame matches maps back to minSame: a cut on a pair's Distance includes it
    const int s = set.empty() ? 0 : set[0].SketchSize;
    if (s > 0 && mash::MinSameForDistance(1 - (double)minSame / s, s) != minSame) return fail("MinSameForDistance does not invert Distance");
    // an empty set is valid; thresholds outside [1, s] and empty sketches fail as documented
    if (mash::Cluster({}, 1).Groups != 0) return fail("empty set");
    for (uint32_t bad : {0u, (uint32_t)s + 1}) {
        try {
            mash::Cluster(set, bad);
            return fail("min_same outside [1, s] accepted");
        } catch (const Error &e) {
            if (e.code != PG_ERR_ARG) return fail("min_same outside [1, s]: wrong code");
        }
    }
    try {
        mash::Cluster({mash::New(21, 0)}, 1);
        return fail("size-0 sketch accepted");
    } catch (const GoPanic &) {
    }
    std::printf("ok: cluster tests pass\n");
    return 0;
}
