// derep_tests.cpp -- greedy representatives through the C++ host mirror (poly::mash::Dereplicate).
// Usage: derep_tests SET.pgsketch MIN_SAME first|nearest
// Prints "n_reps", then the assignments on one line, then "ok: derep tests pass" after its own checks.
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
    if (argc != 4 || (std::strcmp(argv[3], "first") && std::strcmp(argv[3], "nearest"))) return fail("usage: derep_tests SET MIN_SAME first|nearest");
    const auto set = mash::MashesOf(mash::LoadSketchSet(argv[1]));
    const uint32_t minSame = (uint32_t)std::strtoul(argv[2], nullptr, 10);
    const bool nearest = !std::strcmp(argv[3], "nearest");
    const auto res = mash::Dereplicate(set, minSame, nearest);
    std::printf("%llu\n", (unsigned long long)res.NReps);
    for (size_t i = 0; i < res.Rep.size(); ++i) std::printf(i ? " %u" : "%u", res.Rep[i]);
    std::printf("\n");
    // a representative is never above the sketch it represents, and represents itself
    uint64_t reps = 0;
    for (size_t i = 0; i < res.Rep.size(); ++i) {
        if (res.Rep[i] > i || res.Rep[res.Rep[i]] != res.Rep[i]) return fail("an assignment is not an earlier representative");
        reps += res.Rep[i] == i;
    }
    if (reps != res.NReps) return fail("NReps != number of representatives");
    // both modes keep the same representatives
    const auto other = mash::Dereplicate(set, minSame, !nearest);
    for (size_t i = 0; i < res.Rep.size(); ++i)
        if ((res.Rep[i] == i) != (other.Rep[i] == i)) return fail("the modes keep different representatives");
    // an empty set is valid; thresholds outside [1, s] and empty sketches fail as documented
    if (mash::Dereplicate({}, 1, nearest).NReps != 0) return fail("empty set");
    const int s = set.empty() ? 0 : set[0].SketchSize;
    for (uint32_t bad : {0u, (uint32_t)s + 1}) {
        try {
            mash::Dereplicate(set, bad, nearest);
            return fail("min_same outside [1, s] accepted");
        } catch (const Error &e) {
            if (e.code != PG_ERR_ARG) return fail("min_same outside [1, s]: wrong code");
        }
    }
    try {
        mash::Dereplicate({mash::New(21, 0)}, 1, nearest);
        return fail("size-0 sketch accepted");
    } catch (const GoPanic &) {
    }
    std::printf("ok: derep tests pass\n");
    return 0;
}
