// screen_winners_tests.cpp -- Mash Screen's winner-take-all through the C++ host mirror (poly::mash::Screen::Winners).
// Usage: screen_winners_tests REFS.pgsketch READS.txt K BATCHES
// READS.txt holds one read per line.  Screens the reads against the references in BATCHES adds of unequal size and
// prints one line per reference of Winners, "r shared containment_bits multiplicity", then
// "ok: screen winners tests pass" after its own checks: Winners leaves Results as they were, no reference wins more
// than its Results share, one add of every read gives the same Winners, and after a reset Winners are zeros.
#include <cinttypes>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>

#include "poly_b200.hpp"

using namespace poly;

static int fail(const char *what) {
    std::printf("FAIL: %s\n", what);
    return 1;
}

static bool same_results(const mash::Screen::Result &a, const mash::Screen::Result &b) {
    return a.Shared == b.Shared && a.Multiplicity == b.Multiplicity && a.Containment.size() == b.Containment.size() &&
           std::memcmp(a.Containment.data(), b.Containment.data(), 8 * a.Containment.size()) == 0;
}

int main(int argc, char **argv) {
    if (argc != 5) return fail("usage: screen_winners_tests REFS READS K BATCHES");
    const auto refs = mash::MashesOf(mash::LoadSketchSet(argv[1]));
    std::vector<std::string> reads;
    std::ifstream in(argv[2]);
    for (std::string line; std::getline(in, line);) reads.push_back(line);
    const int k = std::atoi(argv[3]);
    const size_t batches = std::strtoul(argv[4], nullptr, 10);
    if (batches < 1) return fail("need one batch");
    mash::Screen sc(refs, k);
    size_t at = 0;
    for (size_t b = 1; b <= batches; ++b) {  // batch b takes a share that grows with b
        const size_t end = b == batches ? reads.size() : std::min(reads.size(), at + reads.size() * 2 * b / (batches * (batches + 1)));
        sc.Add(std::vector<std::string>(reads.begin() + at, reads.begin() + end));
        at = end;
    }
    const auto first = sc.Results();
    const auto got = sc.Winners();
    for (size_t r = 0; r < refs.size(); ++r) {
        uint64_t bits;
        std::memcpy(&bits, &got.Containment[r], 8);
        std::printf("%zu %u %016" PRIx64 " %" PRIu64 "\n", r, got.Shared[r], bits, got.Multiplicity[r]);
    }
    if (!same_results(sc.Results(), first)) return fail("Winners changed Results");
    for (size_t r = 0; r < refs.size(); ++r)
        if (got.Shared[r] > first.Shared[r]) return fail("a reference won more than it shares");
    mash::Screen whole(refs, k);
    whole.Add(reads);
    if (!same_results(whole.Winners(), got)) return fail("one add differs from the batched adds");
    sc.Reset();
    const auto empty = sc.Winners();
    for (size_t r = 0; r < refs.size(); ++r)
        if (empty.Shared[r] != 0 || empty.Multiplicity[r] != 0 || empty.Containment[r] != 0.0) return fail("reset left counts");
    std::printf("ok: screen winners tests pass\n");
    return 0;
}
