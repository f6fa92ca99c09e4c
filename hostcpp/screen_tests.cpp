// screen_tests.cpp -- Mash Screen through the C++ host mirror (poly::mash::Screen).
// Usage: screen_tests REFS.pgsketch READS.txt K BATCHES
// READS.txt holds one read per line.  Screens the reads against the references in BATCHES adds of unequal size and
// prints one line per reference, "r shared containment_bits multiplicity", then "ok: screen tests pass" after its
// own checks: one add of every read, and a reset followed by the same adds, give the same results.
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
    if (argc != 5) return fail("usage: screen_tests REFS READS K BATCHES");
    const auto refs = mash::MashesOf(mash::LoadSketchSet(argv[1]));
    std::vector<std::string> reads;
    std::ifstream in(argv[2]);
    for (std::string line; std::getline(in, line);) reads.push_back(line);
    const int k = std::atoi(argv[3]);
    const size_t batches = std::strtoul(argv[4], nullptr, 10);
    if (batches < 1) return fail("need one batch");
    mash::Screen sc(refs, k);
    auto add_in_batches = [&]() {
        size_t at = 0;
        for (size_t b = 1; b <= batches; ++b) {  // batch b takes a share that grows with b
            const size_t end = b == batches ? reads.size() : std::min(reads.size(), at + reads.size() * 2 * b / (batches * (batches + 1)));
            sc.Add(std::vector<std::string>(reads.begin() + at, reads.begin() + end));
            at = end;
        }
    };
    add_in_batches();
    const auto got = sc.Results();
    for (size_t r = 0; r < refs.size(); ++r) {
        uint64_t bits;
        std::memcpy(&bits, &got.Containment[r], 8);
        std::printf("%zu %u %016" PRIx64 " %" PRIu64 "\n", r, got.Shared[r], bits, got.Multiplicity[r]);
    }
    mash::Screen whole(refs, k);
    whole.Add(reads);
    if (!same_results(whole.Results(), got)) return fail("one add differs from the batched adds");
    sc.Reset();
    const auto empty = sc.Results();
    for (size_t r = 0; r < refs.size(); ++r)
        if (empty.Shared[r] != 0 || empty.Multiplicity[r] != 0 || empty.Containment[r] != 0.0) return fail("reset left counts");
    add_in_batches();
    if (!same_results(sc.Results(), got)) return fail("the adds after a reset differ");
    const auto id = sc.Identity();
    for (size_t r = 0; r < refs.size(); ++r)
        if (id[r] != std::pow(got.Containment[r], 1.0 / k)) return fail("identity is not containment^(1/k)");
    std::printf("ok: screen tests pass\n");
    return 0;
}
