// screen_samples_tests.cpp -- a screen of several samples through the C++ host mirror (poly::mash::Screen::AddSamples,
// ResultsSamples, WinnersSamples).
// Usage: screen_samples_tests REFS.pgsketch READS.txt K SAMPLES
// READS.txt holds one read per line, "q read", q its sample id.  Adds the reads in two halves, then prints one line per
// (sample, reference) of ResultsSamples, "q r shared containment_bits multiplicity", then "ok: screen samples tests
// pass" after its own checks: every row of ResultsSamples and WinnersSamples equals a one-sample screen fed only that
// sample's reads, Results and Winners equal row 0, a sub-range equals the matching rows, and after a reset every row
// is zeros.
#include <cinttypes>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <sstream>

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
    if (argc != 5) return fail("usage: screen_samples_tests REFS READS K SAMPLES");
    const auto refs = mash::MashesOf(mash::LoadSketchSet(argv[1]));
    std::vector<std::string> reads;
    std::vector<uint32_t> ids;
    std::ifstream in(argv[2]);
    for (std::string line; std::getline(in, line);) {
        const size_t sp = line.find(' ');
        if (sp == std::string::npos) return fail("a line without a sample id");
        ids.push_back((uint32_t)std::strtoul(line.substr(0, sp).c_str(), nullptr, 10));
        reads.push_back(line.substr(sp + 1));
    }
    const int k = std::atoi(argv[3]);
    const uint32_t S = (uint32_t)std::strtoul(argv[4], nullptr, 10);
    if (S < 1) return fail("need one sample");
    mash::Screen sc(refs, k, S);
    const size_t half = reads.size() / 2;
    sc.AddSamples(std::vector<std::string>(reads.begin(), reads.begin() + half), std::vector<uint32_t>(ids.begin(), ids.begin() + half));
    sc.AddSamples(std::vector<std::string>(reads.begin() + half, reads.end()), std::vector<uint32_t>(ids.begin() + half, ids.end()));
    const auto got = sc.ResultsSamples(0, S);
    const auto won = sc.WinnersSamples(0, S);
    for (uint32_t q = 0; q < S; ++q)
        for (size_t r = 0; r < refs.size(); ++r) {
            uint64_t bits;
            std::memcpy(&bits, &got[q].Containment[r], 8);
            std::printf("%u %zu %u %016" PRIx64 " %" PRIu64 "\n", q, r, got[q].Shared[r], bits, got[q].Multiplicity[r]);
        }
    for (uint32_t q = 0; q < S; ++q) {
        std::vector<std::string> mine;
        for (size_t i = 0; i < reads.size(); ++i)
            if (ids[i] == q) mine.push_back(reads[i]);
        mash::Screen one(refs, k);
        one.Add(mine);
        if (!same_results(one.Results(), got[q])) return fail("a row of ResultsSamples differs from its one-sample screen");
        if (!same_results(one.Winners(), won[q])) return fail("a row of WinnersSamples differs from its one-sample screen");
    }
    if (!same_results(sc.Results(), got[0]) || !same_results(sc.Winners(), won[0])) return fail("Results or Winners is not row 0");
    if (S > 1) {
        const auto sub = sc.ResultsSamples(1, S - 1);
        for (uint32_t q = 1; q < S; ++q)
            if (!same_results(sub[q - 1], got[q])) return fail("a sub-range differs from the full table");
    }
    sc.Reset();
    for (const auto &row : sc.ResultsSamples(0, S))
        for (size_t r = 0; r < refs.size(); ++r)
            if (row.Shared[r] != 0 || row.Multiplicity[r] != 0 || row.Containment[r] != 0.0) return fail("reset left counts");
    std::printf("ok: screen samples tests pass\n");
    return 0;
}
