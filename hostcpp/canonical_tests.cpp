// canonical_tests.cpp -- canonical k-mers (PG_KMER_CANONICAL) through the C++ host mirror: SketchGroups, Sketcher and
// Screen with canonical = true.
// Usage: canonical_tests GROUPS.txt N_GROUPS K S MIN_COPIES
// GROUPS.txt holds one record per line, "g record", g its group.  Prints one line per group of the canonical
// SketchGroups, "count v0 v1 ...", then the canonical screen's Shared of every group's reads against those sketches,
// "shared x0 x1 ...", then "ok: canonical tests pass" after its own checks: a canonical Sketcher fed one record per add
// gives the same complete rows, every group with its records reverse-complemented gives the same rows, and each
// group's own reads share every value of its sketch in the canonical screen.
#include <cstdio>
#include <cstdlib>
#include <fstream>

#include "poly_b200.hpp"

using namespace poly;

static int fail(const char *what) {
    std::printf("FAIL: %s\n", what);
    return 1;
}

static std::string revcomp(const std::string &s) {
    std::string r(s.size(), '\0');
    for (size_t i = 0; i < s.size(); ++i) {
        const char c = s[s.size() - 1 - i];
        r[i] = c == 'A' ? 'T' : c == 'C' ? 'G' : c == 'G' ? 'C' : c == 'T' ? 'A' : c;
    }
    return r;
}

int main(int argc, char **argv) {
    if (argc != 6) return fail("usage: canonical_tests GROUPS N_GROUPS K S MIN_COPIES");
    const size_t G = std::strtoull(argv[2], nullptr, 10);
    const int k = std::atoi(argv[3]), s = std::atoi(argv[4]);
    const uint32_t m = (uint32_t)std::strtoul(argv[5], nullptr, 10);
    std::vector<std::vector<std::string>> groups(G), flipped(G);
    std::ifstream in(argv[1]);
    for (std::string line; std::getline(in, line);) {
        const size_t sp = line.find(' ');
        if (sp == std::string::npos) return fail("a line without a group");
        const size_t g = std::strtoull(line.substr(0, sp).c_str(), nullptr, 10);
        if (g >= G) return fail("a group out of range");
        groups[g].push_back(line.substr(sp + 1));
        flipped[g].push_back(revcomp(groups[g].back()));  // the records hold upper-case ACGT
    }
    std::vector<uint32_t> count, fcount, scount;
    std::vector<uint8_t> complete;
    const auto rows = mash::SketchGroups(groups, k, s, m, &count, true);
    const auto frows = mash::SketchGroups(flipped, k, s, m, &fcount, true);
    mash::Sketcher sk(G, k, s, m, 0, true);
    for (size_t g = 0; g < G; ++g)
        for (const auto &r : groups[g]) sk.AddRecords(g, {r});
    const auto srows = sk.Sketches(&scount, &complete);
    for (size_t g = 0; g < G; ++g) {
        if (frows[g].Sketches != rows[g].Sketches || fcount[g] != count[g]) return fail("reverse complements changed a canonical row");
        if (complete[g] && (srows[g].Sketches != rows[g].Sketches || scount[g] != count[g])) return fail("a complete sketcher row differs");
        std::printf("%u", count[g]);
        for (uint32_t i = 0; i < count[g]; ++i) std::printf(" %u", rows[g].Sketches[i]);
        std::printf("\n");
    }
    std::printf("shared");
    for (size_t g = 0; g < G; ++g) {
        mash::Screen sc(rows, k, 1, true);
        sc.Add(flipped[g]);
        const auto r = sc.Results();
        if (r.Shared[g] != count[g]) return fail("a group's own reads miss a value of its canonical sketch");
        std::printf(" %u", r.Shared[g]);
    }
    std::printf("\nok: canonical tests pass\n");
    return 0;
}
