// sketcher_tests.cpp -- grouped sketches grown in place through the C++ host mirror (poly::mash::Sketcher).
// Usage: sketcher_tests GROUPS.txt N_GROUPS K S MIN_COPIES
// GROUPS.txt holds one record per line, "g record", g its group (groups without a line are empty).  Feeds every
// record to its group one add per record, prints one line per group, "count v0 v1 ...", then "ok: sketcher tests pass"
// after its own checks: every complete row equals mash::SketchGroups over the same records, every row is a prefix of
// it, and a second sketcher fed each group in one add gives the same rows.
#include <cstdio>
#include <cstdlib>
#include <fstream>

#include "poly_b200.hpp"

using namespace poly;

static int fail(const char *what) {
    std::printf("FAIL: %s\n", what);
    return 1;
}

int main(int argc, char **argv) {
    if (argc != 6) return fail("usage: sketcher_tests GROUPS N_GROUPS K S MIN_COPIES");
    const size_t G = std::strtoull(argv[2], nullptr, 10);
    const int k = std::atoi(argv[3]), s = std::atoi(argv[4]);
    const uint32_t m = (uint32_t)std::strtoul(argv[5], nullptr, 10);
    std::vector<std::vector<std::string>> groups(G);
    std::ifstream in(argv[1]);
    for (std::string line; std::getline(in, line);) {
        const size_t sp = line.find(' ');
        if (sp == std::string::npos) return fail("a line without a group");
        const size_t g = std::strtoull(line.substr(0, sp).c_str(), nullptr, 10);
        if (g >= G) return fail("a group out of range");
        groups[g].push_back(line.substr(sp + 1));
    }
    mash::Sketcher one_by_one(G, k, s, m), whole(G, k, s, m);
    for (size_t g = 0; g < G; ++g)
        for (const auto &r : groups[g]) one_by_one.AddRecords(g, {r});
    whole.Add(groups);
    std::vector<uint32_t> count, wcount, ocount;
    std::vector<uint8_t> complete;
    const auto rows = one_by_one.Sketches(&count, &complete);
    const auto wrows = whole.Sketches(&wcount);
    const auto once = mash::SketchGroups(groups, k, s, m, &ocount);
    if (rows.size() != G || count.size() != G) return fail("one sketch per group");
    for (size_t g = 0; g < G; ++g) {
        const auto &r = rows[g];
        if (r.KmerSize != k || r.SketchSize != s || (int)r.Sketches.size() != s) return fail("a sketch of the wrong shape");
        if (count[g] > ocount[g]) return fail("a row longer than the one-shot row");
        for (uint32_t i = 0; i < count[g]; ++i)
            if (r.Sketches[i] != once[g].Sketches[i]) return fail("a row that is not a prefix of the one-shot row");
        if (complete[g] && (r.Sketches != once[g].Sketches || count[g] != ocount[g])) return fail("a complete row differs from the one-shot row");
        if (complete[g] && (wrows[g].Sketches != r.Sketches || wcount[g] != count[g])) return fail("the split changed a complete row");
        std::printf("%u", count[g]);
        for (uint32_t i = 0; i < count[g]; ++i) std::printf(" %u", r.Sketches[i]);
        std::printf("\n");
    }
    std::printf("ok: sketcher tests pass\n");
    return 0;
}
