// sketch_groups_tests.cpp -- grouped sketches through the C++ host mirror (poly::mash::SketchGroups).
// Usage: sketch_groups_tests GROUPS.txt N_GROUPS K S MIN_COPIES
// GROUPS.txt holds one record per line, "g record", g its group (groups without a line are empty).  Prints one line
// per group, "count v0 v1 ...", then "ok: sketch groups tests pass" after its own checks: every row is ascending with
// no repeat and a zero tail, the groups in reverse order give the same rows, and a group's rows are the same when it is
// sketched alone.
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
    if (argc != 6) return fail("usage: sketch_groups_tests GROUPS N_GROUPS K S MIN_COPIES");
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
    std::vector<uint32_t> count;
    const auto rows = mash::SketchGroups(groups, k, s, m, &count);
    if (rows.size() != G || count.size() != G) return fail("one sketch per group");
    for (size_t g = 0; g < G; ++g) {
        const auto &r = rows[g];
        if (r.KmerSize != k || r.SketchSize != s || (int)r.Sketches.size() != s) return fail("a sketch of the wrong shape");
        for (uint32_t i = 1; i < count[g]; ++i)
            if (r.Sketches[i - 1] >= r.Sketches[i]) return fail("a row that is not strictly ascending");
        for (int i = (int)count[g]; i < s; ++i)
            if (r.Sketches[i]) return fail("a row without its zero tail");
        std::printf("%u", count[g]);
        for (uint32_t i = 0; i < count[g]; ++i) std::printf(" %u", r.Sketches[i]);
        std::printf("\n");
    }
    std::vector<std::vector<std::string>> rev(groups.rbegin(), groups.rend());
    std::vector<uint32_t> rcount;
    const auto back = mash::SketchGroups(rev, k, s, m, &rcount);
    for (size_t g = 0; g < G; ++g)
        if (back[G - 1 - g].Sketches != rows[g].Sketches || rcount[G - 1 - g] != count[g]) return fail("the group order changed a row");
    for (size_t g = 0; g < G; ++g) {
        std::vector<uint32_t> one;
        const auto alone = mash::SketchGroups({groups[g]}, k, s, m, &one);
        if (alone[0].Sketches != rows[g].Sketches || one[0] != count[g]) return fail("a group sketched alone differs");
    }
    std::printf("ok: sketch groups tests pass\n");
    return 0;
}
