// mash_dist_tests.cpp -- Mash distance between grouped sketches through the C++ host mirror (poly::mash::Dist, DistWithin).
// Usage: mash_dist_tests GROUPS.txt N_GROUPS K S MAX_DISTANCE
// GROUPS.txt holds one record per line, "g record", g its group.  The groups are sketched with SketchGroups, each with
// its length the sum of its record lengths, and compared all against all.  Prints one line per pair, "q r common denom
// distance p" (doubles as %a), then "ok: mash dist tests pass" after its own checks: the matrix is symmetric, each group
// has distance 0 to itself, and DistWithin(..., MAX_DISTANCE, upper) lists exactly the pairs r > q of the matrix within
// the cut.
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
    if (argc != 6) return fail("usage: mash_dist_tests GROUPS N_GROUPS K S MAX_DISTANCE");
    const size_t G = std::strtoull(argv[2], nullptr, 10);
    const int k = std::atoi(argv[3]), s = std::atoi(argv[4]);
    const double maxd = std::strtod(argv[5], nullptr);
    std::vector<std::vector<std::string>> groups(G);
    std::vector<uint64_t> len(G, 0);
    std::ifstream in(argv[1]);
    for (std::string line; std::getline(in, line);) {
        const size_t sp = line.find(' ');
        if (sp == std::string::npos) return fail("a line without a group");
        const size_t g = std::strtoull(line.substr(0, sp).c_str(), nullptr, 10);
        if (g >= G) return fail("a group out of range");
        groups[g].push_back(line.substr(sp + 1));
        len[g] += line.size() - sp - 1;
    }
    std::vector<uint32_t> count;
    const auto sk = mash::SketchGroups(groups, k, s, 1, &count);
    const auto d = mash::Dist(sk, count, sk, count, k, len, len);
    for (size_t q = 0; q < G; ++q)
        for (size_t r = 0; r < G; ++r) {
            const size_t o = q * G + r, t = r * G + q;
            if (d.common[o] != d.common[t] || d.denom[o] != d.denom[t] || d.distance[o] != d.distance[t] || d.pValue[o] != d.pValue[t])
                return fail("the matrix is not symmetric");
            std::printf("%zu %zu %u %u %a %a\n", q, r, d.common[o], d.denom[o], d.distance[o], d.pValue[o]);
        }
    for (size_t g = 0; g < G; ++g)
        if (d.distance[g * G + g] != 0.0 || d.common[g * G + g] != count[g] || d.denom[g * G + g] != count[g]) return fail("a group is not at 0 from itself");
    const auto w = mash::DistWithin(sk, count, sk, count, k, len, len, maxd, 1.0, true);
    size_t t = 0;
    for (size_t q = 0; q < G; ++q)
        for (size_t r = q + 1; r < G; ++r) {
            if (!(d.distance[q * G + r] <= maxd)) continue;
            if (t >= w.q.size() || w.q[t] != q || w.r[t] != r || w.common[t] != d.common[q * G + r] || w.distance[t] != d.distance[q * G + r] ||
                w.pValue[t] != d.pValue[q * G + r])
                return fail("DistWithin differs from the filtered matrix");
            ++t;
        }
    if (t != w.q.size()) return fail("DistWithin lists extra pairs");
    std::printf("ok: mash dist tests pass\n");
    return 0;
}
