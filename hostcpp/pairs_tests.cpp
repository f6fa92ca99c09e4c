// pairs_tests.cpp -- the poly::align pair-list functions against the reference's known answers
// (align_test.go, example_test.go) and against the single-pair functions.
#include <cstdio>
#include <string>
#include <vector>

#include "poly_b200.hpp"

static int failures = 0;
#define EXPECT(cond)                                                              \
    do {                                                                          \
        if (!(cond)) { std::printf("FAIL %s:%d: %s\n", __FILE__, __LINE__, #cond); ++failures; } \
    } while (0)

using namespace poly;

int main() {
    auto alphabet = align::NewAlphabet({"-", "A", "C", "G", "T"});
    auto sub = align::NewSubstitutionMatrix(alphabet, alphabet,
                                            {{0, 0, 0, 0, 0}, {0, 3, -3, -3, -3}, {0, -3, 3, -3, -3}, {0, -3, -3, 3, -3}, {0, -3, -3, -3, 3}});
    auto sc = align::NewScoring(&sub, -2);
    const std::vector<std::string> as = {"TGTTACGG", "ACACACTA", "", "G", "ACGX"};
    const std::vector<std::string> bs = {"GGTTGACTA", "AGCACACA", "GAT", "A", "G", "GATTACA", "ACGT"};
    const std::vector<uint32_t> pa = {0, 1, 2, 2, 3, 3, 3, 4}, pb = {0, 1, 2, 3, 3, 4, 5, 6};
    std::vector<std::string> errs;
    auto s = align::SmithWatermanPairScores(as, bs, pa, pb, sc, &errs);
    EXPECT((s == std::vector<int64_t>{13, 17, 0, 0, 0, 3, 3, 0}));
    EXPECT(errs[7] == "Symbol X not in alphabet" && errs[0].empty());
    for (size_t k = 0; k + 1 < pa.size(); ++k) EXPECT(align::NeedlemanWunschPairScores(as, bs, {pa[k]}, {pb[k]}, sc)[0] ==
                                                       align::NeedlemanWunschScore(as[pa[k]], bs[pb[k]], sc));
    auto al = align::SmithWatermanPairAligns(as, bs, pa, pb, sc, &errs);
    EXPECT(al[0].score == 13 && al[0].alignA == "GTT-AC" && al[0].alignB == "GTTGAC");
    EXPECT(al[1].score == 17 && al[1].alignA == "A-CACACTA" && al[1].alignB == "AGCACAC-A");
    EXPECT(al[6].score == 3 && al[6].alignA == "G" && al[6].alignB == "G");
    EXPECT(errs[7] == "Symbol X not in alphabet");
    auto nw = align::NeedlemanWunschPairAligns(as, bs, {0}, {0}, sc);
    auto one = align::NeedlemanWunschAlign(as[0], bs[0], sc);
    EXPECT(nw[0].score == one.score && nw[0].alignA == one.alignA && nw[0].alignB == one.alignB);
    bool threw = false;
    try { align::SmithWatermanPairScores(as, bs, {5}, {0}, sc); } catch (const Error &) { threw = true; }
    EXPECT(threw);
    if (failures) { std::printf("%d failures\n", failures); return 1; }
    std::printf("pairs_tests ok\n");
    return 0;
}
