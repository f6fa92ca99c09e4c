// fold_tests.cpp -- fold_test.go, seqfold_test.go and example_test.go (fold/) restated against the C++ host
// mirror, plus exact parity with the C restatement on a fixture list.
// Usage: fold_tests EXPECTED.tsv -- one "sequence<TAB>temp<TAB>status<TAB>mfe as %a<TAB>dot-bracket" line per
// item, written by tests/test_gpu_fold.py from oracle/fold_oracle.c.  Prints "fold_tests: all passed" when every
// check holds.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <sstream>

#include "poly_b200.hpp"

using namespace poly;

static int failures = 0;
static void expect(bool ok, const std::string &what) {
    if (!ok) {
        std::printf("FAIL: %s\n", what.c_str());
        ++failures;
    }
}

int main(int argc, char **argv) {
    if (argc != 2) {
        std::printf("FAIL: usage: fold_tests EXPECTED.tsv\n");
        return 1;
    }
    // TestFold/FoldDNA and FoldRNA (fold_test.go:25-69): unafold's estimates within 60 % / 50 %
    const struct {
        const char *seq;
        double want, frac;
    } unafold[] = {
        {"GGGAGGTCGTTACATCTGGGTAACACCGGTACTGATCCGGTGACCTCCC", -10.94, 0.6},
        {"GGGAGGTCGCTCCAGCTGGGAGGAGCGTTGGGGGTATATACCCCCAACACCGGTACTGATCCGGTGACCTCCC", -23.4, 0.6},
        {"CGCAGGGAUACCCGCG", -3.8, 0.6},
        {"TAGCTCAGCTGGGAGAGCGCCTGCTTTGCACGCAGGAGGT", -6.85, 0.6},
        {"GGGGGCATAGCTCAGCTGGGAGAGCGCCTGCTTTGCACGCAGGAGGTCTGCGGTTCGATCCCGCGCGCTCCCACCA", -15.50, 0.6},
        {"TGAGACGGAAGGGGATGATTGTCCCCTTCCGTCTCA", -18.10, 0.6},
        {"ACCCCCTCCTTCCTTGGATCAAGGGGCTCAA", -3.65, 0.6},
        {"ACCCCCUCCUUCCUUGGAUCAAGGGGCUCAA", -9.5, 0.5},
        {"AAGGGGUUGGUCGCCUCGACUAAGCGGCUUGGAAUUCC", -10.1, 0.5},
        {"UUGGAGUACACAACCUGUACACUCUUUC", -4.3, 0.5},
        {"AGGGAAAAUCCC", -3.3, 0.5},
        {"GCUUACGAGCAAGUUAAGCAAC", -4.6, 0.5},
        {"UGGGAGGUCGUCUAACGGUAGGACGGCGGACUCUGGAUCCGCUGGUGGAGGUUCGAGUCCUCCCCUCCCAGCCA", -32.8, 0.5},
        {"GGGCGAUGAGGCCCGCCCAAACUGCCCUGAAAAGGGCUGAUGGCCUCUACUG", -20.7, 0.5},
        {"GGGGGCAUAGCUCAGCUGGGAGAGCGCCUGCUUUGCACGCAGGAGGUCUGCGGUUCGAUCCCGCGCGCUCCCACCA", -31.4, 0.5},
    };
    for (auto &u : unafold) {
        const auto r = fold::Zuker(u.seq, 37.0);
        const double d = r.first.MinimumFreeEnergy();
        expect(r.second.empty() && std::fabs(d - u.want) <= std::fabs(u.frac * std::min(d, u.want)), std::string("unafold ") + u.seq);
    }
    // TestFold/DotBracket and ExampleZuker
    expect(fold::Zuker("GGGAGGTCGTTACATCTGGGTAACACCGGTACTGATCCGGTGACCTCCC", 37.0).first.DotBracket() ==
               "((((((((.((((......))))..((((.......)))).))))))))",
           "DotBracket");
    expect(fold::Zuker("ACCCCCUCCUUCCUUGGAUCAAGGGGCUCAA", 37.0).first.DotBracket() == ".((((.(((......)))....))))", "ExampleZuker");
    // TestZuker_ErrorCreatingFoldingContext and TestNewFoldingContext_InvalidSequence
    expect(fold::Zuker("ATGGATTTAGATAGATADFQ#(RSDOFIA)", 4000.0).second ==
               "error creating folding context: the sequence ATGGATTTAGATAGATADFQ#(RSDOFIA) is not RNA or DNA",
           "error message");
    expect(fold::Zuker("XYZ", 37.0).second.find("the sequence XYZ is not RNA or DNA") != std::string::npos, "XYZ");
    // TestResult_MinimumFreeEnergy_LengthZero / TestResult_DotBracket_LengthZero
    expect(fold::Result().MinimumFreeEnergy() == std::numeric_limits<double>::infinity() && fold::Result().DotBracket().empty(), "empty Result");
    bool threw = false;
    try {
        fold::Zuker("", 37.0);
    } catch (const GoPanic &) {
        threw = true;
    }
    expect(threw, "empty sequence panics");
    // exact parity with the C restatement, one GPU call per temperature
    std::map<double, std::vector<std::vector<std::string>>> rows;
    std::ifstream in(argv[1]);
    for (std::string line; std::getline(in, line);) {
        std::vector<std::string> f;
        std::istringstream ls(line);
        for (std::string x; std::getline(ls, x, '\t');) f.push_back(x);
        f.resize(5);
        rows[std::strtod(f[1].c_str(), nullptr)].push_back(f);
    }
    size_t n = 0;
    for (auto &[temp, fs] : rows) {
        std::vector<std::string> seqs;
        for (auto &f : fs) seqs.push_back(f[0]);
        const auto got = fold::ZukerBatch(seqs, temp);
        for (size_t i = 0; i < fs.size(); ++i, ++n) {
            const int st = std::atoi(fs[i][2].c_str());
            bool ok = got[i].status == st;
            if (ok && st == PG_ITEM_OK) {
                const double want = std::strtod(fs[i][3].c_str(), nullptr);
                ok = std::memcmp(&want, &got[i].result.mfe, 8) == 0 && got[i].result.DotBracket() == fs[i][4];
            }
            expect(ok, "parity " + fs[i][0]);
        }
    }
    expect(n > 0, "fixture rows");
    if (failures) return 1;
    std::printf("fold_tests: all passed (%zu parity items)\n", n);
    return 0;
}
