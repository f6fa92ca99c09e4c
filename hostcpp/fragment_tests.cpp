// fragment_tests.cpp -- fragment_test.go and example_test.go (synthesis/fragment/) restated against the C++ host
// mirror, plus exact parity with the C restatement on a fixture list.
// Usage: fragment_tests EXPECTED.tsv -- written by tests/test_gpu_fragment.py from oracle/fragment_oracle.c and
// tests/golden/fragment/pins.json.  Lines:
//   F <name> seq min max excludes includes status efficiency(%a) fragments error     (lists joined with ',')
//   S set efficiency(%a)
//   N set candidates efficiencies(%a)
// Named F rows (the reference's tests) are checked for what the reference asserts; every row is checked for
// exact parity.  Prints "fragment_tests: all passed" when every check holds.
#include <cstdio>
#include <cstdlib>
#include <cstring>
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

static std::vector<std::string> split(const std::string &s, char sep) {
    std::vector<std::string> out;
    if (s.empty()) return out;
    std::istringstream ls(s);
    for (std::string x; std::getline(ls, x, sep);) out.push_back(x);
    if (s.back() == sep) out.push_back("");
    return out;
}

static bool same_bits(double a, double b) { return std::memcmp(&a, &b, 8) == 0; }

int main(int argc, char **argv) {
    if (argc != 2) {
        std::printf("FAIL: usage: fragment_tests EXPECTED.tsv\n");
        return 1;
    }
    size_t n = 0;
    std::ifstream in(argv[1]);
    for (std::string line; std::getline(in, line); ++n) {
        const std::vector<std::string> f = split(line, '\t');
        if (f[0] == "F") {
            const std::string &name = f[1], &seq = f[2];
            const int64_t mn = std::strtoll(f[3].c_str(), nullptr, 10), mx = std::strtoll(f[4].c_str(), nullptr, 10);
            const auto ex = split(f[5], ','), inc = split(f[6], ',');
            const int st = std::atoi(f[7].c_str());
            const double eff = std::strtod(f[8].c_str(), nullptr);
            const auto frags = split(f[9], ',');
            const fragment::Fragments got = inc.empty() ? fragment::Fragment(seq, mn, mx, ex) : fragment::FragmentWithOverhangs(seq, mn, mx, ex, inc);
            expect((st == PG_ITEM_OK) == got.error.empty() && got.fragments == frags && same_bits(got.efficiency, eff) && got.error == f[10],
                   "parity " + name + " " + seq.substr(0, 40));
            // what the reference's tests assert
            if (name == "TestFragment" || name == "TestSmallFragmentSize" || name == "TestFragmentWithOverhangs") expect(got.error.empty(), name);
            if (name == "TestUnfragmentable" || name == "TestFragmentSizes") expect(!got.error.empty(), name);
            if (name == "TestLongFragment") {
                expect(got.error.empty(), name);
                for (auto &x : got.fragments) expect(x.size() <= 94, "TestLongFragment: fragment of " + std::to_string(x.size()));
            }
        } else if (f[0] == "S") {
            expect(same_bits(fragment::SetEfficiency(split(f[1], ',')), std::strtod(f[2].c_str(), nullptr)), "SetEfficiency " + f[1]);
        } else if (f[0] == "N") {
            const auto got = fragment::NextOverhangs(split(f[1], ','));
            const auto effs = split(f[3], ',');
            bool ok = got.first == split(f[2], ',') && got.second.size() == effs.size();
            for (size_t i = 0; ok && i < effs.size(); ++i) ok = same_bits(got.second[i], std::strtod(effs[i].c_str(), nullptr));
            expect(ok, "NextOverhangs " + f[1]);
        }
    }
    expect(n > 0, "fixture rows");
    // TestCheckLongRegresssion: GTCT is the reverse complement of AGAC
    for (auto &c : fragment::NextOverhangs({"AGAC"}).first) expect(c != "GTCT", "GTCT offered after AGAC");
    // TestRegressionTestMatching12
    const double e = fragment::SetEfficiency({"CGAG", "GTCT", "TACT", "AATG", "ATCC", "CGCT", "AAAA", "AAGT", "ATAG", "ATTA", "ACAA", "ACGC",
                                              "TATC", "TAGA", "TTAC", "TTCA", "TGTG", "TCGG", "TCCC", "GAAG", "GTGC", "GCCG", "CAGG", "TACG"});
    expect(e <= 1 && e >= 0.965, "TestRegressionTestMatching12");
    // ExampleNextOverhang
    std::vector<std::string> primers{"ATAA"};
    for (int i = 0; i < 3; ++i) primers.push_back(fragment::NextOverhang(primers));
    expect(primers == std::vector<std::string>({"ATAA", "AAAT", "AATA", "AAGA"}), "ExampleNextOverhang");
    // the reference panics on fewer than 4 bytes
    bool threw = false;
    try {
        fragment::Fragment("ACG", 12, 30, {});
    } catch (const GoPanic &) {
        threw = true;
    }
    expect(threw, "a 3-byte sequence panics");
    if (failures) return 1;
    std::printf("fragment_tests: all passed (%zu fixture rows)\n", n);
    return 0;
}
