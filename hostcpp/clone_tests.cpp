// clone_tests.cpp -- clone_test.go and example_test.go (clone/) restated against the C++ host mirror.
// Usage: clone_tests FIXTURES.tsv -- one "group<TAB>name<TAB>circular(0/1)<TAB>sequence" line per part of the
// reference's tests (groups: popen, TestSignalKilledGoldenGate, TestPanicGoldenGate, TestCircularCutRegression,
// example, example_output).  Prints "clone_tests: all passed" when every check holds.
#include <cstdio>
#include <fstream>
#include <sstream>

#include "poly_b200.hpp"

using namespace poly;
using namespace poly::clone;

static int failures = 0;
static void expect(bool ok, const std::string &what) {
    if (!ok) {
        std::printf("FAIL: %s\n", what.c_str());
        ++failures;
    }
}

int main(int argc, char **argv) {
    if (argc != 2) {
        std::printf("FAIL: usage: clone_tests FIXTURES.tsv\n");
        return 1;
    }
    std::map<std::string, std::vector<Part>> fx;
    std::ifstream in(argv[1]);
    for (std::string line; std::getline(in, line);) {
        std::istringstream ls(line);
        std::string group, name, circ, seq;
        std::getline(ls, group, '\t'); std::getline(ls, name, '\t'); std::getline(ls, circ, '\t'); std::getline(ls, seq, '\t');
        fx[group].push_back(Part{seq, circ == "1"});
    }
    const Part popen = fx["popen"].at(0);
    EnzymeManager em = NewEnzymeManager(GetBaseRestrictionEnzymes());
    // TestCutWithEnzymeByName (clone_test.go:10-16)
    expect(!em.CutWithEnzymeByName(popen, true, "EcoFake").second.empty(), "EcoFake must not be found");
    // TestCutWithEnzyme (:18-97)
    const std::string bsai = "GGTCTCAATGC", bsaiComplement = "ATGCAGAGACC";
    Part seq{"ATATATA" + bsaiComplement + bsai + "ATGCATCGATCGACTAGCATG" + bsaiComplement + bsai.substr(0, 8), false};
    auto f = em.CutWithEnzymeByName(seq, true, "BsaI").first;
    expect(f.size() == 1 && f[0].Sequence == "ATGCATCGATCGACTAGCATG", "test(1)");
    seq.Circular = true;
    f = em.CutWithEnzymeByName(seq, true, "BsaI").first;
    expect(f.size() == 2 && f[0].Sequence == "ATGCATCGATCGACTAGCATG" && f[1].Sequence == "TATA", "test(2)");
    seq = Part{"ATATATATATATATAT" + bsai + "GCGCGCGCGCGCGCGCGCGC", false};
    f = em.CutWithEnzymeByName(seq, false, "BsaI").first;
    expect(f.size() == 2 && f[0].Sequence == "GCGCGCGCGCGCGCGCGCGC" && f[1].Sequence == "ATATATATATATATATGGTCTCA", "test(3)");
    seq.Circular = true;
    f = em.CutWithEnzymeByName(seq, false, "BsaI").first;
    expect(f.size() == 1 && f[0].Sequence == "GCGCGCGCGCGCGCGCGCGCATATATATATATATATGGTCTCA", "test(4)");
    expect(em.CutWithEnzymeByName(popen, false, "BbsI").first.size() == 2, "test(5)");
    // TestCutWithEnzymeRegression (:99-140)
    const std::string reg = "AGCTGCTGTTTAAAGCTATTACTTTGAGACC";
    f = CutWithEnzyme(Part{reg, false}, false, em.GetEnzymeByName("BsaI").first);
    expect(f.size() == 2 && f[0].ForwardOverhang.empty() && f[0].ReverseOverhang == "ACTT" && f[1].ForwardOverhang == "ACTT" &&
               f[1].ReverseOverhang.empty() && f[0].Sequence + f[0].ReverseOverhang + f[1].Sequence == reg,
           "regression overhangs");
    // TestCircularLigate (:142-154)
    auto lig = CircularLigate({Fragment{"AAAAAA", "GTTG", "CTAT"}, Fragment{"AAAAAA", "CAAC", "ATAG"}});
    expect(lig.first.size() == 1 && lig.second.empty(), "CircularLigate: 1 construct, no loops");
    // TestEnzymeManage_GetEnzymeByName_NotFound (:156-165)
    expect(em.GetEnzymeByName("EcoRFake").second == "Enzyme EcoRFake not found", "not-found message");
    const Enzyme bbsI = em.GetEnzymeByName("BbsI").first;
    // TestSignalKilledGoldenGate (:167-194)
    std::vector<Part> parts{popen};
    for (const Part &p : fx["TestSignalKilledGoldenGate"]) parts.push_back(p);
    auto gg = GoldenGate(parts, bbsI);
    expect(gg.first.size() == 1 && gg.second.size() == 4, "SignalKilled: 1 clone, 4 looping constructs");
    // TestPanicGoldenGate (:196-214): runs and returns
    parts = {popen};
    for (const Part &p : fx["TestPanicGoldenGate"]) parts.push_back(p);
    GoldenGate(parts, bbsI);
    // TestCircularCutRegression (:216-228)
    expect(em.CutWithEnzymeByName(fx["TestCircularCutRegression"].at(0), true, "BsaI").first.size() == 1, "circular cut regression");
    // ExampleGoldenGate (example_test.go:11-31)
    parts = fx["example"];
    parts.push_back(popen);
    gg = GoldenGate(parts, bbsI);
    expect(!gg.first.empty() && seqhash::RotateSequence(gg.first[0]) == fx["example_output"].at(0).Sequence, "ExampleGoldenGate output");
    if (failures) return 1;
    std::printf("clone_tests: all passed\n");
    return 0;
}
