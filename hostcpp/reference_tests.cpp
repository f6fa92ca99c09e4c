// reference_tests.cpp -- the reference's own tests for the hot path, restated against the C++
// host mirror (hostcpp/poly_b200.hpp) so that they read like the originals:
//   search/mash/mash_test.go:9-62, search/mash/example_test.go:9-22,
//   search/align/align_test.go:139-292, search/align/example_test.go:49-111,
//   primers/primers_test.go:29-84, primers/pcr/pcr_test.go:12-101, primers/pcr/example_test.go:10-69.
// Needs an H100: every call below lands in libpolyb200.so.  Run by tests/test_gpu_hostcpp.py.
#include <cmath>
#include <cstdio>
#include <cstdlib>

#include "poly_b200.hpp"

static int failures = 0;
#define EXPECT(cond)                                                              \
    do {                                                                          \
        if (!(cond)) { std::printf("FAIL %s:%d: %s\n", __FILE__, __LINE__, #cond); ++failures; } \
    } while (0)

using namespace poly;

static void TestMash() {  // mash_test.go:9-62
    const std::string A = "ATGCGATCGATCGATCGATCGATCGATCGATCGATCGATCGATCGATCGATCGATCGATCGA";
    const std::string B = "ATCGATCGATCGATCGATCGATCGATCGATCGATCGAATGCGATCGATCGATCGATCGATCG";
    auto fingerprint1 = mash::New(17, 10); fingerprint1.Sketch(A);
    auto fingerprint2 = mash::New(17, 9); fingerprint2.Sketch(A);
    EXPECT(fingerprint1.Distance(fingerprint2) == 0);
    EXPECT(fingerprint2.Distance(fingerprint1) == 0);
    auto spoofed = mash::New(17, 10); spoofed.Sketches[0] = 0;
    EXPECT(fingerprint1.Distance(spoofed) == 1);
    spoofed = mash::New(17, 9);
    EXPECT(fingerprint1.Distance(spoofed) == 1);
    fingerprint1 = mash::New(17, 10); fingerprint1.Sketch(A);
    fingerprint2 = mash::New(17, 5); fingerprint2.Sketch(B);
    double d = fingerprint1.Distance(fingerprint2);
    EXPECT(d > 0.19 && d < 0.21 && d == 0.19999999999999996);
    fingerprint1 = mash::New(17, 10); fingerprint1.Sketch(B);
    fingerprint2 = mash::New(17, 5); fingerprint2.Sketch(A);
    EXPECT(fingerprint1.Distance(fingerprint2) == 0);
    // batched addition agrees with the object API
    auto batch = mash::SketchBatch({A, B, "ACGT", ""}, 17, 10);
    auto one = mash::New(17, 10); one.Sketch(B);
    EXPECT(batch[1].Sketches == one.Sketches);
    EXPECT(batch[2].Sketches == std::vector<uint32_t>(10, 0u));
    bool panicked = false;
    try { mash::New(17, 0).Distance(mash::New(17, 3)); } catch (const GoPanic &) { panicked = true; }
    EXPECT(panicked);
}

static void TestSmithWaterman() {  // align_test.go:139-292 (scores)
    auto alphabet = align::NewAlphabet({"-", "A", "C", "G", "T"});
    auto sub = align::NewSubstitutionMatrix(alphabet, alphabet,
                                            {{0, 0, 0, 0, 0}, {0, 3, -3, -3, -3}, {0, -3, 3, -3, -3}, {0, -3, -3, 3, -3}, {0, -3, -3, -3, 3}});
    auto scoring = align::NewScoring(&sub, -2);
    EXPECT(align::SmithWaterman("TGTTACGG", "GGTTGACTA", scoring) == 13);
    EXPECT(align::SmithWaterman("ACACACTA", "AGCACACA", scoring) == 17);
    EXPECT(align::SmithWaterman("", "GAT", scoring) == 0);
    EXPECT(align::SmithWaterman("", "", scoring) == 0);
    EXPECT(align::SmithWaterman("G", "A", scoring) == 0);
    EXPECT(align::SmithWaterman("G", "G", scoring) == 3);
    EXPECT(align::SmithWaterman("G", "GATTACA", scoring) == 3);
    // example_test.go:49-111
    auto a5 = align::NewAlphabet({"A", "C", "G", "T", "U"});
    std::vector<std::vector<int64_t>> m5(5, std::vector<int64_t>(5, -1));
    for (int i = 0; i < 5; ++i) m5[i][i] = 1;
    auto s5 = align::NewSubstitutionMatrix(a5, a5, m5);
    EXPECT(align::SmithWaterman("GATTACA", "GCATGCU", align::NewScoring(&s5, -1)) == 2);
    auto an = align::NewAlphabet({"A", "C", "G", "T", "-"});
    auto nuc4 = align::NewSubstitutionMatrix(an, an, {{0, 0, 0, 0, 0}, {0, 5, -4, -4, -4}, {0, -4, 5, -4, -4}, {0, -4, -4, 5, -4}, {0, -4, -4, -4, 5}});
    EXPECT(align::SmithWaterman("GATTACA", "GCATGCT", align::NewScoring(&nuc4, -1)) == 15);
    EXPECT(align::SmithWaterman("GATTACA", "GCATGCU", align::NewScoring(nullptr, -1)) == 2);
    // aligned strings (align_test.go:167-196, example_test.go:82,110)
    auto al = align::SmithWatermanAlign("TGTTACGG", "GGTTGACTA", scoring);
    EXPECT(al.score == 13 && al.alignA == "GTT-AC" && al.alignB == "GTTGAC");
    al = align::SmithWatermanAlign("ACACACTA", "AGCACACA", scoring);
    EXPECT(al.score == 17 && al.alignA == "A-CACACTA" && al.alignB == "AGCACAC-A");
    al = align::SmithWatermanAlign("GATTACA", "GCATGCT", align::NewScoring(&nuc4, -1));
    EXPECT(al.score == 15 && al.alignA == "GATTAC" && al.alignB == "GCATGC");
    al = align::SmithWatermanAlign("", "GAT", scoring);
    EXPECT(al.score == 0 && al.alignA.empty() && al.alignB.empty());
    // TestNeedlemanWunsch scores (align_test.go:11-137)
    auto nws = align::NewScoring(&s5, -1);
    EXPECT(align::NeedlemanWunschScore("GATTACA", "GCATGCU", nws) == 0);
    EXPECT(align::NeedlemanWunschScore("GATTACA", "GATTACA", nws) == 7);
    EXPECT(align::NeedlemanWunschScore("GATTACA", "GAT", nws) == -1);
    EXPECT(align::NeedlemanWunschScore("", "GAT", nws) == -3);
    EXPECT(align::NeedlemanWunschScore("G", "GATTACA", nws) == -5);
    al = align::NeedlemanWunschAlign("GATTACA", "GCATGCU", nws);  // example_test.go:10-47
    EXPECT(al.score == 0 && al.alignA == "G-ATTACA" && al.alignB == "GCA-TGCU");
    bool err = false;
    try { align::SmithWaterman("ACGT", "ACGX", scoring); } catch (const align::AlphabetError &e) { err = std::string(e.what()) == "Symbol X not in alphabet"; }
    EXPECT(err);
}

static void TestSantaLucia() {  // primers_test.go:29-84
    auto t = primers::SantaLucia("ACGATGGCAGTAGCATGC", 0.1e-6, 350e-3, 0.0);
    EXPECT(std::fabs(62.7 - t.meltingTemp) / 62.7 < 0.02);
    t = primers::SantaLucia("ACGTAGATCTACGT", 0.1e-6, 350e-3, 0.0);
    EXPECT(std::fabs(47.428514 - t.meltingTemp) / 47.428514 < 0.02);
    double tm = primers::MeltingTemp("GTAAAACGACGGCCAGT");
    EXPECT(std::fabs(52.8 - tm) / 52.8 < 0.02);
    EXPECT(std::fabs(tm - 52.63382276100299) <= 1e-6 * 52.63382276100299);
    bool panicked = false;
    try { primers::MeltingTemp(""); } catch (const GoPanic &) { panicked = true; }
    EXPECT(panicked);
}

static void TestFastaParser() {  // io/fasta/fasta_test.go:135-170,199-237
    using fasta::Fasta;
    for (bool alias : {true, false}) {
        auto r = fasta::ParseAll(">humen\nGATTACA\nCATGAT", 256, alias);  // EOF-ended Fasta not valid
        EXPECT(r.err_code == 0 && r.fastas.empty());
        r = fasta::ParseAll(">humen\nGATTACA\nCATGAT\n", 256, alias);
        EXPECT(r.err_code == 0 && r.fastas == std::vector<Fasta>({{"humen", "GATTACACATGAT"}}));
        r = fasta::ParseAll(">doggy or something\nGATTACA\n\nCATGAT\n>homunculus\nAAAA\n", 256, alias);
        EXPECT(r.err_code == 0 && r.fastas == std::vector<Fasta>({{"doggy or something", "GATTACACATGAT"}, {"homunculus", "AAAA"}}));
        r = fasta::Parse("testing\natagtagtagtagtagatgatgatgatgagatg\n\n\n\n\n\n\n\n\n\n\n", alias);  // TestReadEmptyFasta
        EXPECT(r.err_code != 0 && r.fastas.empty() && r.error() == "did not find fasta start '>', got to line 13");
        r = fasta::ParseAll(">0\n0123456789ABCDEF\n>1\nCAC\n", 2, alias);  // TestParseBufferFail
        EXPECT(r.err_code == 3);
        r = fasta::ParseAll(">OK Fasta\nABGABA\n>NotOKFasta\n", 2, alias);  // TestParseEOFAfterName
        EXPECT(r.err_code == 2 && r.fastas.size() == 1);
    }
}


static const std::string kGene = "aataattacaccgagataacacatcatggataaaccgatactcaaagattctatgaagctatttgaggcacttggtacgatcaagtcgcgctcaatgtttggtggcttcggacttttcgctgatgaaacgatgtttgcactggttgtgaatgatcaacttcacatacgagcagaccagcaaacttcatctaacttcgagaagcaagggctaaaaccgtacgtttataaaaagcgtggttttccagtcgttactaagtactacgcgatttccgacgacttgtgggaatccagtgaacgcttgatagaagtagcgaagaagtcgttagaacaagccaatttggaaaaaaagcaacaggcaagtagtaagcccgacaggttgaaagacctgcctaacttacgactagcgactgaacgaatgcttaagaaagctggtataaaatcagttgaacaacttgaagagaaaggtgcattgaatgcttacaaagcgatacgtgactctcactccgcaaaagtaagtattgagctactctgggctttagaaggagcgataaacggcacgcactggagcgtcgttcctcaatctcgcagagaagagctggaaaatgcgctttcttaa";
static const std::string kBadFragment = "ATGACCATGATTACGCCAAGCTTGCATGCCTGCAGGTCGACTCTAGAGGATCCCCGGGTACCGAGCTCGAATTCACTGGCCGTCGTTTTACAACGTCGTGACTGGGAAAACCCTGGCGTTACCCAACTTAATCGCCTTGCAGCACATCCCCCTTTCGCCAGCTGGCGTAATAGCGAAGAGGCCCGCACCGATCGCCCTTCCCAACAGTTGCGCAGCCTGAATGGCGAATGGCGCCTGATGCGGTATTTTCTCCTTACGCATCTGTGCGGTATTTCACACCGCATATGGTGCACTCTCAGTACAATCTGCTCTGATGCCGCATAG";
static const std::string kFullAmplicon = "TTATAGGTCTCATACTAATAATTACACCGAGATAACACATCATGGATAAACCGATACTCAAAGATTCTATGAAGCTATTTGAGGCACTTGGTACGATCAAGTCGCGCTCAATGTTTGGTGGCTTCGGACTTTTCGCTGATGAAACGATGTTTGCACTGGTTGTGAATGATCAACTTCACATACGAGCAGACCAGCAAACTTCATCTAACTTCGAGAAGCAAGGGCTAAAACCGTACGTTTATAAAAAGCGTGGTTTTCCAGTCGTTACTAAGTACTACGCGATTTCCGACGACTTGTGGGAATCCAGTGAACGCTTGATAGAAGTAGCGAAGAAGTCGTTAGAACAAGCCAATTTGGAAAAAAAGCAACAGGCAAGTAGTAAGCCCGACAGGTTGAAAGACCTGCCTAACTTACGACTAGCGACTGAACGAATGCTTAAGAAAGCTGGTATAAAATCAGTTGAACAACTTGAAGAGAAAGGTGCATTGAATGCTTACAAAGCGATACGTGACTCTCACTCCGCAAAAGTAAGTATTGAGCTACTCTGGGCTTTAGAAGGAGCGATAAACGGCACGCACTGGAGCGTCGTTCCTCAATCTCGCAGAGAAGAGCTGGAAAATGCGCTTTCTTAAATGAAGAGACCATATA";
static const std::string kCircularTarget = "ACTCTGGGCTTTAGAAGGAGCGATAAACGGCACGCACTGGAGCGTCGTTCCTCAATCTCGCAGAGAAGAGCTGGAAAATGCGCTTTCTTAAAATAATTACACCGAGATAACACATCATGGATAAACCGATACTCAAAGATTCTATGAAGCTATTTGAGGCACTT";

static void TestPcr() {  // primers/pcr/pcr_test.go:12-101, example_test.go:10-69
    using pcr::Simulate;
    // ExampleDesignPrimers / ExampleDesignPrimersWithOverhangs (example_test.go:39-55)
    auto pr = pcr::DesignPrimers(kGene, 55.0);
    EXPECT(pr.first == "AATAATTACACCGAGATAACACATCATGG" && pr.second == "TTAAGAAAGCGCATTTTCCAGC");
    auto po = pcr::DesignPrimersWithOverhangs(kGene, "TTATAGGTCTCATACT", "ATGAAGAGACCATATA", 55.0);
    EXPECT(po.first == "TTATAGGTCTCATACTAATAATTACACCGAGATAACACATCATGG" && po.second == "TATATGGTCTCTTCATTTAAGAAAGCGCATTTTCCAGC");
    // ExampleSimulate / TestIssue279PCRBug
    std::vector<std::string> primers = {po.first, po.second};
    auto sim = Simulate({kGene}, 55.0, false, primers);
    EXPECT(sim.error.empty() && sim.fragments == std::vector<std::string>({kFullAmplicon}));
    // Example_basic: the second template adds nothing
    primers = {po.first, po.second};
    EXPECT(Simulate({kGene, kBadFragment}, 55.0, false, primers).fragments.size() == 1);
    // TestSimulatePrimerRejection: CTGCAGGTCGACTCTAG never reaches the target Tm and is ignored
    primers = {"TATATGGTCTCTTCATTTAAGAAAGCGCATTTTCCAGC", "TTATAGGTCTCATACTAATAATTACACCGAGATAACACATCATGG", "CTGCAGGTCGACTCTAG"};
    EXPECT(Simulate({kGene}, 55.0, false, primers).fragments.size() == 1);
    // TestSimulateMoreThanOneForward
    primers = {"gatactcaaagattctatgaagctatttgaggcacttggtacg", "tatcgctttgtaagcattcaatgcacctttctcttcaagttg", "gtcgttcctcaatctcgcagagaagagctggaaaatg"};
    EXPECT(Simulate({kGene}, 55.0, false, primers).fragments.size() == 1);
    EXPECT(primers[0] == "GATACTCAAAGATTCTATGAAGCTATTTGAGGCACTTGGTACG");  // upper-cased in place, pcr.go:76-78
    // TestSimulateCircular
    primers = {"actctgggctttagaaggagcgataaacggc", "aagtgcctcaaatagcttcatagaatctttgagtatcgg"};
    sim = Simulate({kGene}, 55.0, true, primers);
    EXPECT(!sim.fragments.empty() && sim.fragments[0] == kCircularTarget);
    // TestSimulateConcatemerization
    primers = {"AATAATTACACCGAGATAACACATCATGG", "CCATGATGTGTTATCTCGGTGTAATTATTTTAAGAAAGCGCATTTTCCAGC"};
    EXPECT(Simulate({kGene}, 55.0, false, primers).error == "Concatemerization detected in PCR.");
    // pcr.go:174-178: shorter than minimalPrimerLength (7)
    primers = {po.first, "ACGT"};
    sim = Simulate({kGene}, 55.0, false, primers);
    EXPECT(!sim.hasFragments && sim.error == "Primers are too short.");
    primers = {po.first, "ACGTACG"};  // exactly 7 nt is legal; its whole length stays below the target and it is ignored
    EXPECT(Simulate({kGene}, 55.0, false, primers).error.empty());
    bool panicked = false;
    try { primers = {"ACGT"}; pcr::SimulateSimple({kGene}, 55.0, false, primers); } catch (const GoPanic &) { panicked = true; }
    EXPECT(panicked);
}

static void TestFastqParser() {  // io/fastq/fastq_test.go:8-66 restated on in-line records (the fixtures are not in this repo)
    const std::string two = "@r1 runid=abc ch=7\nACGTTGCA\n+\nIIIIHHHH\n@r2\nGG\n+\n#!\n";
    auto r = fastq::Parse(two);
    EXPECT(r.err_code == 0 && r.fastqs.size() == 2);
    EXPECT(r.fastqs[0].Identifier == "r1" && r.fastqs[0].Optionals.size() == 2 && r.fastqs[0].Optionals["runid"] == "abc" &&
           r.fastqs[0].Optionals["ch"] == "7" && r.fastqs[0].Sequence == "ACGTTGCA" && r.fastqs[0].Quality == "IIIIHHHH");
    EXPECT(r.fastqs[1].Identifier == "r2" && r.fastqs[1].Optionals.empty() && r.fastqs[1].Sequence == "GG" && r.fastqs[1].Quality == "#!");
    r = fastq::Parse("@r1\nACGT\n+\nIIII\n@r2\n\n+\nII\n");  // "empty seq"
    EXPECT(r.fastqs.size() == 1 && r.err_code == 2 && r.err_line == 6 && r.error() == "empty fastq sequence, got to line 6");
    r = fastq::Parse("@r1\nACGT\n+\nIIII\nr2\nAC\n+\nII\n");  // "no identifier": reported after the 4th line of the record
    EXPECT(r.fastqs.size() == 1 && r.err_code == 4 && r.err_line == 8);
    r = fastq::Parse("@r1\nACGT\n+\nIIII\n@r2\nAC\n+\n\n");  // "no quality"
    EXPECT(r.fastqs.size() == 1 && r.err_code == 3 && r.err_line == 8);
    r = fastq::Parse("@r1\nACGT\n+\nIIII\n@r2\nAC\n");  // "no plus EOF"
    EXPECT(r.fastqs.size() == 1 && r.err_code == 1 && r.err_line == 7);
    r = fastq::Parse("");
    EXPECT(r.fastqs.empty() && r.err_code == 0);
}

static void TestSketchPersistenceAndMulti(const char *out_path) {  // SURVEY.md 8f.4 + the *_multi entry points
    const std::string A = "ATGCGATCGATCGATCGATCGATCGATCGATCGATCGATCGATCGATCGATCGATCGATCGA";
    auto m = mash::New(17, 10); m.Sketch(A);
    const std::string js = mash::ToJSON(m);
    EXPECT(js.rfind("{\"KmerSize\":17,\"SketchSize\":10,\"Sketches\":[", 0) == 0 && js.back() == '}' && js.find(' ') == std::string::npos);
    auto back = mash::FromJSON(js);
    EXPECT(back.KmerSize == 17 && back.SketchSize == 10 && back.Sketches == m.Sketches);
    {   // in-place batch form: informative words written, tails left alone (what Sketch does to an existing Mash)
        const std::vector<std::string> seqs = {A, A.substr(0, 20), A.substr(3), std::string()};
        std::vector<uint32_t> slab(seqs.size() * 50, 0xDEADBEEFu);
        auto cnt = mash::SketchInto(seqs, 17, 50, slab);
        for (size_t i = 0; i < seqs.size(); ++i) {
            auto one = mash::New(17, 50); one.Sketch(seqs[i]);
            const uint32_t c = (uint32_t)std::min<size_t>(seqs[i].size() > 17 ? seqs[i].size() - 17 : 0, 50);
            EXPECT(cnt[i] == c);
            for (uint32_t j = 0; j < 50; ++j) EXPECT(slab[i * 50 + j] == (j < c ? one.Sketches[j] : 0xDEADBEEFu));
        }
    }
    EXPECT(mash::FromJSON("{\"KmerSize\":3,\"SketchSize\":2,\"Sketches\":null}").Sketches.empty());
    // a set: fill-regime (compact) and select-regime rows together
    std::vector<std::string> reads;
    std::string flat;
    for (int i = 0; i < 40; ++i) {
        std::string r(300, 'A');
        uint64_t x = 0x9E3779B97F4A7C15ull * (uint64_t)(i / 4 + 1);
        for (int j = 0; j < 300; ++j) {
            x ^= x << 13; x ^= x >> 7; x ^= x << 17;
            r[j] = "ACGT"[(x >> 11) & 3];
        }
        if (i % 4) r[17 * (i % 4)] = 'N';  // family of 4: three mutated copies
        reads.push_back(r);
        flat += r;
    }
    auto batch = mash::SketchBatch(reads, 21, 64);                 // sharded over every visible GPU
    auto one_gpu = mash::SketchBatch(reads, 21, 64, {0});
    for (size_t i = 0; i < reads.size(); ++i) {
        auto single = mash::New(21, 64); single.Sketch(reads[i]);
        EXPECT(batch[i].Sketches == single.Sketches && one_gpu[i].Sketches == single.Sketches);
    }
    mash::SketchSet set;
    set.KmerSize = 21; set.SketchSize = 64;
    for (auto &b : batch) set.rows.push_back(b.Sketches);
    set.rows.push_back({1u, 2u, 3u});                              // a compact (fill-regime) row: 3 informative words
    auto blob = mash::EncodeSketchSet(set);
    auto dec = mash::DecodeSketchSet(blob);
    EXPECT(dec.KmerSize == 21 && dec.SketchSize == 64 && dec.rows == set.rows && dec.count.back() == 3);
    blob[50] ^= 1;
    bool rejected = false;
    try { mash::DecodeSketchSet(blob); } catch (const std::invalid_argument &) { rejected = true; }
    EXPECT(rejected);
    if (out_path) mash::SaveSketchSet(out_path, set);             // read back by the Python implementation in the pytest
    // fused sketch + all-gather + row-block distance on all GPUs == per-pair API
    auto sd = mash::SketchDistanceMulti(flat, reads.size(), 300, 21, 64);
    const size_t n = reads.size();
    bool ok = true;
    for (size_t i = 0; i < n; ++i) {
        ok = ok && std::equal(batch[i].Sketches.begin(), batch[i].Sketches.end(), sd.sketches.begin() + i * 64);
        for (size_t j = 0; j < n; j += 3) {
            auto p = batch[i].pair(batch[j]);
            ok = ok && (int64_t)sd.same[i * n + j] == p.same && sd.distance[i * n + j] == p.distance;
        }
    }
    EXPECT(ok);
    EXPECT(sd.same[0 * n + 1] > 0 && sd.same[0 * n + 4] == 0);     // same family shares hashes, another family does not
}

int main(int argc, char **argv) {
    check(pg_init(0));
    TestFastaParser();
    TestFastqParser();
    TestMash();
    TestSmithWaterman();
    TestSantaLucia();
    TestPcr();
    TestSketchPersistenceAndMulti(argc > 1 ? argv[1] : nullptr);
    std::printf(failures ? "FAILED (%d)\n" : "ok: reference tests pass through the C++ host mirror\n", failures);
    return failures ? 1 : 0;
}
