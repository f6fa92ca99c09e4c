// seqhash_tests.cpp -- seqhash_test.go and example_test.go (seqhash/) restated against the C++ host mirror.
// Usage: seqhash_tests PUC19.txt  (the pUC19 sequence, as genbank.Read returns it from data/puc19.gbk)
// Prints "ok: seqhash tests pass" when every check holds.
#include <cstdio>
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
        std::printf("FAIL: usage: seqhash_tests PUC19.txt\n");
        return 1;
    }
    // TestHash (seqhash_test.go:12-65)
    expect(!seqhash::Hash("ATGGGCTAA", "TNA", true, true).second.empty(), "TNA is not a valid sequenceType");
    expect(!seqhash::Hash("XTGGCCTAA", seqhash::DNA, true, true).second.empty(), "X is not a valid DNA letter");
    expect(!seqhash::Hash("MGCJ*", seqhash::PROTEIN, false, false).second.empty(), "J is not a valid protein letter");
    expect(!seqhash::Hash("MGCS*", seqhash::PROTEIN, false, true).second.empty(), "proteins cannot be double stranded");
    const struct {
        const char *seq, *type;
        bool circular, ds;
        const char *want;
    } pins[] = {
        {"TTAGCCCAT", "DNA", true, true, "v1_DCD_a376845b679740014f3eb501429b45e592ecc32a6ba8ba922cbe99217f6e9287"},
        {"TTAGCCCAT", "DNA", true, false, "v1_DCS_ef79b6e62394e22a176942dfc6a5e62eeef7b5281ffcb2686ecde208ec836ba4"},
        {"TTAGCCCAT", "DNA", false, true, "v1_DLD_c2c9fc44df72035082a152e94b04492182331bc3be2f62729d203e072211bdbf"},
        {"TTAGCCCAT", "DNA", false, false, "v1_DLS_063ea37d1154351639f9a48546bdae62fd8a3c18f3d3d3061060c9a55352d967"},
        {"TTAGCCCAT", "RNA", false, false, "v1_RLS_063ea37d1154351639f9a48546bdae62fd8a3c18f3d3d3061060c9a55352d967"},
        {"MGC*", "PROTEIN", false, false, "v1_PLS_922ec11f5227ce77a42f07f565a7a1a479772b5cf3f1f6e93afc5ecbc0fd5955"},
        // Example_basic / ExampleHash (example_test.go:11-31)
        {"ATGC", "DNA", false, true, "v1_DLD_f4028f93e08c5c23cbb8daa189b0a9802b378f1a1c919dcbcf1608a615f46350"},
    };
    for (auto &p : pins) {
        const auto got = seqhash::Hash(p.seq, p.type, p.circular, p.ds);
        expect(got.first == p.want && got.second.empty(), std::string("pin ") + p.want + " got " + got.first + got.second);
    }
    // TestLeastRotation (seqhash_test.go:67-91): every rotation of pUC19 rotates to one string, in one call
    std::ifstream in(argv[1]);
    std::stringstream ss;
    ss << in.rdbuf();
    std::string puc = ss.str();
    while (!puc.empty() && (puc.back() == '\n' || puc.back() == '\r')) puc.pop_back();
    expect(puc.size() == 2686, "pUC19 length");
    std::vector<std::string> rots;
    for (size_t r = 0; r < puc.size(); ++r) rots.push_back(puc.substr(r) + puc.substr(0, r));
    const auto rotated = seqhash::RotateSequences(rots);
    bool same = true;
    for (auto &r : rotated) same = same && r == rotated[0];
    expect(same, "every rotation of pUC19 gives one rotated sequence");
    // ExampleRotateSequence (example_test.go:33-40)
    const size_t half = puc.size() / 2;
    expect(seqhash::RotateSequence(puc) == seqhash::RotateSequence(puc.substr(half) + puc.substr(0, half)), "ExampleRotateSequence");
    // the package doc's example hash (seqhash.go:46) is pUC19's
    expect(seqhash::Hash(puc, seqhash::DNA, true, true).first == "v1_DCD_4b0616d1b3fc632e42d78521deb38b44fba95cca9fde159e01cd567fa996ceb9",
           "pUC19 Seqhash");
    if (failures) return 1;
    std::printf("ok: seqhash tests pass\n");
    return 0;
}
