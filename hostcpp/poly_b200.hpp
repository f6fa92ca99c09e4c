// poly_b200.hpp -- header-only C++ host mirror of the reference's Go API for the hot path,
// over the C ABI of libpolyb200.so (include/poly_b200.h).
//
// The reference is Go (compiled code) and no Go toolchain exists in this image, so the host
// side above the C ABI is written in C++ with the reference's names, argument meaning and
// failure behaviour:
//   poly::mash::New / Mash{KmerSize,SketchSize,Sketches} / Sketch / Similarity / Distance
//        <- /root/reference/search/mash/mash.go:52-140
//   poly::align::NewAlphabet / NewSubstitutionMatrix / NewScoring / SmithWaterman (score)
//        <- alphabet/alphabet.go:25-41, search/align/matrix/matrix.go:13-38,
//           search/align/align.go:73-95,171-203
//   poly::primers::SantaLucia / MeltingTemp <- primers/primers.go:70-105,121-128
//   poly::fasta::Parse / ParseAll            <- io/fasta/fasta.go:72-77,89-118,149-243
//   poly::pcr::DesignPrimers* / SimulateSimple / Simulate <- primers/pcr/pcr.go:44-186
//   poly::mash::ToJSON / FromJSON (the encoding/json shape of mash.Mash) and the PGSKETCH container
//   poly::seqhash::Hash / HashBatch / RotateSequence <- seqhash/seqhash.go:78-223
// A Go panic surfaces as poly::GoPanic; align's alphabet.Error as poly::align::AlphabetError.
// The Go package in go/ (cgo) is the real drop-in; this header is what the tests in this
// repository can compile and run (tests/test_gpu_hostcpp.py).  No compute happens here.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <limits>
#include <map>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "../include/poly_b200.h"

namespace poly {

struct GoPanic : std::runtime_error {
    using std::runtime_error::runtime_error;
};
struct Error : std::runtime_error {
    int code;
    Error(int c, const std::string &m) : std::runtime_error(m), code(c) {}
};
inline void check(int rc) {
    if (rc != PG_OK) throw Error(rc, std::string("libpolyb200: ") + pg_last_error());
}

// []string -> bytes + offsets (what the cgo shim does before crossing the ABI)
struct Flat {
    std::vector<uint8_t> bases;
    std::vector<uint64_t> offsets;
    explicit Flat(const std::vector<std::string> &seqs) {
        offsets.reserve(seqs.size() + 1);
        offsets.push_back(0);
        size_t total = 0;
        for (auto &s : seqs) total += s.size();
        bases.reserve(total);
        for (auto &s : seqs) {
            bases.insert(bases.end(), s.begin(), s.end());
            offsets.push_back(bases.size());
        }
    }
};

namespace mash {

// mash.Mash, mash.go:52-56
struct Mash {
    int KmerSize;
    int SketchSize;
    std::vector<uint32_t> Sketches;

    // (*Mash).Sketch, mash.go:68-104 (mutates the receiver)
    void Sketch(const std::string &sequence) {
        const int64_t n = (int64_t)sequence.size() - KmerSize;
        if (n <= 0) return;
        if (KmerSize < 0) throw GoPanic("slice bounds out of range");
        const uint64_t cnt = (uint64_t)std::min<int64_t>(n, SketchSize);
        std::vector<uint32_t> out(cnt ? cnt : 1);
        int32_t status = 0;
        int rc = pg_mash_sketch_uniform(reinterpret_cast<const uint8_t *>(sequence.data()), 1, (uint32_t)sequence.size(),
                                        KmerSize, SketchSize, 0, out.data(), cnt, &status);
        if (rc == PG_ERR_PANIC || status == PG_ITEM_PANIC) throw GoPanic("index out of range [-1]");  // mash.go:96-98
        check(rc);
        for (uint64_t i = 0; i < cnt; ++i) Sketches[i] = out[i];  // n < s: the tail is left untouched (mash.go:81-84)
    }

    struct Pair { int64_t same; double similarity, distance; };
    Pair pair(const Mash &other) const {
        if ((int)Sketches.size() < SketchSize || (int)other.Sketches.size() < other.SketchSize) throw GoPanic("index out of range");
        std::vector<uint32_t> sk(Sketches.begin(), Sketches.begin() + SketchSize);
        sk.insert(sk.end(), other.Sketches.begin(), other.Sketches.begin() + other.SketchSize);
        const uint64_t off[3] = {0, (uint64_t)SketchSize, (uint64_t)SketchSize + (uint64_t)other.SketchSize};
        const uint32_t a = 0, b = 1;
        Pair p{};
        int32_t st = 0;
        int rc = pg_mash_similarity_pairs(sk.data(), off, 2, &a, &b, 1, &p.same, &p.similarity, &p.distance, &st);
        if (rc == PG_ERR_PANIC) throw GoPanic("index out of range [-1]");
        check(rc);
        return p;
    }
    double Similarity(const Mash &other) const { return pair(other).similarity; }  // mash.go:107-135
    double Distance(const Mash &other) const { return pair(other).distance; }      // mash.go:138-140
};

// mash.New, mash.go:59-65
inline Mash New(int kmerSize, int sketchSize) {
    if (sketchSize < 0) throw GoPanic("makeslice: len out of range");
    return Mash{kmerSize, sketchSize, std::vector<uint32_t>((size_t)sketchSize, 0u)};
}

// batched addition: []string -> []Mash, each == New(k, s) + Sketch(seq).  One call, sharded over the
// GPUs of this process (devices empty: every visible GPU; reads are independent, mash.go:68-104).
inline std::vector<Mash> SketchBatch(const std::vector<std::string> &seqs, int k, int s, const std::vector<int32_t> &devices = {}) {
    Flat f(seqs);
    size_t maxlen = 0;
    for (auto &q : seqs) maxlen = std::max(maxlen, q.size());
    const uint64_t stride = std::max<int64_t>(1, std::min<int64_t>((int64_t)maxlen - k, s));
    std::vector<uint32_t> out(seqs.size() * stride), count(seqs.size());
    std::vector<int32_t> status(seqs.size());
    int rc = pg_mash_sketch_batch_multi(f.bases.data(), f.offsets.data(), seqs.size(), k, s, 0, out.data(), stride, count.data(), status.data(),
                                        devices.empty() ? nullptr : devices.data(), (int32_t)devices.size());
    if (rc != PG_OK && rc != PG_ERR_PANIC) check(rc);
    std::vector<Mash> res;
    res.reserve(seqs.size());
    for (size_t i = 0; i < seqs.size(); ++i) {
        if (status[i] == PG_ITEM_PANIC) throw GoPanic("index out of range [-1]");
        Mash m = New(k, s);
        for (uint32_t j = 0; j < count[i]; ++j) m.Sketches[j] = out[i * stride + j];
        res.push_back(std::move(m));
    }
    return res;
}

// One Mash per group of sequences (an assembly's contigs, a sample's reads): the smallest s distinct window hashes of
// the group seen at least minCopies times, ascending, then a zero tail (`mash sketch`, `mash sketch -r -m`).  Windows
// never cross a sequence.  count (may be null) receives how many values each group holds.  canonical hashes canonical
// k-mers (PG_KMER_CANONICAL: windows 0 .. L - k, each the smaller of itself and its reverse complement).
inline std::vector<Mash> SketchGroups(const std::vector<std::vector<std::string>> &groups, int k, int s, uint32_t minCopies,
                                      std::vector<uint32_t> *count = nullptr, bool canonical = false) {
    std::vector<std::string> seqs;
    std::vector<uint64_t> goff(1, 0);
    for (const auto &g : groups) {
        seqs.insert(seqs.end(), g.begin(), g.end());
        goff.push_back(seqs.size());
    }
    Flat f(seqs);
    const uint64_t stride = (uint64_t)std::max(s, 1);
    std::vector<uint32_t> out(groups.size() * stride), cnt(groups.size());
    check(pg_mash_sketch_groups_flags(f.bases.data(), f.offsets.data(), seqs.size(), goff.data(), groups.size(), k, s, minCopies,
                                      canonical ? PG_KMER_CANONICAL : 0u, out.data(), stride, cnt.data()));
    std::vector<Mash> res;
    res.reserve(groups.size());
    for (size_t g = 0; g < groups.size(); ++g)
        res.push_back(Mash{k, s, std::vector<uint32_t>(out.begin() + g * stride, out.begin() + (g + 1) * stride)});
    if (count) *count = cnt;
    return res;
}

// Grouped sketches grown in place (pg_mash_sketcher): nGroups sketches fed batch by batch, each add counting its
// sequences into one group or a run of groups.  A row is complete when it holds s values or the group's cap is still
// 2^32; a complete row equals SketchGroups over every sequence added to the group, whatever the split, and every row
// is a prefix of it.  maxValues (0: 64 s) is the most distinct values a group keeps between adds.  canonical counts
// canonical k-mers, as SketchGroups(..., canonical = true).
class Sketcher {
public:
    Sketcher(uint64_t nGroups, int k, int s, uint32_t minCopies, uint64_t maxValues = 0, bool canonical = false) : k_(k), s_(s), n_(nGroups) {
        check(pg_mash_sketcher_create_flags(nGroups, k, s, minCopies, maxValues ? maxValues : 64 * (uint64_t)std::max(s, 1),
                                            canonical ? PG_KMER_CANONICAL : 0u, &h_));
    }
    Sketcher(const Sketcher &) = delete;
    Sketcher &operator=(const Sketcher &) = delete;
    ~Sketcher() { pg_mash_sketcher_free(h_); }
    // sequences of groups [firstGroup, firstGroup + groups.size()), groups[i] going to group firstGroup + i
    void Add(const std::vector<std::vector<std::string>> &groups, uint64_t firstGroup = 0) {
        std::vector<std::string> seqs;
        std::vector<uint64_t> goff(1, 0);
        for (const auto &g : groups) {
            seqs.insert(seqs.end(), g.begin(), g.end());
            goff.push_back(seqs.size());
        }
        Flat f(seqs);
        check(pg_mash_sketcher_add(h_, f.bases.data(), f.offsets.data(), seqs.size(), goff.data(), firstGroup, groups.size()));
    }
    void AddRecords(uint64_t group, const std::vector<std::string> &seqs) { Add({seqs}, group); }
    // one Mash per group; count, complete and held (each may be null) receive the row sizes, whether each row is
    // complete, and the values each group holds
    std::vector<Mash> Sketches(std::vector<uint32_t> *count = nullptr, std::vector<uint8_t> *complete = nullptr,
                               std::vector<uint64_t> *held = nullptr) const {
        std::vector<uint32_t> out(n_ * s_), cnt(n_);
        std::vector<uint8_t> c(n_);
        std::vector<uint64_t> h(n_);
        check(pg_mash_sketcher_rows(h_, 0, n_, out.data(), s_, cnt.data(), c.data(), h.data()));
        std::vector<Mash> res;
        res.reserve(n_);
        for (uint64_t g = 0; g < n_; ++g) res.push_back(Mash{k_, s_, std::vector<uint32_t>(out.begin() + g * s_, out.begin() + (g + 1) * s_)});
        if (count) *count = cnt;
        if (complete) *complete = c;
        if (held) *held = h;
        return res;
    }

private:
    pg_mash_sketcher *h_ = nullptr;
    int k_, s_;
    uint64_t n_;
};

// Mash distance between grouped sketches (`mash dist`): queries and refs as SketchGroups / Sketcher::Sketches return
// them, with their counts; one SketchSize for all.  Outputs are nq x nr, row-major, query = row: common and denom from
// Mash's compareSketches (denom = min(s, |A u B|), common = shared values among the denom smallest of A u B), distance =
// -ln(2J / (1 + J)) / k, and p = Mash's p-value from the genome lengths (bases per sketch, >= 1).  Without lengths
// (both empty) pValue stays empty.
struct DistResult {
    std::vector<uint32_t> common, denom;
    std::vector<double> distance, pValue;
};
// the pairs with distance <= maxDistance and p <= maxPValue (upper: r > q only, for a set against itself), sorted by (q, r)
struct DistPairs {
    std::vector<uint32_t> q, r, common, denom;
    std::vector<double> distance, pValue;
};
namespace detail {
inline int dist_slab(const std::vector<Mash> &set, const std::vector<uint32_t> &count, int s, std::vector<uint32_t> &rows) {
    if (count.size() != set.size()) throw std::invalid_argument("one count per sketch");
    rows.assign(set.size() * (size_t)std::max(s, 1), 0);
    for (size_t i = 0; i < set.size(); ++i) {
        if (set[i].SketchSize != s || (int)set[i].Sketches.size() < s) throw std::invalid_argument("sketches of one SketchSize");
        std::copy(set[i].Sketches.begin(), set[i].Sketches.begin() + s, rows.begin() + i * (size_t)s);
    }
    return s;
}
inline int dist_size(const std::vector<Mash> &q, const std::vector<Mash> &r) {
    return !q.empty() ? q[0].SketchSize : !r.empty() ? r[0].SketchSize : 1;
}
inline void dist_lengths(const std::vector<uint64_t> &qLen, const std::vector<uint64_t> &rLen, size_t nq, size_t nr) {
    if (qLen.empty() != rLen.empty()) throw std::invalid_argument("pass both length vectors, or neither");
    if (!qLen.empty() && (qLen.size() != nq || rLen.size() != nr)) throw std::invalid_argument("one length per sketch");
}
}  // namespace detail

inline DistResult Dist(const std::vector<Mash> &queries, const std::vector<uint32_t> &qCount, const std::vector<Mash> &refs,
                       const std::vector<uint32_t> &rCount, int k, const std::vector<uint64_t> &qLen = {}, const std::vector<uint64_t> &rLen = {}) {
    const int s = detail::dist_size(queries, refs);
    std::vector<uint32_t> q, r;
    detail::dist_slab(queries, qCount, s, q);
    detail::dist_slab(refs, rCount, s, r);
    detail::dist_lengths(qLen, rLen, queries.size(), refs.size());
    const size_t n = queries.size() * refs.size();
    DistResult out{std::vector<uint32_t>(n), std::vector<uint32_t>(n), std::vector<double>(n), std::vector<double>(qLen.empty() ? 0 : n)};
    check(pg_mash_dist(q.data(), qCount.data(), queries.size(), r.data(), rCount.data(), refs.size(), (uint64_t)s, s, k,
                       qLen.empty() ? nullptr : qLen.data(), rLen.empty() ? nullptr : rLen.data(), out.common.data(), out.denom.data(),
                       out.distance.data(), qLen.empty() ? nullptr : out.pValue.data()));
    return out;
}

inline DistPairs DistWithin(const std::vector<Mash> &queries, const std::vector<uint32_t> &qCount, const std::vector<Mash> &refs,
                            const std::vector<uint32_t> &rCount, int k, const std::vector<uint64_t> &qLen = {}, const std::vector<uint64_t> &rLen = {},
                            double maxDistance = 1.0, double maxPValue = 1.0, bool upper = false) {
    const int s = detail::dist_size(queries, refs);
    std::vector<uint32_t> q, r;
    detail::dist_slab(queries, qCount, s, q);
    detail::dist_slab(refs, rCount, s, r);
    detail::dist_lengths(qLen, rLen, queries.size(), refs.size());
    const bool p = !qLen.empty();
    uint64_t cap = std::max<uint64_t>(1024, 4 * queries.size()), n = 0;
    DistPairs out;
    for (;;) {
        out = DistPairs{std::vector<uint32_t>(cap), std::vector<uint32_t>(cap), std::vector<uint32_t>(cap), std::vector<uint32_t>(cap),
                        std::vector<double>(cap), std::vector<double>(p ? cap : 0)};
        const int rc = pg_mash_dist_within(q.data(), qCount.data(), queries.size(), r.data(), rCount.data(), refs.size(), (uint64_t)s, s, k,
                                           p ? qLen.data() : nullptr, p ? rLen.data() : nullptr, maxDistance, maxPValue, upper ? PG_PAIRS_UPPER : 0u,
                                           out.q.data(), out.r.data(), out.common.data(), out.denom.data(), out.distance.data(),
                                           p ? out.pValue.data() : nullptr, cap, &n);
        if (rc == PG_ERR_ARG && n > cap) { cap = n; continue; }
        check(rc);
        break;
    }
    std::vector<size_t> order(n);
    for (size_t i = 0; i < n; ++i) order[i] = i;
    std::sort(order.begin(), order.end(), [&](size_t a, size_t b) { return out.q[a] != out.q[b] ? out.q[a] < out.q[b] : out.r[a] < out.r[b]; });
    DistPairs sorted;
    for (size_t i : order) {
        sorted.q.push_back(out.q[i]); sorted.r.push_back(out.r[i]); sorted.common.push_back(out.common[i]); sorted.denom.push_back(out.denom[i]);
        sorted.distance.push_back(out.distance[i]);
        if (p) sorted.pValue.push_back(out.pValue[i]);
    }
    return sorted;
}

// In-place form: `slab` holds the Sketches arrays of seqs.size() Mash values back to back (n x s words).  Row i
// receives its min(len_i - k, s) words, the rest of the row is left as it is -- what (*Mash).Sketch does to an
// existing Mash (mash.go:73-80); a zeroed slab ends up as n fresh sketches.  Returns the per-read counts.
inline std::vector<uint32_t> SketchInto(const std::vector<std::string> &seqs, int k, int s, std::vector<uint32_t> &slab,
                                        const std::vector<int32_t> &devices = {}) {
    Flat f(seqs);
    if (slab.size() < seqs.size() * (size_t)std::max(s, 0)) throw std::invalid_argument("slab smaller than n x s");
    std::vector<uint32_t> count(seqs.size());
    std::vector<int32_t> status(seqs.size());
    uint32_t dummy = 0;
    int rc = pg_mash_sketch_batch_multi(f.bases.data(), f.offsets.data(), seqs.size(), k, s, PG_SKETCH_TAIL_KEEP,
                                        slab.empty() ? &dummy : slab.data(), (uint64_t)std::max(s, 0), count.data(), status.data(),
                                        devices.empty() ? nullptr : devices.data(), (int32_t)devices.size());
    if (rc != PG_OK && rc != PG_ERR_PANIC) check(rc);
    for (int32_t st : status)
        if (st == PG_ITEM_PANIC) throw GoPanic("index out of range [-1]");
    return count;
}

// batched addition: sketches of fixed-length reads + the all-pairs matrix on several GPUs of this process
// (sketch kernels store into every device's gathered buffer: fused all-gather; device r computes row block r)
struct SketchDistance {
    std::vector<uint32_t> sketches;  // n x s, full Go arrays
    std::vector<uint32_t> same;      // n x n matching counts, receiver = row
    std::vector<double> distance;    // n x n, 1 - same/s (mash.go:134,139)
};
inline SketchDistance SketchDistanceMulti(const std::string &reads, uint64_t n, uint32_t readLen, int k, int s,
                                          const std::vector<int32_t> &devices = {}) {
    SketchDistance r;
    r.sketches.resize(n * (uint64_t)s);
    r.same.resize(n * n);
    r.distance.resize(n * n);
    int rc = pg_mash_sketch_distance_multi(reinterpret_cast<const uint8_t *>(reads.data()), n, readLen, k, s,
                                           devices.empty() ? nullptr : devices.data(), (int32_t)devices.size(), r.sketches.data(), r.same.data(),
                                           r.distance.data());
    if (rc == PG_ERR_PANIC) throw GoPanic("index out of range [-1]");
    check(rc);
    return r;
}

// ---- sketch persistence (SURVEY.md 8f.4) -----------------------------------------------------------
// encoding/json of mash.Mash (mash.go:52-56): exported fields in declaration order, no spaces -- byte for
// byte what Go's json.Marshal emits, so single sketches interoperate with the reference.
inline std::string ToJSON(const Mash &m) {
    std::string out = "{\"KmerSize\":" + std::to_string(m.KmerSize) + ",\"SketchSize\":" + std::to_string(m.SketchSize) + ",\"Sketches\":";
    if (m.Sketches.empty() && m.SketchSize != 0) return out + "null}";  // nil slice
    out += "[";
    for (size_t i = 0; i < m.Sketches.size(); ++i) out += (i ? "," : "") + std::to_string(m.Sketches[i]);
    return out + "]}";
}
inline Mash FromJSON(const std::string &text) {
    auto number_after = [&](const char *key) -> long long {
        const size_t p = text.find(key);
        if (p == std::string::npos) throw std::invalid_argument(std::string("missing ") + key);
        return std::stoll(text.substr(p + std::strlen(key)));
    };
    Mash m{(int)number_after("\"KmerSize\":"), (int)number_after("\"SketchSize\":"), {}};
    size_t p = text.find("\"Sketches\":");
    if (p == std::string::npos) throw std::invalid_argument("missing Sketches");
    p += 11;
    if (text.compare(p, 4, "null") == 0) return m;
    if (text[p] != '[') throw std::invalid_argument("Sketches is not an array");
    ++p;
    while (p < text.size() && text[p] != ']') {
        size_t used = 0;
        m.Sketches.push_back((uint32_t)std::stoull(text.substr(p), &used));
        p += used;
        if (p < text.size() && text[p] == ',') ++p;
    }
    return m;
}

// PGSKETCH v1 container for sketch SETS (layout: poly_b200/sketchfile.py; little endian):
//   "PGSKETCH" | version 1 | KmerSize | SketchSize | flags (bit 0: dense) | n (u64) | words (u64) |
//   count[n] (absent when dense) | the informative words of sketch 0, 1, ... | CRC-32 of everything before
struct SketchSet {
    int KmerSize = 0, SketchSize = 0;
    std::vector<uint32_t> count;               // informative words per sketch
    std::vector<std::vector<uint32_t>> rows;   // rows[i].size() == count[i]
};
namespace detail {
inline uint32_t crc32(const uint8_t *p, size_t n, uint32_t crc = 0) {  // zlib's CRC-32 (reflected 0xEDB88320)
    static uint32_t table[256];
    static bool init = false;
    if (!init) {
        for (uint32_t i = 0; i < 256; ++i) {
            uint32_t c = i;
            for (int k = 0; k < 8; ++k) c = (c & 1) ? 0xEDB88320u ^ (c >> 1) : c >> 1;
            table[i] = c;
        }
        init = true;
    }
    crc = ~crc;
    for (size_t i = 0; i < n; ++i) crc = table[(crc ^ p[i]) & 0xff] ^ (crc >> 8);
    return ~crc;
}
template <typename T>
inline void put(std::vector<uint8_t> &b, T v) {
    for (size_t i = 0; i < sizeof(T); ++i) b.push_back((uint8_t)(v >> (8 * i)));
}
template <typename T>
inline T get(const std::vector<uint8_t> &b, size_t &pos) {
    if (pos + sizeof(T) > b.size()) throw std::invalid_argument("truncated sketch file");
    T v = 0;
    for (size_t i = 0; i < sizeof(T); ++i) v |= (T)b[pos + i] << (8 * i);
    pos += sizeof(T);
    return v;
}
}  // namespace detail
inline std::vector<uint8_t> EncodeSketchSet(const SketchSet &set) {
    std::vector<uint8_t> b;
    const uint64_t n = set.rows.size();
    bool dense = n > 0;
    uint64_t words = 0;
    for (auto &r : set.rows) { dense = dense && (int)r.size() == set.SketchSize; words += r.size(); }
    b.insert(b.end(), {'P', 'G', 'S', 'K', 'E', 'T', 'C', 'H'});
    detail::put<uint32_t>(b, 1);
    detail::put<uint32_t>(b, (uint32_t)set.KmerSize);
    detail::put<uint32_t>(b, (uint32_t)set.SketchSize);
    detail::put<uint32_t>(b, dense ? 1u : 0u);
    detail::put<uint64_t>(b, n);
    detail::put<uint64_t>(b, words);
    if (!dense)
        for (auto &r : set.rows) detail::put<uint32_t>(b, (uint32_t)r.size());
    for (auto &r : set.rows)
        for (uint32_t w : r) detail::put<uint32_t>(b, w);
    detail::put<uint32_t>(b, detail::crc32(b.data(), b.size()));
    return b;
}
inline SketchSet DecodeSketchSet(const std::vector<uint8_t> &b) {
    if (b.size() < 44 || std::memcmp(b.data(), "PGSKETCH", 8) != 0) throw std::invalid_argument("not a PGSKETCH file");
    size_t tail = b.size() - 4, pos = 8;
    if (detail::crc32(b.data(), tail) != detail::get<uint32_t>(b, tail)) throw std::invalid_argument("sketch file checksum mismatch");
    if (detail::get<uint32_t>(b, pos) != 1) throw std::invalid_argument("not a PGSKETCH v1 file");
    SketchSet set;
    set.KmerSize = (int)detail::get<uint32_t>(b, pos);
    set.SketchSize = (int)detail::get<uint32_t>(b, pos);
    const uint32_t flags = detail::get<uint32_t>(b, pos);
    const uint64_t n = detail::get<uint64_t>(b, pos), words = detail::get<uint64_t>(b, pos);
    set.count.assign(n, (uint32_t)set.SketchSize);
    if (!(flags & 1u))
        for (uint64_t i = 0; i < n; ++i) set.count[i] = detail::get<uint32_t>(b, pos);
    uint64_t total = 0;
    for (uint32_t c : set.count) total += c;
    if (total != words || pos + 4 * words + 4 != b.size()) throw std::invalid_argument("sketch file is inconsistent");
    set.rows.resize(n);
    for (uint64_t i = 0; i < n; ++i) {
        set.rows[i].resize(set.count[i]);
        for (uint32_t j = 0; j < set.count[i]; ++j) set.rows[i][j] = detail::get<uint32_t>(b, pos);
    }
    return set;
}
inline void SaveSketchSet(const std::string &path, const SketchSet &set) {
    auto b = EncodeSketchSet(set);
    FILE *f = std::fopen(path.c_str(), "wb");
    if (!f || std::fwrite(b.data(), 1, b.size(), f) != b.size()) { if (f) std::fclose(f); throw std::runtime_error("cannot write " + path); }
    std::fclose(f);
}
inline SketchSet LoadSketchSet(const std::string &path) {
    FILE *f = std::fopen(path.c_str(), "rb");
    if (!f) throw std::runtime_error("cannot read " + path);
    std::vector<uint8_t> b;
    uint8_t buf[65536];
    for (size_t got; (got = std::fread(buf, 1, sizeof buf, f)) > 0;) b.insert(b.end(), buf, buf + got);
    std::fclose(f);
    return DecodeSketchSet(b);
}
// the set as Mash values (zero tail of a fresh Mash re-materialised)
inline std::vector<Mash> MashesOf(const SketchSet &set) {
    std::vector<Mash> out;
    for (auto &r : set.rows) {
        Mash m = New(set.KmerSize, set.SketchSize);
        std::copy(r.begin(), r.end(), m.Sketches.begin());
        out.push_back(std::move(m));
    }
    return out;
}

namespace detail {
// The n x s rows of mashes of one SketchSize s (0 for none) as the C ABI takes them; `what` names the set in the error.
inline std::vector<uint32_t> FlatRows(const std::vector<Mash> &mashes, const char *what, int *s) {
    *s = mashes.empty() ? 0 : mashes[0].SketchSize;
    std::vector<uint32_t> flat;
    flat.reserve(mashes.size() * (size_t)std::max(*s, 0));
    for (auto &m : mashes) {
        if (m.SketchSize != *s || (int)m.Sketches.size() < *s) throw std::invalid_argument(std::string(what) + " must share one SketchSize");
        flat.insert(flat.end(), m.Sketches.begin(), m.Sketches.begin() + *s);
    }
    return flat;
}
}  // namespace detail

// ---- sketch index: top-k nearest references (pg_mash_index_*) ----------------------------------------
// One reference of a query's result: refs[Ref], its matching count as queries[q].Similarity(refs[Ref]) counts it
// (the query is the receiver, mash.go:107-135), and queries[q].Distance(refs[Ref]).
struct Neighbor {
    uint32_t Ref;
    uint32_t Same;
    double Distance;
};
// RAII owner of a device-resident index over a reference set of one SketchSize (the library copies the sketches).
class Index {
    pg_mash_index *h_ = nullptr;
    int s_ = 0;

public:
    explicit Index(const std::vector<Mash> &refs) {
        const std::vector<uint32_t> flat = detail::FlatRows(refs, "references", &s_);
        int rc = pg_mash_index_create(flat.data(), refs.size(), s_, &h_);
        if (rc == PG_ERR_PANIC) throw GoPanic("index out of range [-1]");
        check(rc);
    }
    Index(const Index &) = delete;
    Index &operator=(const Index &) = delete;
    ~Index() { pg_mash_index_free(h_); }
    // Appends references on the device: they take the next ids, and later queries answer as an index built over
    // the whole set would.  An empty index takes the batch's SketchSize.
    void Add(const std::vector<Mash> &refs) {
        int s;
        const std::vector<uint32_t> flat = detail::FlatRows(refs, "references", &s);
        int rc = pg_mash_index_add(h_, flat.data(), refs.size(), s);
        if (rc == PG_ERR_PANIC) throw GoPanic("index out of range [-1]");
        check(rc);
    }
    // For each query, up to k references with Same >= minSame, by Same descending and then Ref ascending.
    std::vector<std::vector<Neighbor>> Nearest(const std::vector<Mash> &queries, uint32_t k, uint32_t minSame = 1) const {
        int sq;
        const std::vector<uint32_t> flat = detail::FlatRows(queries, "queries", &sq);
        const size_t nq = queries.size();
        std::vector<uint32_t> ref(nq * k), same(nq * k), nh(nq);
        std::vector<double> dist(nq * k);
        int rc = pg_mash_index_query(h_, flat.data(), nq, sq, k, minSame, ref.data(), same.data(), dist.data(), nh.data());
        if (rc == PG_ERR_PANIC) throw GoPanic("index out of range [-1]");
        check(rc);
        std::vector<std::vector<Neighbor>> out(nq);
        for (size_t q = 0; q < nq; ++q)
            for (uint32_t t = 0; t < nh[q]; ++t) out[q].push_back(Neighbor{ref[q * k + t], same[q * k + t], dist[q * k + t]});
        return out;
    }
    // For each query, every reference with Same >= minSame (>= 1), however many, by Ref ascending.
    std::vector<std::vector<Neighbor>> Within(const std::vector<Mash> &queries, uint32_t minSame = 1) const {
        int sq;
        const std::vector<uint32_t> flat = detail::FlatRows(queries, "queries", &sq);
        const size_t nq = queries.size();
        std::vector<uint64_t> off(nq + 1);
        uint64_t total = 0;
        // count first, then fill lists of the exact size
        int rc = pg_mash_index_query_within(h_, flat.data(), nq, sq, minSame, off.data(), nullptr, nullptr, nullptr, 0, &total);
        std::vector<uint32_t> ref(total + 1), same(total + 1);
        std::vector<double> dist(total + 1);
        if (rc == PG_OK)
            rc = pg_mash_index_query_within(h_, flat.data(), nq, sq, minSame, off.data(), ref.data(), same.data(), dist.data(), total, &total);
        if (rc == PG_ERR_PANIC) throw GoPanic("index out of range [-1]");
        check(rc);
        std::vector<std::vector<Neighbor>> out(nq);
        for (size_t q = 0; q < nq; ++q)
            for (uint64_t h = off[q]; h < off[q + 1]; ++h) out[q].push_back(Neighbor{ref[h], same[h], dist[h]});
        return out;
    }
};

// ---- cluster: single-linkage groups of a sketch set (pg_mash_cluster) --------------------------------
// Labels[i] = the smallest index in i's group; Groups = number of groups; Links = number of linked pairs i < j.
struct Clusters {
    std::vector<uint32_t> Labels;
    uint64_t Groups = 0, Links = 0;
};
// The smallest matching count whose Distance over sketches of size `den` is <= maxDistance, by Distance's own
// expression 1 - same/den (mash.go:134,139); den + 1 when no count qualifies.
inline uint32_t MinSameForDistance(double maxDistance, int den) {
    uint32_t same = 0;
    while ((int64_t)same <= den && !(1 - (double)same / (double)std::max(den, 1) <= maxDistance)) ++same;
    return same;
}
// Sketches i < j of one SketchSize are linked when mashes[i].Similarity(mashes[j]) counts at least minSame matching
// hashes (the lower index is the receiver); the groups are the connected components.
inline Clusters Cluster(const std::vector<Mash> &mashes, uint32_t minSame) {
    int s;
    const std::vector<uint32_t> flat = detail::FlatRows(mashes, "sketches", &s);
    Clusters out;
    out.Labels.resize(mashes.size());
    int rc = pg_mash_cluster(flat.data(), mashes.size(), s, minSame, out.Labels.data(), &out.Groups, &out.Links);
    if (rc == PG_ERR_PANIC) throw GoPanic("index out of range [-1]");
    check(rc);
    return out;
}

// ---- dereplicate: greedy representatives of a sketch set (pg_mash_dereplicate) ---------------------------
// Rep[i] = i for a representative, otherwise i's representative; NReps = number of representatives.
struct Representatives {
    std::vector<uint32_t> Rep;
    uint64_t NReps = 0;
};
// Links as in Cluster.  In index order, i is a representative iff no representative r < i is linked to i; any
// other i gets the smallest linked representative, or with `nearest` the one with the largest count (ties to the
// smaller index).
inline Representatives Dereplicate(const std::vector<Mash> &mashes, uint32_t minSame, bool nearest = false) {
    int s;
    const std::vector<uint32_t> flat = detail::FlatRows(mashes, "sketches", &s);
    Representatives out;
    out.Rep.resize(mashes.size());
    int rc = pg_mash_dereplicate(flat.data(), mashes.size(), s, minSame, nearest ? PG_DEREP_NEAREST : 0u, out.Rep.data(), &out.NReps);
    if (rc == PG_ERR_PANIC) throw GoPanic("index out of range [-1]");
    check(rc);
    return out;
}

// A growing dereplication: each Add assigns a batch against the representatives kept so far, on the device.
// Sketches are numbered in the order they are added, and the concatenated Rep of any sequence of Adds equals
// Dereplicate of the concatenated batches.
class Dereplicator {
    pg_mash_dereplicator *h_ = nullptr;

public:
    Dereplicator(int sketchSize, uint32_t minSame, bool nearest = false) {
        int rc = pg_mash_dereplicator_create(sketchSize, minSame, nearest ? PG_DEREP_NEAREST : 0u, &h_);
        if (rc == PG_ERR_PANIC) throw GoPanic("index out of range [-1]");
        check(rc);
    }
    Dereplicator(const Dereplicator &) = delete;
    Dereplicator &operator=(const Dereplicator &) = delete;
    ~Dereplicator() { pg_mash_dereplicator_free(h_); }
    // Rep[i] = the id of batch row i's representative (First + i for a new one); NReps = the new representatives
    struct Batch {
        std::vector<uint32_t> Rep;
        uint64_t First = 0, NReps = 0;
    };
    Batch Add(const std::vector<Mash> &mashes) {
        int s;
        const std::vector<uint32_t> flat = detail::FlatRows(mashes, "sketches", &s);
        Batch out;
        out.Rep.resize(mashes.size());
        int rc = pg_mash_dereplicator_add(h_, flat.data(), mashes.size(), s, out.Rep.data(), &out.First, &out.NReps);
        if (rc == PG_ERR_PANIC) throw GoPanic("index out of range [-1]");
        check(rc);
        return out;
    }
    // the ids of the representatives kept so far, ascending
    std::vector<uint32_t> Reps() const {
        uint64_t n = 0;
        std::vector<uint32_t> ids;
        int rc;
        do {  // an add on another thread may keep more between two calls
            ids.resize(n);
            rc = pg_mash_dereplicator_reps(h_, ids.data(), ids.size(), &n);
        } while (rc == PG_ERR_ARG && n > ids.size());
        check(rc);
        return ids;
    }
};

// A growing clustering: each Add merges a batch into the single-linkage groups of the sketches added so far, on
// the device.  Sketches are numbered in the order they are added; after every Add, Labels() equals Cluster of the
// concatenated batches, and the Links of the Adds sum to its Links.  Earlier labels change when a batch joins two
// earlier groups (Merged > 0).
class Clusterer {
    pg_mash_clusterer *h_ = nullptr;

public:
    Clusterer(int sketchSize, uint32_t minSame) {
        int rc = pg_mash_clusterer_create(sketchSize, minSame, &h_);
        if (rc == PG_ERR_PANIC) throw GoPanic("index out of range [-1]");
        check(rc);
    }
    Clusterer(const Clusterer &) = delete;
    Clusterer &operator=(const Clusterer &) = delete;
    ~Clusterer() { pg_mash_clusterer_free(h_); }
    // Labels = the batch rows' labels (global ids) after the add; Groups = every group after it; Links = the
    // links this add found; Merged = the earlier groups it absorbed into another
    struct Batch {
        std::vector<uint32_t> Labels;
        uint64_t First = 0, Groups = 0, Links = 0, Merged = 0;
    };
    Batch Add(const std::vector<Mash> &mashes) {
        int s;
        const std::vector<uint32_t> flat = detail::FlatRows(mashes, "sketches", &s);
        Batch out;
        out.Labels.resize(mashes.size());
        int rc = pg_mash_clusterer_add(h_, flat.data(), mashes.size(), s, out.Labels.data(), &out.First, &out.Groups, &out.Links,
                                       &out.Merged);
        if (rc == PG_ERR_PANIC) throw GoPanic("index out of range [-1]");
        check(rc);
        return out;
    }
    // the current labels of sketches [begin, end)
    std::vector<uint32_t> Labels(uint64_t begin, uint64_t end) const {
        std::vector<uint32_t> out(end > begin ? end - begin : 0);
        check(pg_mash_clusterer_labels(h_, begin, end, out.data()));
        return out;
    }
};

// Mash Screen on the device (pg_mash_screen): which references of a sketch set a pool of reads contains.  Add hashes
// every window a Sketch would hash of every read into the pool; Results gives, per reference, Shared = sum over v of
// min(c_r(v), c_pool(v)), Containment = Shared / s and Multiplicity = the lower median pool count of the shared
// hashes; Winners gives them after Mash Screen's winner-take-all.  Any split of the pool into Adds gives the same
// Results and Winners; Reset empties the pool.  A screen of several samples holds one pool per sample over the
// one reference set: AddSamples tags each read with its sample, and row q of ResultsSamples / WinnersSamples is what
// a one-sample screen fed only sample q's reads answers.  Add counts into sample 0; Results and Winners give row 0.
// canonical counts canonical k-mers (PG_KMER_CANONICAL), for references sketched the same way.
class Screen {
    pg_mash_screen *h_ = nullptr;
    size_t n_ = 0;
    int k_ = 0;

public:
    Screen(const std::vector<Mash> &refs, int kmerSize, uint32_t samples = 1, bool canonical = false) : n_(refs.size()), k_(kmerSize) {
        int s;
        const std::vector<uint32_t> flat = detail::FlatRows(refs, "references", &s);
        int rc = pg_mash_screen_create_flags(flat.data(), refs.size(), s, kmerSize, samples, canonical ? PG_KMER_CANONICAL : 0u, &h_);
        if (rc == PG_ERR_PANIC) throw GoPanic("index out of range [-1]");
        check(rc);
    }
    Screen(const Screen &) = delete;
    Screen &operator=(const Screen &) = delete;
    ~Screen() { pg_mash_screen_free(h_); }
    void Add(const std::vector<std::string> &reads) {
        const Flat f(reads);
        check(pg_mash_screen_add(h_, f.bases.data(), f.offsets.data(), reads.size()));
    }
    // read i goes to sample ids[i]; an id that is not a sample is an error and nothing is added
    void AddSamples(const std::vector<std::string> &reads, const std::vector<uint32_t> &ids) {
        if (ids.size() != reads.size()) throw std::invalid_argument("one sample id per read");
        const Flat f(reads);
        check(pg_mash_screen_add_samples(h_, f.bases.data(), f.offsets.data(), ids.data(), reads.size()));
    }
    void Reset() { check(pg_mash_screen_reset(h_)); }
    struct Result {
        std::vector<uint32_t> Shared;
        std::vector<double> Containment;
        std::vector<uint64_t> Multiplicity;
    };
    Result Results() const {
        Result r;
        r.Shared.resize(n_);
        r.Containment.resize(n_);
        r.Multiplicity.resize(n_);
        check(pg_mash_screen_results(h_, r.Shared.data(), r.Containment.data(), r.Multiplicity.data()));
        return r;
    }
    // Mash Screen's winner-take-all: each pool hash goes to the reference that holds it with the largest Shared of
    // Results (ties to the smallest index), and the three arrays are recomputed over the hashes each one won
    Result Winners() const {
        Result r;
        r.Shared.resize(n_);
        r.Containment.resize(n_);
        r.Multiplicity.resize(n_);
        check(pg_mash_screen_winners(h_, r.Shared.data(), r.Containment.data(), r.Multiplicity.data()));
        return r;
    }
    // Results and Winners of samples [first, first + count), one Result per sample, from one call each
    std::vector<Result> ResultsSamples(uint32_t first, uint32_t count) const { return Table(pg_mash_screen_results_samples, first, count); }
    std::vector<Result> WinnersSamples(uint32_t first, uint32_t count) const { return Table(pg_mash_screen_winners_samples, first, count); }
    // Mash Screen's identity estimate, Containment^(1/k), on the host
    std::vector<double> Identity() const {
        std::vector<double> out = Results().Containment;
        for (double &c : out) c = std::pow(c, 1.0 / k_);
        return out;
    }

private:
    using TableFn = int (*)(const pg_mash_screen *, uint32_t, uint32_t, uint32_t *, double *, uint64_t *);
    std::vector<Result> Table(TableFn fn, uint32_t first, uint32_t count) const {
        std::vector<uint32_t> shared(n_ * count);
        std::vector<double> cont(n_ * count);
        std::vector<uint64_t> mult(n_ * count);
        check(fn(h_, first, count, shared.data(), cont.data(), mult.data()));
        std::vector<Result> out(count);
        for (uint32_t q = 0; q < count; ++q) {
            out[q].Shared.assign(shared.begin() + q * n_, shared.begin() + (q + 1) * n_);
            out[q].Containment.assign(cont.begin() + q * n_, cont.begin() + (q + 1) * n_);
            out[q].Multiplicity.assign(mult.begin() + q * n_, mult.begin() + (q + 1) * n_);
        }
        return out;
    }
};

}  // namespace mash

namespace align {

struct AlphabetError : std::runtime_error {  // alphabet.Error, alphabet.go:14-22
    using std::runtime_error::runtime_error;
};

// Go's string(byte b): the UTF-8 encoding of code point b (align.go:90)
inline std::string go_string_of_byte(uint8_t b) {
    if (b < 0x80) return std::string(1, (char)b);
    return std::string{(char)(0xC0 | (b >> 6)), (char)(0x80 | (b & 0x3F))};
}

struct Alphabet {  // alphabet.go:9-12
    std::vector<std::string> symbols;
    std::map<std::string, int> encoding;
    int Encode(const std::string &symbol) const {  // alphabet.go:35-41
        auto it = encoding.find(symbol);
        if (it == encoding.end()) throw AlphabetError("Symbol " + symbol + " not in alphabet");
        return it->second;
    }
    std::vector<int16_t> byte_lut() const {
        std::vector<int16_t> lut(256, -1);
        for (int b = 0; b < 256; ++b) {
            auto it = encoding.find(go_string_of_byte((uint8_t)b));
            if (it != encoding.end()) lut[b] = (int16_t)it->second;
        }
        return lut;
    }
};
inline Alphabet NewAlphabet(const std::vector<std::string> &symbols) {  // alphabet.go:25-32
    Alphabet a;
    a.symbols = symbols;
    for (size_t i = 0; i < symbols.size(); ++i) a.encoding[symbols[i]] = (int)i;
    return a;
}

struct SubstitutionMatrix {  // matrix.go:13-17
    Alphabet FirstAlphabet, SecondAlphabet;
    std::vector<std::vector<int64_t>> scores;
    int64_t Score(const std::string &a, const std::string &b) const {  // matrix.go:28-38
        return scores[FirstAlphabet.Encode(a)][SecondAlphabet.Encode(b)];
    }
};
inline SubstitutionMatrix NewSubstitutionMatrix(const Alphabet &first, const Alphabet &second,
                                                const std::vector<std::vector<int64_t>> &scores) {
    if (first.symbols.size() != scores.size() || scores.empty() || second.symbols.size() != scores[0].size())
        throw std::invalid_argument("invalid dimensions of substitution matrix");  // matrix.go:21-23
    return SubstitutionMatrix{first, second, scores};
}
inline SubstitutionMatrix Default() {  // matrix.go:41-74: +1 / -1 over A..Z
    std::vector<std::string> letters;
    for (char c = 'A'; c <= 'Z'; ++c) letters.emplace_back(1, c);
    std::vector<std::vector<int64_t>> m(26, std::vector<int64_t>(26, -1));
    for (int i = 0; i < 26; ++i) m[i][i] = 1;
    return NewSubstitutionMatrix(NewAlphabet(letters), NewAlphabet(letters), m);
}

struct Scoring {  // align.go:73-76
    SubstitutionMatrix Matrix;
    int64_t GapPenalty;
};
inline Scoring NewScoring(const SubstitutionMatrix *m, int64_t gap) {  // align.go:79-87 (nil -> Default)
    return Scoring{m ? *m : Default(), gap};
}

// batched addition: score of SmithWaterman(query_i, template) for every query
inline std::vector<int64_t> SmithWatermanScores(const std::vector<std::string> &queries, const std::string &templ,
                                                const Scoring &sc, std::vector<std::string> *errors = nullptr) {
    Flat f(queries);
    auto lut_a = sc.Matrix.FirstAlphabet.byte_lut(), lut_b = sc.Matrix.SecondAlphabet.byte_lut();
    const int na = (int)sc.Matrix.scores.size(), nb = (int)sc.Matrix.scores[0].size();
    std::vector<int64_t> table((size_t)na * nb);
    for (int i = 0; i < na; ++i)
        for (int j = 0; j < nb; ++j) table[(size_t)i * nb + j] = sc.Matrix.scores[i][j];
    std::vector<int64_t> score(queries.size()), epos(queries.size());
    std::vector<int32_t> ecode(queries.size());
    check(pg_sw_score_batch(f.bases.data(), f.offsets.data(), queries.size(), reinterpret_cast<const uint8_t *>(templ.data()),
                            templ.size(), 1, lut_a.data(), lut_b.data(), table.data(), na, nb, sc.GapPenalty, score.data(),
                            ecode.data(), epos.data()));
    if (errors) {
        errors->assign(queries.size(), "");
        for (size_t i = 0; i < queries.size(); ++i)
            if (ecode[i]) {
                const uint8_t b = ecode[i] == 1 ? (uint8_t)queries[i][epos[i]] : (uint8_t)templ[epos[i]];
                (*errors)[i] = "Symbol " + go_string_of_byte(b) + " not in alphabet";  // alphabet.go:38
            }
    }
    return score;
}

// Score of align.SmithWaterman(stringA, stringB, scoring) (align.go:171-203).  The aligned
// strings (traceback, align.go:205-231) are a "next" row of SURVEY.md 8f.
inline int64_t SmithWaterman(const std::string &a, const std::string &b, const Scoring &sc) {
    std::vector<std::string> errs;
    auto s = SmithWatermanScores({a}, b, sc, &errs);
    if (!errs[0].empty()) throw AlphabetError(errs[0]);
    return s[0];
}

// Full align.SmithWaterman (align.go:171-232): score and the two aligned strings of the
// reference's traceback.  The shorter string (<= 64 symbols) rides in registers on the GPU.
struct Alignment {
    int64_t score;
    std::string alignA, alignB;
};
inline Alignment align_strings(bool global, const std::string &a, const std::string &b, const Scoring &sc) {
    const bool query_is_a = a.size() <= 64;
    const std::string &q = query_is_a ? a : b, &t = query_is_a ? b : a;
    Flat f({q});
    auto lut_a = sc.Matrix.FirstAlphabet.byte_lut(), lut_b = sc.Matrix.SecondAlphabet.byte_lut();
    const int na = (int)sc.Matrix.scores.size(), nb = (int)sc.Matrix.scores[0].size();
    std::vector<int64_t> table((size_t)na * nb);
    for (int i = 0; i < na; ++i)
        for (int j = 0; j < nb; ++j) table[(size_t)i * nb + j] = sc.Matrix.scores[i][j];
    uint64_t stride = global ? q.size() + t.size() + 8 : 2 * q.size() + 64;
    for (;;) {
        std::vector<uint8_t> oa(stride), ob(stride);
        int64_t score = 0, epos = 0;
        int32_t ecode = 0, status = 0;
        uint32_t len = 0;
        check((global ? pg_nw_align_batch : pg_sw_align_batch)(
            f.bases.data(), f.offsets.data(), 1, reinterpret_cast<const uint8_t *>(t.data()), t.size(), query_is_a ? 1 : 0,
            lut_a.data(), lut_b.data(), table.data(), na, nb, sc.GapPenalty, &score, &ecode, &epos, oa.data(), ob.data(), stride,
            &len, &status));
        if (ecode) {
            const uint8_t bad = ecode == 1 ? (uint8_t)a[epos] : (uint8_t)b[epos];
            throw AlphabetError("Symbol " + go_string_of_byte(bad) + " not in alphabet");
        }
        if (status == PG_ITEM_UNSUPPORTED) { stride = len + 8; continue; }
        return Alignment{score, std::string(oa.begin(), oa.begin() + len), std::string(ob.begin(), ob.begin() + len)};
    }
}

inline Alignment SmithWatermanAlign(const std::string &a, const std::string &b, const Scoring &sc) {
    return align_strings(false, a, b, sc);
}
// Full align.NeedlemanWunsch (align.go:100-166), including its loop condition (align.go:141).
inline Alignment NeedlemanWunschAlign(const std::string &a, const std::string &b, const Scoring &sc) {
    return align_strings(true, a, b, sc);
}

// Score of align.NeedlemanWunsch (align.go:100-134,166)
inline int64_t NeedlemanWunschScore(const std::string &a, const std::string &b, const Scoring &sc) {
    Flat f({a});
    auto lut_a = sc.Matrix.FirstAlphabet.byte_lut(), lut_b = sc.Matrix.SecondAlphabet.byte_lut();
    const int na = (int)sc.Matrix.scores.size(), nb = (int)sc.Matrix.scores[0].size();
    std::vector<int64_t> table((size_t)na * nb);
    for (int i = 0; i < na; ++i)
        for (int j = 0; j < nb; ++j) table[(size_t)i * nb + j] = sc.Matrix.scores[i][j];
    int64_t score = 0, epos = 0;
    int32_t ecode = 0;
    check(pg_nw_score_batch(f.bases.data(), f.offsets.data(), 1, reinterpret_cast<const uint8_t *>(b.data()), b.size(), 1,
                            lut_a.data(), lut_b.data(), table.data(), na, nb, sc.GapPenalty, &score, &ecode, &epos));
    if (ecode) {
        const uint8_t bad = ecode == 1 ? (uint8_t)a[epos] : (uint8_t)b[epos];
        throw AlphabetError("Symbol " + go_string_of_byte(bad) + " not in alphabet");
    }
    return score;
}

// Pair lists: pair p aligns stringA = as[pairA[p]] against stringB = bs[pairB[p]] in one call.  Indices must
// lie in [0, as.size()) / [0, bs.size()) (Error PG_ERR_ARG otherwise); errors[p] is "" or the
// reference's alphabet error of that pair.
inline std::vector<int64_t> table_of(const Scoring &sc) {
    const int na = (int)sc.Matrix.scores.size(), nb = (int)sc.Matrix.scores[0].size();
    std::vector<int64_t> table((size_t)na * nb);
    for (int i = 0; i < na; ++i)
        for (int j = 0; j < nb; ++j) table[(size_t)i * nb + j] = sc.Matrix.scores[i][j];
    return table;
}
inline std::string pair_error(int32_t ecode, int64_t epos, const std::string &a, const std::string &b) {
    if (!ecode) return "";
    return "Symbol " + go_string_of_byte(ecode == 1 ? (uint8_t)a[epos] : (uint8_t)b[epos]) + " not in alphabet";
}
inline std::vector<int64_t> pair_scores(bool global, const std::vector<std::string> &as, const std::vector<std::string> &bs,
                                        const std::vector<uint32_t> &pairA, const std::vector<uint32_t> &pairB, const Scoring &sc,
                                        std::vector<std::string> *errors) {
    if (pairA.size() != pairB.size()) throw std::invalid_argument("pairA and pairB differ in length");
    Flat fa(as), fb(bs);
    auto lut_a = sc.Matrix.FirstAlphabet.byte_lut(), lut_b = sc.Matrix.SecondAlphabet.byte_lut();
    auto table = table_of(sc);
    const size_t n = pairA.size();
    std::vector<int64_t> score(n), epos(n);
    std::vector<int32_t> ecode(n);
    check((global ? pg_nw_score_pairs : pg_sw_score_pairs)(fa.bases.data(), fa.offsets.data(), as.size(), fb.bases.data(), fb.offsets.data(),
                                                           bs.size(), pairA.data(), pairB.data(), n, lut_a.data(), lut_b.data(), table.data(),
                                                           (int)sc.Matrix.scores.size(), (int)sc.Matrix.scores[0].size(), sc.GapPenalty,
                                                           score.data(), ecode.data(), epos.data()));
    if (errors) {
        errors->assign(n, "");
        for (size_t k = 0; k < n; ++k) (*errors)[k] = pair_error(ecode[k], epos[k], as[pairA[k]], bs[pairB[k]]);
    }
    return score;
}
inline std::vector<int64_t> SmithWatermanPairScores(const std::vector<std::string> &as, const std::vector<std::string> &bs,
                                                    const std::vector<uint32_t> &pairA, const std::vector<uint32_t> &pairB,
                                                    const Scoring &sc, std::vector<std::string> *errors = nullptr) {
    return pair_scores(false, as, bs, pairA, pairB, sc, errors);
}
inline std::vector<int64_t> NeedlemanWunschPairScores(const std::vector<std::string> &as, const std::vector<std::string> &bs,
                                                      const std::vector<uint32_t> &pairA, const std::vector<uint32_t> &pairB,
                                                      const Scoring &sc, std::vector<std::string> *errors = nullptr) {
    return pair_scores(true, as, bs, pairA, pairB, sc, errors);
}
// aligned strings per pair ({0, "", ""} where errors[p] is set)
inline std::vector<Alignment> pair_aligns(bool global, const std::vector<std::string> &as, const std::vector<std::string> &bs,
                                          const std::vector<uint32_t> &pairA, const std::vector<uint32_t> &pairB, const Scoring &sc,
                                          std::vector<std::string> *errors) {
    if (pairA.size() != pairB.size()) throw std::invalid_argument("pairA and pairB differ in length");
    Flat fa(as), fb(bs);
    auto lut_a = sc.Matrix.FirstAlphabet.byte_lut(), lut_b = sc.Matrix.SecondAlphabet.byte_lut();
    auto table = table_of(sc);
    const size_t n = pairA.size();
    uint64_t stride = 1;  // an alignment has at most len(a) + len(b) columns
    for (size_t k = 0; k < n; ++k)
        if (pairA[k] < as.size() && pairB[k] < bs.size()) stride = std::max<uint64_t>(stride, as[pairA[k]].size() + bs[pairB[k]].size());
    std::vector<int64_t> score(n), epos(n);
    std::vector<int32_t> ecode(n), status(n);
    std::vector<uint32_t> len(n);
    std::vector<uint8_t> oa(std::max<size_t>(n, 1) * stride), ob(std::max<size_t>(n, 1) * stride);
    check((global ? pg_nw_align_pairs : pg_sw_align_pairs)(fa.bases.data(), fa.offsets.data(), as.size(), fb.bases.data(), fb.offsets.data(),
                                                           bs.size(), pairA.data(), pairB.data(), n, lut_a.data(), lut_b.data(), table.data(),
                                                           (int)sc.Matrix.scores.size(), (int)sc.Matrix.scores[0].size(), sc.GapPenalty,
                                                           score.data(), ecode.data(), epos.data(), oa.data(), ob.data(), stride, len.data(),
                                                           status.data()));
    std::vector<Alignment> out(n);
    if (errors) errors->assign(n, "");
    for (size_t k = 0; k < n; ++k) {
        if (ecode[k]) {
            if (errors) (*errors)[k] = pair_error(ecode[k], epos[k], as[pairA[k]], bs[pairB[k]]);
            out[k] = Alignment{0, "", ""};
            continue;
        }
        const char *pa = reinterpret_cast<const char *>(oa.data() + k * stride), *pb = reinterpret_cast<const char *>(ob.data() + k * stride);
        out[k] = Alignment{score[k], std::string(pa, len[k]), std::string(pb, len[k])};
    }
    return out;
}
inline std::vector<Alignment> SmithWatermanPairAligns(const std::vector<std::string> &as, const std::vector<std::string> &bs,
                                                      const std::vector<uint32_t> &pairA, const std::vector<uint32_t> &pairB,
                                                      const Scoring &sc, std::vector<std::string> *errors = nullptr) {
    return pair_aligns(false, as, bs, pairA, pairB, sc, errors);
}
inline std::vector<Alignment> NeedlemanWunschPairAligns(const std::vector<std::string> &as, const std::vector<std::string> &bs,
                                                        const std::vector<uint32_t> &pairA, const std::vector<uint32_t> &pairB,
                                                        const Scoring &sc, std::vector<std::string> *errors = nullptr) {
    return pair_aligns(true, as, bs, pairA, pairB, sc, errors);
}

}  // namespace align

namespace primers {

struct Tm { double meltingTemp, dH, dS; };

// primers.SantaLucia, primers.go:70-105
inline Tm SantaLucia(const std::string &sequence, double primerConcentration, double saltConcentration,
                     double magnesiumConcentration) {
    const uint64_t off[2] = {0, sequence.size()};
    Tm t{};
    int32_t st = 0;
    int rc = pg_tm_batch(reinterpret_cast<const uint8_t *>(sequence.data()), off, 1, primerConcentration, saltConcentration,
                         magnesiumConcentration, &t.meltingTemp, &t.dH, &t.dS, &st);
    if (st == PG_ITEM_PANIC) throw GoPanic("index out of range [-1]");  // primers.go:89
    if (st == PG_ITEM_UNSUPPORTED) throw std::invalid_argument("byte >= 0x80 in primer (unsupported)");
    check(rc);
    return t;
}
// primers.MeltingTemp, primers.go:121-128
inline double MeltingTemp(const std::string &sequence) { return SantaLucia(sequence, 500e-9, 50e-3, 0.0).meltingTemp; }

inline std::vector<double> MeltingTemps(const std::vector<std::string> &seqs) {
    Flat f(seqs);
    std::vector<double> tm(seqs.size());
    std::vector<int32_t> st(seqs.size());
    int rc = pg_tm_batch(f.bases.data(), f.offsets.data(), seqs.size(), 500e-9, 50e-3, 0.0, tm.data(), nullptr, nullptr, st.data());
    for (auto s : st)
        if (s == PG_ITEM_PANIC) throw GoPanic("index out of range [-1]");
    check(rc);
    return tm;
}

}  // namespace primers

namespace transform {
// transform.ReverseComplement, transform/transform.go:15-23,78-109: bytes outside the table become 0
inline std::string ReverseComplement(const std::string &seq) {
    static const char *from = "ABCDGHKMNRSTVWYabcdghkmnrstvwy", *to = "TVGHCDMKNYSABWRtvghcdmknysabwr";
    uint8_t table[256] = {0};
    for (int i = 0; from[i]; ++i) table[(uint8_t)from[i]] = (uint8_t)to[i];
    std::string out(seq.size(), '\0');
    for (size_t i = 0; i < seq.size(); ++i) out[i] = (char)table[(uint8_t)seq[seq.size() - 1 - i]];
    return out;
}
}  // namespace transform

// primers/pcr (primers/pcr/pcr.go): the Tm searches (pcr.go:44-60, 93-100) and the binding-site search the
// reference does with a suffix array (pcr.go:87,110-115) run on the GPU; the fragment bookkeeping
// (pcr.go:117-166,181-195) is host work, as in the reference.
namespace pcr {

inline std::string upper_ascii(const std::string &s) {
    std::string u = s;
    for (char &c : u) {
        if ((uint8_t)c >= 0x80) throw std::invalid_argument("byte >= 0x80: strings.ToUpper on non-ASCII input is unsupported");
        if (c >= 'a' && c <= 'z') c = (char)(c - 32);
    }
    return u;
}

// pcr.DesignPrimersWithOverhangs, pcr.go:44-60
inline std::pair<std::string, std::string> DesignPrimersWithOverhangs(const std::string &sequence, const std::string &forwardOverhang,
                                                                       const std::string &reverseOverhang, double targetTm) {
    const std::string templ = upper_ascii(sequence);
    const uint64_t off[2] = {0, templ.size()};
    uint32_t fwd = 0, rev = 0;
    int32_t st = 0;
    int rc = pg_design_primers_batch(reinterpret_cast<const uint8_t *>(templ.data()), off, 1, targetTm, &fwd, &rev, &st);
    if (rc == PG_ERR_PANIC || st == PG_ITEM_PANIC) throw GoPanic("slice bounds out of range");  // the reference slices past the end
    check(rc);
    return {forwardOverhang + templ.substr(0, fwd), transform::ReverseComplement(reverseOverhang) + transform::ReverseComplement(templ.substr(templ.size() - rev))};
}
// pcr.DesignPrimers, pcr.go:62-66
inline std::pair<std::string, std::string> DesignPrimers(const std::string &sequence, double targetTm) {
    return DesignPrimersWithOverhangs(sequence, "", "", targetTm);
}

// pcr.SimulateSimple, pcr.go:73-169.  Like the reference it upper-cases primerList in place.
inline std::vector<std::string> SimulateSimple(const std::vector<std::string> &sequences, double targetTm, bool circular,
                                               std::vector<std::string> &primerList) {
    for (auto &p : primerList) p = upper_ascii(p);  // pcr.go:76-78
    std::vector<std::string> fragments;
    if (sequences.empty()) return fragments;
    std::vector<std::string> templates;
    for (auto &q : sequences) templates.push_back(upper_ascii(q));  // pcr.go:82
    // GPU pass 1: the minimal binding part of every primer (pcr.go:93-103)
    std::vector<std::string> minimal(primerList.size());
    std::vector<std::string> patterns;
    std::vector<std::pair<int, bool>> owner;  // (primer, is reverse complement)
    if (!primerList.empty()) {
        Flat f(primerList);
        std::vector<uint32_t> ml(primerList.size());
        std::vector<int32_t> st(primerList.size());
        int rc = pg_pcr_minimal_primer_batch(f.bases.data(), f.offsets.data(), primerList.size(), targetTm, ml.data(), st.data());
        for (int32_t x : st)
            if (x == PG_ITEM_PANIC) throw GoPanic("slice bounds out of range");  // primer shorter than 7 nt (pcr.go:35,96)
        if (rc != PG_ERR_PANIC) check(rc);
        for (size_t p = 0; p < primerList.size(); ++p) {
            const std::string part = primerList[p].substr(primerList[p].size() - ml[p]);
            if (part == primerList[p]) continue;  // pcr.go:103: ignored
            minimal[p] = part;
            patterns.push_back(part);
            owner.emplace_back((int)p, false);
            patterns.push_back(transform::ReverseComplement(part));
            owner.emplace_back((int)p, true);
        }
    }
    // GPU pass 2: every occurrence of every pattern in every template (pcr.go:110,113)
    struct Hit { uint32_t seq; uint64_t pos; uint32_t pat; };
    std::vector<Hit> hits;
    if (!patterns.empty()) {
        Flat ft(templates), fp(patterns);
        uint64_t cap = 1024, found = 0;
        for (;;) {
            std::vector<uint32_t> hs(cap), hq(cap);
            std::vector<uint64_t> hp(cap);
            int rc = pg_find_sites_batch(ft.bases.data(), ft.offsets.data(), templates.size(), fp.bases.data(), fp.offsets.data(),
                                         (uint32_t)patterns.size(), 0, hs.data(), hp.data(), hq.data(), cap, &found);
            if (rc == PG_ERR_ARG && found > cap) { cap = found; continue; }
            check(rc);
            for (uint64_t i = 0; i < found; ++i) hits.push_back({hs[i], hp[i], hq[i]});
            break;
        }
        // the order in which the reference fills its maps: by template, then primer (forward lookup first), then position
        std::sort(hits.begin(), hits.end(), [](const Hit &a, const Hit &b) {
            if (a.seq != b.seq) return a.seq < b.seq;
            if (a.pat != b.pat) return a.pat < b.pat;
            return a.pos < b.pos;
        });
    }
    size_t cursor = 0;
    for (size_t t = 0; t < templates.size(); ++t) {
        const std::string &templ = templates[t];
        std::map<uint64_t, std::vector<int>> fwd, rev;  // position -> primers bound there, in primer-list order; keys ascending
        for (; cursor < hits.size() && hits[cursor].seq == t; ++cursor)
            (owner[hits[cursor].pat].second ? rev : fwd)[hits[cursor].pos].push_back(owner[hits[cursor].pat].first);
        auto emit = [&](const std::string &text, uint64_t from, uint64_t to, const std::vector<int> &fps, const std::vector<int> &rps) {
            for (int fp : fps)      // generatePcrFragments, pcr.go:181-195
                for (int rp : rps)
                    fragments.push_back(primerList[fp].substr(0, primerList[fp].size() - minimal[fp].size()) + text.substr(from, to - from) +
                                        transform::ReverseComplement(primerList[rp]));
        };
        for (auto f = fwd.begin(); f != fwd.end(); ++f) {
            auto next = std::next(f);
            auto r = rev.upper_bound(f->first);  // reverse sites strictly to the right
            if (next != fwd.end()) {             // pcr.go:133-143: the first reverse site before the next forward site
                if (r != rev.end() && r->first < next->first) emit(templ, f->first, r->first, f->second, r->second);
                continue;
            }
            const bool found = r != rev.end();
            for (; r != rev.end(); ++r) emit(templ, f->first, r->first, f->second, r->second);  // pcr.go:146-151
            if (circular && !found) {            // pcr.go:153-164: look across the origin
                const std::string rotated = templ.substr(f->first) + templ.substr(0, f->first);
                for (auto q = rev.begin(); q != rev.end() && q->first < fwd.begin()->first; ++q)
                    emit(rotated, 0, templ.size() - f->first + q->first, f->second, q->second);
            }
        }
    }
    return fragments;
}

// pcr.Simulate, pcr.go:171-186: (fragments, error message; empty = nil)
struct Simulation {
    std::vector<std::string> fragments;
    bool hasFragments = true;  // false: the reference returns nil
    std::string error;
};
inline Simulation Simulate(const std::vector<std::string> &sequences, double targetTm, bool circular, std::vector<std::string> &primerList) {
    for (auto &p : primerList)
        if (p.size() < 7) return {{}, false, "Primers are too short."};  // minimalPrimerLength, pcr.go:35,174-178
    Simulation sim;
    sim.fragments = SimulateSimple(sequences, targetTm, circular, primerList);
    std::vector<std::string> again = primerList;
    again.insert(again.end(), sim.fragments.begin(), sim.fragments.end());
    if (SimulateSimple(sequences, targetTm, circular, again).size() != sim.fragments.size()) sim.error = "Concatemerization detected in PCR.";
    return sim;
}

}  // namespace pcr

namespace fasta {

// fasta.Fasta, io/fasta/fasta.go:66-69
struct Fasta {
    std::string Name, Sequence;
    bool operator==(const Fasta &o) const { return Name == o.Name && Sequence == o.Sequence; }
};
// the `error` half of ([]Fasta, error): code as pg_fasta_ingest reports it, 0 = nil
struct ParseResult {
    std::vector<Fasta> fastas;
    int32_t err_code = 0;
    uint64_t err_line = 0;
    std::string error() const {
        switch (err_code) {
            case 1: return "did not find fasta start '>', got to line " + std::to_string(err_line);
            case 2: return "empty fasta sequence, got to line " + std::to_string(err_line);
            case 3: return "line " + std::to_string(err_line) + " too large for buffer, use larger maxLineSize";
            case 4: return "bufio: buffer full";
            default: return "";
        }
    }
};

// NewParser(r, maxLineSize).ParseAll(), fasta.go:89-99; bufioAlias = give exactly what the reference
// gives over a strings.Reader / *os.File (see include/poly_b200.h, PG_FASTA_BUFIO_ALIAS)
inline ParseResult ParseAll(const std::string &text, uint32_t maxLineSize, bool bufioAlias = true) {
    uint64_t lines = 1;
    for (char c : text) lines += c == '\n';
    std::vector<uint8_t> bases(text.size() + 1), names(text.size() + 1);
    std::vector<uint64_t> off(lines + 1), noff(lines + 1);
    uint64_t n = 0, tot = 0, ntot = 0;
    ParseResult r;
    check(pg_fasta_ingest(reinterpret_cast<const uint8_t *>(text.data()), text.size(), maxLineSize,
                          bufioAlias ? PG_FASTA_BUFIO_ALIAS : 0u, bases.data(), bases.size(), off.data(), names.data(),
                          names.size(), noff.data(), lines, &n, &tot, &ntot, &r.err_code, &r.err_line));
    r.fastas.reserve(n);
    for (uint64_t i = 0; i < n; ++i)
        r.fastas.push_back({std::string(names.begin() + noff[i], names.begin() + noff[i + 1]),
                            std::string(bases.begin() + off[i], bases.begin() + off[i + 1])});
    return r;
}
// fasta.Parse, fasta.go:72-77
inline ParseResult Parse(const std::string &text, bool bufioAlias = true) { return ParseAll(text, 2 * 32 * 1024, bufioAlias); }

}  // namespace fasta

namespace fastq {

// fastq.Fastq, io/fastq/fastq.go:46-51
struct Fastq {
    std::string Identifier;
    std::map<std::string, std::string> Optionals;
    std::string Sequence, Quality;
};
// ([]Fastq, error) of fastq.Parse: the records before the first one the reference rejects, and that error
// (code as pg_fastq_ingest reports it, 0 = nil; err_line = the 1-based line the parser stopped at)
struct ParseResult {
    std::vector<Fastq> fastqs;
    int32_t err_code = 0;
    uint64_t err_line = 0;
    std::string error() const {
        const std::string l = std::to_string(err_line);
        switch (err_code) {
            case 1: return "line " + l + " failed: unexepcted EOF encountered";  // sic, fastq.go:150
            case 2: return "empty fastq sequence, got to line " + l;
            case 3: return "empty quality sequence, got to line " + l;
            case 4: return "did not find fastq start '@', got to line " + l;
            case 5: return "reference panics (index out of range) while parsing the identifier at line " + l;
            case 6: return "line " + l + " too large for buffer, use larger maxLineSize";
            default: return "";
        }
    }
};

// fastq.Parse, io/fastq/fastq.go:54-59 (ParseNext :117-214): records on the GPU (line index, per-record checks in the
// reference's order, dense sequences); Identifier / Optionals / Quality are cut out of `text` with the line spans.
inline ParseResult Parse(const std::string &text) {
    uint64_t cap = 1;
    for (char c : text) cap += c == '\n';
    cap = cap / 4 + 1;
    std::vector<uint8_t> bases(text.size() + 1);
    std::vector<uint64_t> off(cap + 1), spans(4 * (cap + 1));
    uint64_t n = 0, tot = 0;
    ParseResult r;
    check(pg_fastq_ingest_records(reinterpret_cast<const uint8_t *>(text.data()), text.size(), bases.data(), bases.size(), off.data(),
                                  spans.data(), cap, &n, &tot, &r.err_code, &r.err_line));
    r.fastqs.reserve(n);
    for (uint64_t i = 0; i < n; ++i) {
        Fastq f;
        const std::string line = text.substr(spans[4 * i], spans[4 * i + 1]);
        size_t pos = 0;
        bool first = true;
        while (pos <= line.size()) {  // strings.Split(line, " "), fastq.go:157
            size_t sp = line.find(' ', pos);
            if (sp == std::string::npos) sp = line.size();
            const std::string tok = line.substr(pos, sp - pos);
            if (first) {
                f.Identifier = tok.substr(1);  // without the '@', fastq.go:158
                first = false;
            } else {  // "key=value": strings.Split(datum, "=")[0], [1] (every datum holds '=': checked on the GPU)
                const size_t eq = tok.find('=');
                const size_t eq2 = tok.find('=', eq + 1);
                f.Optionals[tok.substr(0, eq)] = tok.substr(eq + 1, eq2 == std::string::npos ? std::string::npos : eq2 - eq - 1);
            }
            pos = sp + 1;
        }
        f.Sequence.assign(bases.begin() + off[i], bases.begin() + off[i + 1]);
        f.Quality = text.substr(spans[4 * i + 2], spans[4 * i + 3]);
        r.fastqs.push_back(std::move(f));
    }
    return r;
}

}  // namespace fastq

namespace seqhash {
// seqhash.go:64-68
inline const std::string DNA = "DNA", RNA = "RNA", PROTEIN = "PROTEIN";

// (seqhash, error message) per sequence; the message is empty on success.  A byte >= 0x80 ahead of any
// letter outside the alphabet is reported as unsupported rather than guessed at (DESIGN.md §7).
inline std::vector<std::pair<std::string, std::string>> HashBatch(const std::vector<std::string> &seqs, const std::string &sequenceType,
                                                                  bool circular, bool doubleStranded) {
    std::vector<std::pair<std::string, std::string>> out(seqs.size());
    const int32_t type = sequenceType == DNA ? PG_SEQHASH_DNA : sequenceType == RNA ? PG_SEQHASH_RNA : sequenceType == PROTEIN ? PG_SEQHASH_PROTEIN : -1;
    if (type < 0) {  // seqhash.go:151-153, before any GPU call
        for (auto &o : out) o.second = "Only sequenceTypes of DNA, RNA, or PROTEIN allowed. Got sequenceType: " + sequenceType;
        return out;
    }
    if (seqs.empty()) return out;
    Flat f(seqs);
    std::vector<uint8_t> digest(32 * seqs.size());
    std::vector<int32_t> code(seqs.size());
    std::vector<uint64_t> pos(seqs.size());
    check(pg_seqhash_batch(f.bases.data(), f.offsets.data(), seqs.size(), type,
                           (circular ? PG_SEQHASH_CIRCULAR : 0u) | (doubleStranded ? PG_SEQHASH_DOUBLE_STRANDED : 0u), digest.data(), code.data(),
                           pos.data()));
    static const char hex[] = "0123456789abcdef";
    for (size_t i = 0; i < seqs.size(); ++i) {
        if (code[i] == 1) {
            char c = seqs[i][pos[i]];
            if (c >= 'a' && c <= 'z') c -= 32;
            out[i].second = (type == PG_SEQHASH_PROTEIN ? "Only letters ACDEFGHIKLMNPQRSTVWYUO*BXZ are allowed for Proteins. Got letter: "
                                                        : "Only letters ATUGCYRSWKMBDHVNZ are allowed for DNA/RNA. Got letter: ") + std::string(1, c);
        } else if (code[i] == 2) {
            out[i].second = "Proteins cannot be double stranded";
        } else if (code[i] == 3) {
            out[i].second = "unsupported: byte >= 0x80 at " + std::to_string(pos[i]) + " (strings.ToUpper would re-encode it)";
        } else {
            std::string h = "v1_";
            h += sequenceType[0];
            h += circular ? 'C' : 'L';
            h += doubleStranded ? 'D' : 'S';
            h += '_';
            for (int k = 0; k < 32; ++k) {
                h += hex[digest[32 * i + k] >> 4];
                h += hex[digest[32 * i + k] & 15];
            }
            out[i].first = h;
        }
    }
    return out;
}

// seqhash.Hash (seqhash.go:141): (seqhash, error message)
inline std::pair<std::string, std::string> Hash(const std::string &sequence, const std::string &sequenceType, bool circular, bool doubleStranded) {
    return HashBatch({sequence}, sequenceType, circular, doubleStranded)[0];
}

// seqhash.RotateSequence (seqhash.go:127) of every sequence, in one call
inline std::vector<std::string> RotateSequences(const std::vector<std::string> &seqs) {
    std::vector<std::string> out(seqs.size());
    if (seqs.empty()) return out;
    Flat f(seqs);
    std::vector<uint64_t> rot(seqs.size());
    check(pg_least_rotation_batch(f.bases.data(), f.offsets.data(), seqs.size(), rot.data()));
    for (size_t i = 0; i < seqs.size(); ++i) out[i] = seqs[i].substr(rot[i]) + seqs[i].substr(0, rot[i]);
    return out;
}
inline std::string RotateSequence(const std::string &sequence) { return RotateSequences({sequence})[0]; }
}  // namespace seqhash
// ---- clone (clone/clone.go:138-355) over pg_clone_digest_batch / pg_clone_golden_gate_batch /
// pg_clone_circular_ligate_batch.  Enzyme patterns must be literals (UnsupportedError otherwise).
namespace clone {
struct UnsupportedError : std::runtime_error {
    using std::runtime_error::runtime_error;
};
struct Part {
    std::string Sequence;
    bool Circular = false;
};
struct Fragment {
    std::string Sequence, ForwardOverhang, ReverseOverhang;
};
struct Enzyme {
    std::string Name, RegexpFor, RegexpRev;
    int Skip = 0, OverheadLength = 0;
    std::string RecognitionSite;
};
inline pg_clone_enzyme to_pg(const Enzyme &e) {
    for (const std::string *p : {&e.RegexpFor, &e.RegexpRev})
        if (p->empty() || p->size() > 32 || p->find_first_of("\\.+*?()|[]{}^$") != std::string::npos)
            throw UnsupportedError("enzyme " + e.Name + ": pattern " + *p + " is not a literal (only literal sites are supported)");
    return pg_clone_enzyme{(const uint8_t *)e.RegexpFor.data(), (uint32_t)e.RegexpFor.size(), (const uint8_t *)e.RegexpRev.data(),
                           (uint32_t)e.RegexpRev.size(), (const uint8_t *)e.RecognitionSite.data(), (uint32_t)e.RecognitionSite.size(), e.Skip,
                           e.OverheadLength};
}
inline std::vector<Enzyme> GetBaseRestrictionEnzymes() {  // clone.go:358-364
    return {{"BsaI", "GGTCTC", "GAGACC", 1, 4, "GGTCTC"}, {"BbsI", "GAAGAC", "GTCTTC", 2, 4, "GAAGAC"}, {"BtgZI", "GCGATG", "CATCGC", 10, 4, "GCGATG"}};
}
inline void item_status(int32_t st) {
    if (st == PG_ITEM_PANIC) throw GoPanic("slice bounds out of range");
    if (st == PG_ITEM_UNSUPPORTED) throw UnsupportedError("a byte >= 0x80: strings.ToUpper would re-encode it (unsupported)");
}
// CutWithEnzyme of every part x enzyme: out[p][e]; an item that panics throws GoPanic
inline std::vector<std::vector<std::vector<Fragment>>> CutWithEnzymeBatch(const std::vector<Part> &parts, bool directional,
                                                                          const std::vector<Enzyme> &enzymes) {
    std::vector<std::vector<std::vector<Fragment>>> out(parts.size(), std::vector<std::vector<Fragment>>(enzymes.size()));
    if (parts.empty() || enzymes.empty()) return out;
    std::vector<std::string> seqs;
    std::vector<uint8_t> circ;
    for (const Part &p : parts) { seqs.push_back(p.Sequence); circ.push_back(p.Circular); }
    std::vector<pg_clone_enzyme> enz;
    for (const Enzyme &e : enzymes) enz.push_back(to_pg(e));
    Flat f(seqs);
    const size_t n = parts.size() * enzymes.size();
    std::vector<uint32_t> cnt(n);
    std::vector<int32_t> st(n);
    uint64_t caps[3] = {0, 0, 0}, need[3];
    std::vector<uint8_t> sb, ob;
    std::vector<uint64_t> so, oo;
    for (;;) {
        sb.assign(caps[1] + 1, 0); ob.assign(caps[2] + 1, 0); so.assign(caps[0] + 1, 0); oo.assign(2 * caps[0] + 1, 0);
        const int rc = pg_clone_digest_batch(f.bases.data(), f.offsets.data(), circ.data(), parts.size(), enz.data(), (uint32_t)enz.size(), directional,
                                             cnt.data(), st.data(), sb.data(), caps[1], so.data(), ob.data(), caps[2], oo.data(), caps[0], &need[0],
                                             &need[1], &need[2]);
        if (rc == PG_ERR_ARG && (need[0] > caps[0] || need[1] > caps[1] || need[2] > caps[2])) {
            for (int k = 0; k < 3; ++k) caps[k] = need[k];
            continue;
        }
        if (rc != PG_ERR_PANIC && rc != PG_ERR_UNSUPPORTED) check(rc);
        break;
    }
    size_t fr = 0;
    for (size_t i = 0; i < n; ++i)
        for (uint32_t k = 0; k < cnt[i]; ++k, ++fr)
            out[i / enzymes.size()][i % enzymes.size()].push_back(
                Fragment{std::string((const char *)sb.data() + so[fr], so[fr + 1] - so[fr]), std::string((const char *)ob.data() + oo[2 * fr], oo[2 * fr + 1] - oo[2 * fr]),
                         std::string((const char *)ob.data() + oo[2 * fr + 1], oo[2 * fr + 2] - oo[2 * fr + 1])});
    for (size_t i = 0; i < n; ++i)
        if (st[i] == PG_ITEM_PANIC) item_status(st[i]);
    for (size_t i = 0; i < n; ++i) item_status(st[i]);
    return out;
}
inline std::vector<Fragment> CutWithEnzyme(const Part &part, bool directional, const Enzyme &enzyme) {
    return CutWithEnzymeBatch({part}, directional, {enzyme})[0][0];
}
class EnzymeManager {
    std::map<std::string, Enzyme> enzymeMap;

public:
    explicit EnzymeManager(const std::vector<Enzyme> &enzymes) {
        for (const Enzyme &e : enzymes) enzymeMap[e.Name] = e;
    }
    // (enzyme, error message); the message is "Enzyme X not found" when it is missing (clone.go:134)
    std::pair<Enzyme, std::string> GetEnzymeByName(const std::string &name) const {
        auto it = enzymeMap.find(name);
        if (it == enzymeMap.end()) return {Enzyme{}, "Enzyme " + name + " not found"};
        return {it->second, ""};
    }
    std::pair<std::vector<Fragment>, std::string> CutWithEnzymeByName(const Part &part, bool directional, const std::string &name) const {
        auto e = GetEnzymeByName(name);
        if (!e.second.empty()) return {{}, e.second};
        return {CutWithEnzyme(part, directional, e.first), ""};
    }
};
inline EnzymeManager NewEnzymeManager(const std::vector<Enzyme> &enzymes) { return EnzymeManager(enzymes); }

using Constructs = std::pair<std::vector<std::string>, std::vector<std::string>>;  // (clones, looping constructs)
// call(bytes_cap, constructs_cap, out, offsets, kinds, counts, status, need_bytes, need_constructs)
// per_reaction: the call reports unsupported input per reaction (GoldenGate); otherwise it refuses the call
template <typename Call>
std::vector<Constructs> ligation_outputs(size_t n_reactions, Call call, bool per_reaction = true) {
    uint64_t bcap = 1 << 20, ccap = 1 << 12, nb = 0, nc = 0;
    std::vector<uint8_t> out, kinds;
    std::vector<uint64_t> off, counts(2 * n_reactions + 2);
    std::vector<int32_t> st(n_reactions + 1);
    for (;;) {
        out.assign(bcap + 1, 0); off.assign(ccap + 1, 0); kinds.assign(ccap + 1, 0);
        const int rc = call(bcap, ccap, out.data(), off.data(), kinds.data(), counts.data(), st.data(), &nb, &nc);
        if (rc == PG_ERR_ARG && (nb > bcap || nc > ccap)) {
            bcap = std::max(bcap, nb);
            ccap = std::max(ccap, nc);
            continue;
        }
        if (rc == PG_ERR_UNSUPPORTED && !per_reaction) throw UnsupportedError(pg_last_error());
        if (rc != PG_ERR_PANIC && rc != PG_ERR_UNSUPPORTED) check(rc);
        break;
    }
    std::vector<Constructs> res(n_reactions);
    size_t k = 0;
    for (size_t r = 0; r < n_reactions; ++r) {
        item_status(st[r]);
        for (uint64_t j = 0; j < counts[2 * r] + counts[2 * r + 1]; ++j, ++k)
            (kinds[k] == 0 ? res[r].first : res[r].second).emplace_back((const char *)out.data() + off[k], off[k + 1] - off[k]);
    }
    return res;
}
inline std::vector<Constructs> GoldenGateBatch(const std::vector<std::vector<Part>> &reactions, const Enzyme &enzyme) {
    std::vector<std::string> seqs;
    std::vector<uint8_t> circ;
    std::vector<uint64_t> roff{0};
    for (const auto &r : reactions) {
        for (const Part &p : r) { seqs.push_back(p.Sequence); circ.push_back(p.Circular); }
        roff.push_back(seqs.size());
    }
    circ.push_back(0);
    Flat f(seqs);
    const pg_clone_enzyme e = to_pg(enzyme);
    return ligation_outputs(reactions.size(), [&](uint64_t bcap, uint64_t ccap, uint8_t *out, uint64_t *off, uint8_t *kinds, uint64_t *counts,
                                                  int32_t *st, uint64_t *nb, uint64_t *nc) {
        return pg_clone_golden_gate_batch(f.bases.data(), f.offsets.data(), circ.data(), seqs.size(), roff.data(), reactions.size(), &e, bcap, ccap, out,
                                          off, kinds, nullptr, counts, st, nb, nc);
    });
}
inline Constructs GoldenGate(const std::vector<Part> &sequences, const Enzyme &cuttingEnzyme) { return GoldenGateBatch({sequences}, cuttingEnzyme)[0]; }
inline Constructs CircularLigate(const std::vector<Fragment> &fragments) {
    std::vector<std::string> seqs, ohs;
    for (const Fragment &f : fragments) { seqs.push_back(f.Sequence); ohs.push_back(f.ForwardOverhang); ohs.push_back(f.ReverseOverhang); }
    Flat s(seqs), o(ohs);
    const uint64_t roff[2] = {0, fragments.size()};
    return ligation_outputs(1, [&](uint64_t bcap, uint64_t ccap, uint8_t *out, uint64_t *off, uint8_t *kinds, uint64_t *counts, int32_t *st,
                                   uint64_t *nb, uint64_t *nc) {
        st[0] = PG_ITEM_OK;
        return pg_clone_circular_ligate_batch(s.bases.data(), s.offsets.data(), o.bases.data(), o.offsets.data(), fragments.size(), roff, 1, bcap, ccap,
                                              out, off, kinds, nullptr, counts, nb, nc);
    }, false)[0];
}
}  // namespace clone
// ---- fold (fold/fold.go, fold/seqfold.go) over pg_fold_zuker_batch --------------------------------------
namespace fold {
struct UnsupportedError : std::runtime_error {
    using std::runtime_error::runtime_error;
};
// fold.Result: the minimum free energy and dot-bracket of the folded structure (Result{} gives +inf and "")
struct Result {
    double mfe = std::numeric_limits<double>::infinity();
    std::string dot_bracket;
    double MinimumFreeEnergy() const { return mfe; }
    std::string DotBracket() const { return dot_bracket; }
};
// one item of ZukerBatch: status is PG_ITEM_OK, PG_ITEM_FOLD_NOT_NUCLEIC (error holds the reference's message),
// PG_ITEM_PANIC, PG_ITEM_UNSUPPORTED or PG_ITEM_FOLD_INTERNAL
struct Item {
    Result result;
    std::string error;
    int32_t status = PG_ITEM_OK;
};
// Zuker of every sequence in one GPU call
inline std::vector<Item> ZukerBatch(const std::vector<std::string> &seqs, double temp) {
    std::vector<Item> out(seqs.size());
    if (seqs.empty()) return out;
    Flat f(seqs);
    std::vector<double> mfe(seqs.size());
    std::vector<uint8_t> db(std::max<size_t>(f.bases.size(), 1));
    std::vector<uint64_t> len(seqs.size());
    std::vector<int32_t> st(seqs.size());
    const int rc = pg_fold_zuker_batch(f.bases.data(), f.offsets.data(), seqs.size(), temp, mfe.data(), db.data(), len.data(), st.data());
    if (rc != PG_ERR_PANIC && rc != PG_ERR_UNSUPPORTED) check(rc);
    for (size_t i = 0; i < seqs.size(); ++i) {
        out[i].status = st[i];
        if (st[i] == PG_ITEM_OK) {
            out[i].result.mfe = mfe[i];
            out[i].result.dot_bracket.assign((const char *)db.data() + f.offsets[i], len[i]);
        } else if (st[i] == PG_ITEM_FOLD_NOT_NUCLEIC) {
            std::string up = seqs[i];
            for (auto &c : up)
                if (c >= 'a' && c <= 'z') c -= 32;
            out[i].error = "error creating folding context: the sequence " + up + " is not RNA or DNA";
        } else if (st[i] == PG_ITEM_FOLD_INTERNAL) {
            out[i].error = "fold.Zuker: an internal error of the reference fired on this sequence";
        }
    }
    return out;
}
// fold.Zuker (fold.go:56): (Result, error message, empty on success); throws GoPanic where the reference
// panics and UnsupportedError for a byte >= 0x80 or more than PG_FOLD_MAX_LEN nt
inline std::pair<Result, std::string> Zuker(const std::string &seq, double temp) {
    Item it = ZukerBatch({seq}, temp)[0];
    if (it.status == PG_ITEM_PANIC) throw GoPanic("index out of range");
    if (it.status == PG_ITEM_UNSUPPORTED) throw UnsupportedError("a byte >= 0x80 or more than PG_FOLD_MAX_LEN nt (unsupported)");
    return {it.result, it.error};
}
}  // namespace fold
// ---- synthesis/fragment (synthesis/fragment/fragment.go) over pg_fragment_batch and the set entry points ----
namespace fragment {
struct UnsupportedError : std::runtime_error {
    using std::runtime_error::runtime_error;
};
// one item of FragmentWithOverhangsBatch: status is PG_ITEM_OK, PG_ITEM_FRAGMENT_* (error holds the reference's
// message and fragments is empty), PG_ITEM_PANIC or PG_ITEM_UNSUPPORTED
struct Item {
    std::vector<std::string> fragments;
    double efficiency = 0;
    std::string error;
    int32_t status = PG_ITEM_OK;
};
// FragmentWithOverhangs of every sequence in one GPU call (an empty include list is Fragment)
inline std::vector<Item> FragmentWithOverhangsBatch(const std::vector<std::string> &seqs, int64_t minFragmentSize, int64_t maxFragmentSize,
                                                    const std::vector<std::string> &excludeOverhangs,
                                                    const std::vector<std::string> &includeOverhangs) {
    const size_t n = seqs.size();
    std::vector<Item> out(n);
    if (n == 0) return out;
    Flat f(seqs), ex(excludeOverhangs), inc(includeOverhangs);
    ex.bases.push_back(0);
    inc.bases.push_back(0);
    std::vector<int32_t> st(n);
    std::vector<double> eff(n);
    std::vector<int64_t> emin(n), emax(n);
    std::vector<uint64_t> foff(n + 1), ends(f.bases.size() / 8 + 2 * n);
    uint64_t total = 0;
    int rc;
    for (;;) {
        rc = pg_fragment_batch(f.bases.data(), f.offsets.data(), n, minFragmentSize, maxFragmentSize, ex.bases.data(), ex.offsets.data(),
                               excludeOverhangs.size(), inc.bases.data(), inc.offsets.data(), includeOverhangs.size(), st.data(), eff.data(),
                               emin.data(), emax.data(), foff.data(), ends.data(), ends.size(), &total);
        if (rc != PG_ERR_ARG || total <= ends.size()) break;
        ends.resize(total);  // the first guess was too small: once more with the exact count
    }
    if (rc != PG_ERR_PANIC && rc != PG_ERR_UNSUPPORTED) check(rc);
    for (size_t i = 0; i < n; ++i) {
        Item &it = out[i];
        it.status = st[i];
        it.efficiency = eff[i];
        if (st[i] == PG_ITEM_OK) {
            std::string up = seqs[i];
            for (auto &c : up)
                if (c >= 'a' && c <= 'z') c -= 32;
            for (uint64_t j = foff[i]; j < foff[i + 1]; ++j) {
                const uint64_t b = j == foff[i] ? 0 : ends[j - 1] - 4;
                it.fragments.push_back(up.substr(b, ends[j] - b));
            }
        } else if (st[i] == PG_ITEM_FRAGMENT_MIN_GT_MAX) {
            it.error = "minFragmentSize (" + std::to_string(emin[i]) + ") larger than maxFragmentSize (" + std::to_string(emax[i]) + ")";
        } else if (st[i] == PG_ITEM_FRAGMENT_MIN_LT_12) {
            it.error = "minFragmentSize must be equal to or greater than 12 . Got size of " + std::to_string(emin[i]);
        } else if (st[i] == PG_ITEM_FRAGMENT_NO_POSITION) {
            it.error = "bestOverhangPosition failed by equaling zero";
        }
    }
    return out;
}
inline std::vector<Item> FragmentBatch(const std::vector<std::string> &seqs, int64_t minFragmentSize, int64_t maxFragmentSize,
                                       const std::vector<std::string> &excludeOverhangs) {
    return FragmentWithOverhangsBatch(seqs, minFragmentSize, maxFragmentSize, excludeOverhangs, {});
}
// fragment.FragmentWithOverhangs (fragment.go:199): (fragments, efficiency, error message, empty on success);
// throws GoPanic where the reference panics (fewer than 4 bytes) and UnsupportedError for a byte >= 0x80
struct Fragments {
    std::vector<std::string> fragments;
    double efficiency;
    std::string error;
};
inline Fragments FragmentWithOverhangs(const std::string &sequence, int64_t minFragmentSize, int64_t maxFragmentSize,
                                       const std::vector<std::string> &excludeOverhangs, const std::vector<std::string> &includeOverhangs) {
    Item it = FragmentWithOverhangsBatch({sequence}, minFragmentSize, maxFragmentSize, excludeOverhangs, includeOverhangs)[0];
    if (it.status == PG_ITEM_PANIC) throw GoPanic("slice bounds out of range");
    if (it.status == PG_ITEM_UNSUPPORTED) throw UnsupportedError("a byte >= 0x80 (unsupported)");
    return {it.fragments, it.efficiency, it.error};
}
// fragment.Fragment (fragment.go:191)
inline Fragments Fragment(const std::string &sequence, int64_t minFragmentSize, int64_t maxFragmentSize,
                          const std::vector<std::string> &excludeOverhangs) {
    return FragmentWithOverhangs(sequence, minFragmentSize, maxFragmentSize, excludeOverhangs, {});
}
namespace detail {
struct Sets {
    std::vector<uint8_t> bases;
    std::vector<uint64_t> offsets, set_offsets{0};
    explicit Sets(const std::vector<std::vector<std::string>> &sets) {
        std::vector<std::string> all;
        for (auto &s : sets) {
            all.insert(all.end(), s.begin(), s.end());
            set_offsets.push_back(all.size());
        }
        Flat f(all);
        bases = std::move(f.bases);
        bases.push_back(0);
        offsets = std::move(f.offsets);
    }
};
}  // namespace detail
// SetEfficiency of every set in one GPU call
inline std::vector<double> SetEfficiencyBatch(const std::vector<std::vector<std::string>> &sets) {
    std::vector<double> eff(sets.size());
    if (sets.empty()) return eff;
    detail::Sets s(sets);
    check(pg_fragment_set_efficiency_batch(s.bases.data(), s.offsets.data(), s.set_offsets.data(), sets.size(), eff.data()));
    return eff;
}
// fragment.SetEfficiency (fragment.go:24)
inline double SetEfficiency(const std::vector<std::string> &overhangs) { return SetEfficiencyBatch({overhangs})[0]; }
// NextOverhangs of every set in one GPU call: (candidates, efficiencies) per set
inline std::vector<std::pair<std::vector<std::string>, std::vector<double>>> NextOverhangsBatch(const std::vector<std::vector<std::string>> &sets) {
    std::vector<std::pair<std::vector<std::string>, std::vector<double>>> out(sets.size());
    if (sets.empty()) return out;
    detail::Sets s(sets);
    std::vector<uint8_t> cands(1024 * sets.size());
    std::vector<uint32_t> nc(sets.size());
    std::vector<double> eff(256 * sets.size());
    check(pg_fragment_next_overhangs_batch(s.bases.data(), s.offsets.data(), s.set_offsets.data(), sets.size(), cands.data(), nc.data(), eff.data()));
    for (size_t i = 0; i < sets.size(); ++i)
        for (uint32_t j = 0; j < nc[i]; ++j) {
            out[i].first.emplace_back((const char *)cands.data() + 1024 * i + 4 * j, 4);
            out[i].second.push_back(eff[256 * i + j]);
        }
    return out;
}
// fragment.NextOverhangs (fragment.go:43)
inline std::pair<std::vector<std::string>, std::vector<double>> NextOverhangs(const std::vector<std::string> &currentOverhangs) {
    return NextOverhangsBatch({currentOverhangs})[0];
}
// fragment.NextOverhang (fragment.go:85): the first strict maximum above 0, or ""
inline std::string NextOverhang(const std::vector<std::string> &currentOverhangs) {
    const auto r = NextOverhangs(currentOverhangs);
    double best = 0;
    std::string pick;
    for (size_t i = 0; i < r.first.size(); ++i)
        if (r.second[i] > best) {
            best = r.second[i];
            pick = r.first[i];
        }
    return pick;
}
}  // namespace fragment
}  // namespace poly
