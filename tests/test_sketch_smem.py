"""CPU tier: the shared-memory layouts of the sketch kernels (poly_b200/csrc/sketch_smem.cuh), compiled on the host
with nvcc.  Every launcher sizes its launch and every kernel carves its memory from one layout; this checks the
layouts against the sizes the launchers used before they existed (restated below), that every TMA stage buffer
starts on a 16-byte boundary, that the regions do not overlap, and the list of walk k values."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "poly_b200", "csrc")

PROGRAM = r"""
#include <cstdio>
#include <vector>
#include "kmer_walk.cuh"
#include "sketch_smem.cuh"
using namespace pg;

static long fails = 0, checks = 0;
#define CHECK(c, ...) do { ++checks; if (!(c)) { if (fails++ < 20) { std::printf("FAIL %s: ", #c); std::printf(__VA_ARGS__); std::printf("\n"); } } } while (0)

// SelSmem kernels: the carve agrees with the offsets, regions are in order and large enough, stages are aligned
static void sel_regions(const SelLayout &l, uint32_t cap, uint32_t keep_need, uint32_t kv_need, uint32_t stage_need,
                        uint32_t misc_need, const char *what, uint32_t s) {
    std::vector<uint32_t> w(l.bytes() / 4);
    const SelSmem m = l.carve(w.data());
    CHECK(m.cand == w.data() && m.keep - m.cand == (long)cap, "%s s=%u", what, s);
    CHECK(m.kv - m.cand == (long)l.kv() && m.bytes - m.cand == (long)l.stage() && m.hist - m.cand == (long)l.hist() &&
          m.misc - m.cand == (long)(l.hist() + SEL_NBK + 1) && m.tmpcap == l.hist() - cap, "%s s=%u: carve vs offsets", what, s);
    CHECK(l.kv() - cap >= keep_need && l.stage() - l.kv() >= kv_need && l.hist() - l.stage() >= 2 * (size_t)stage_need &&
          l.bytes() / 4 - (l.hist() + SEL_NBK + 1) >= misc_need, "%s s=%u cap=%u: region sizes", what, s, cap);
    if (stage_need)
        CHECK(l.stage() % 4 == 0 && (l.stage() + l.stage_w) % 4 == 0, "%s s=%u cap=%u: stage alignment", what, s, cap);
}

int main() {
    // the walk k list
    std::vector<int> ks;
    for (int k = -4; k <= 2048; ++k) {
        int seen = -1;
        if (with_walk_k(k, [&](auto kk) { seen = decltype(kk)::value; })) ks.push_back(seen);
        CHECK(seen == -1 || seen == k, "k=%d dispatched as %d", k, seen);
    }
    const std::vector<int> want{11, 13, 15, 16, 17, 19, 21, 23, 24, 25, 27, 29, 31, 32};
    CHECK(ks == want, "walk k list has %zu entries", ks.size());

    // K2t stage A, per listed k: 2 stage buffers | strip [SEG][32]
    auto geom = [&](auto kk) {
        constexpr int K = decltype(kk)::value;
        using G = SeltGeom<K>;
        CHECK(G::SMEM_BYTES == 2 * (size_t)G::STAGE + (size_t)G::SEG * 32 * 4, "K2t A k=%d bytes", K);
        CHECK(G::STAGE % 16 == 0 && G::STRIP * 4 == 2 * (uint32_t)G::STAGE, "K2t A k=%d stage alignment", K);
        CHECK((uint32_t)G::STAGE >= 15 + G::CHUNK + K + 32, "K2t A k=%d stage holds head + chunk + k + pad", K);
    };
    for (int k : want) with_walk_k(k, geom);

    for (uint32_t s = 1; s <= 16384; ++s) {
        uint32_t P = 1;
        while (P < s) P <<= 1;
        if (P < 2) P = 2;
        const uint32_t s4 = ((s + 3u) & ~3u);
        // the launchers' cap (max(P, s + 8192) in 16-byte granules, all three) and other multiples of 4
        for (uint32_t room : {8192u, 0u, 4u, 1000u}) {
            const uint32_t cap = ((P > s + room ? P : s + room) + 3u) & ~3u;
            const SelLayout g = sel_generic_layout(cap, s), w = sel_walk_layout(cap, s), m = sel_merge_layout(cap, s);
            CHECK(g.bytes() == ((size_t)cap + (((size_t)s + 3) & ~(size_t)3) + 4 + (2048 + 1024) + 2 * ((15 + 2048 + 1024 + 32 + 15) / 16 * 4) + (2048 + 1) + 8) * 4,
                  "generic s=%u cap=%u", s, cap);
            CHECK(w.bytes() == ((size_t)cap + (((size_t)s + 3) & ~(size_t)3) + 4 + 2 * ((15 + 5120 + 32 + 48 + 15) / 16 * 4) + (2048 + 1) + 16) * 4, "K2w s=%u cap=%u", s, cap);
            CHECK(m.bytes() == ((size_t)cap + s + 2048 + 64 + 2048 + 1 + 8) * 4, "merge s=%u cap=%u", s, cap);
            sel_regions(g, cap, s4, SEL_CHUNK + SEL_LOOKAHEAD, SEL_STAGE_WORDS, 8, "generic", s);
            sel_regions(w, cap, s4, 0, SELW_STAGE_WORDS, SELW_CHUNK_CTR + 3, "K2w", s);
            sel_regions(m, cap, s + SEL_NBK + 64, 0, 0, 8, "merge", s);
        }
        // K2t stage B: the cap of launch_select_thresh, and every cap near it (multiple of 4 or not)
        const uint32_t mu = s + 6u * (uint32_t)__builtin_ceil(__builtin_sqrt((double)s)) + 48u;
        const uint32_t cap0 = ((mu + 8u * (uint32_t)__builtin_ceil(__builtin_sqrt((double)mu)) + 96u) + 3u) & ~3u;
        for (uint32_t cap = cap0 - 3; cap <= cap0 + 3; ++cap) {
            const SeltSelLayout b(cap);
            CHECK(b.bytes() == ((((size_t)cap + 3) & ~(size_t)3) + 2048 + 16) * 4, "K2t B cap=%u", cap);
            CHECK(b.tmp == 0 && b.cur >= cap && b.cur % 4 == 0 && b.flag == b.cur + SEL_NBK && b.words > b.flag, "K2t B cap=%u regions", cap);
            CHECK(b.bytes() <= 80 * 1024, "K2t B s=%u cap=%u: %zu bytes of shared memory", s, cap, b.bytes());
        }
    }
    // K1: 2 input stages | out tile [32][nk]
    for (uint32_t L = 1; L <= 4096; ++L)
        for (uint32_t nk : {1u, 7u, L, 3u * L + 1}) {
            CHECK(k1_smem_bytes(L, nk) == 2 * (size_t)((32u * L + 16u + 15u) & ~15u) + (size_t)32 * nk * 4, "K1 L=%u nk=%u", L, nk);
            CHECK(k1_in_bytes(L) % 16 == 0 && k1_in_bytes(L) >= 32 * L + 16, "K1 L=%u stage", L);
        }
    // K1r: input stage [in_cap bytes] | out tile [32][stride]
    for (uint64_t len = 0; len <= 2048; ++len) {
        const uint64_t in_cap = k1r_in_bytes(len);
        CHECK(in_cap == ((32 * len + 48 + 15) & ~15ull) && in_cap % 16 == 0 && in_cap >= 32 * len + 47, "K1r len=%llu", (unsigned long long)len);
        for (uint32_t stride : {1u, 5u, 129u, 768u})
            CHECK(k1r_smem_bytes((uint32_t)in_cap, stride) == in_cap + (size_t)32 * stride * 4, "K1r len=%llu stride=%u", (unsigned long long)len, stride);
    }
    std::printf("checks %ld fails %ld\n", checks, fails);
    return fails != 0;
}
"""


def nvcc():
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    pytest.fail("nvcc not found: the layout header is checked by compiling it")


def test_sketch_smem_layouts(tmp_path):
    src = tmp_path / "layouts.cu"
    src.write_text(PROGRAM)
    exe = tmp_path / "layouts"
    subprocess.run([nvcc(), "-std=c++17", "-O1", "--expt-relaxed-constexpr", "-gencode", "arch=compute_90a,code=sm_90a",
                    "-I", CSRC, str(src), "-o", str(exe)], check=True, capture_output=True, text=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout
    assert "fails 0" in out.stdout and int(out.stdout.split()[1]) > 1_000_000, out.stdout
