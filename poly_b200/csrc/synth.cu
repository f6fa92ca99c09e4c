// synth.cu -- device generators for the synthetic workloads of SURVEY.md 8d (bench and
// test tooling; byte-identical to poly_b200/synth.py).  Not a reference API.
#include <algorithm>

#include "common.cuh"

namespace pg {

namespace {

__device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
    uint64_t z = x + 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
__device__ __forceinline__ uint32_t code_at(uint64_t seed, uint64_t g) {
    return (uint32_t)(splitmix64(seed + (g >> 5)) >> (2 * (g & 31))) & 3u;
}
__device__ __forceinline__ uint8_t acgt(uint32_t c) { return (uint8_t)("ACGT"[c]); }

// kind 0: 32 bases (one splitmix word) per thread-iteration
__global__ void synth_independent_kernel(uint8_t *__restrict__ out, uint64_t g0, uint64_t count,
                                         uint64_t seed) {
    // word w covers global bases [32w, 32w+32)
    const uint64_t w_first = g0 >> 5, w_last = (g0 + count - 1) >> 5;
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t w = w_first + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; w <= w_last;
         w += stride) {
        const uint64_t bits = splitmix64(seed + w);
        const uint64_t gb = w << 5;
        if (gb >= g0 && gb + 32 <= g0 + count && ((uintptr_t)(out + (gb - g0)) & 15u) == 0) {
            uint32_t v[8];
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                uint32_t x = 0;
#pragma unroll
                for (int b = 0; b < 4; ++b)
                    x |= (uint32_t)acgt((uint32_t)(bits >> (2 * (4 * q + b))) & 3u) << (8 * b);
                v[q] = x;
            }
            uint4 *dst = reinterpret_cast<uint4 *>(out + (gb - g0));
            dst[0] = make_uint4(v[0], v[1], v[2], v[3]);
            dst[1] = make_uint4(v[4], v[5], v[6], v[7]);
        } else {
            for (int b = 0; b < 32; ++b) {
                const uint64_t g = gb + b;
                if (g >= g0 && g < g0 + count) out[g - g0] = acgt((uint32_t)(bits >> (2 * b)) & 3u);
            }
        }
    }
}

// kind 1: family reads (template shared by `family` consecutive reads, 1/64 substitutions)
__global__ void synth_family_kernel(uint8_t *__restrict__ out, uint64_t first_read, uint64_t n_reads,
                                    uint32_t L, uint64_t seed, uint32_t family) {
    const uint64_t total = n_reads * (uint64_t)L;
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t x = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; x < total; x += stride) {
        const uint64_t i = first_read + x / L;
        const uint64_t j = x % L;
        const uint64_t t = i / family;
        const uint32_t T = code_at(seed, t * L + j);
        const uint64_t m = splitmix64((seed ^ 0xD157ull) + i * L + j);
        const uint32_t c = (m & 63) == 0 ? (T + 1 + (uint32_t)((m >> 6) % 3)) & 3u : T;
        out[x] = acgt(c);
    }
}

}  // namespace

int launch_synth_reads(uint8_t *d_bases, uint64_t first_read, uint64_t n_reads, uint32_t read_len,
                       uint64_t seed, int kind, uint32_t family, cudaStream_t st) {
    if (n_reads == 0 || read_len == 0) return PG_OK;
    const uint64_t count = n_reads * (uint64_t)read_len;
    if (kind == 0) {
        const uint64_t words = (count >> 5) + 2;
        const unsigned blocks = (unsigned)std::min<uint64_t>((words + 255) / 256, (uint64_t)sm_count() * 32);
        synth_independent_kernel<<<blocks, 256, 0, st>>>(d_bases, first_read * read_len, count, seed);
        PG_LAUNCH_CHECK("synth_independent_kernel");
    } else if (kind == 1) {
        if (family == 0) { set_error("family must be > 0"); return PG_ERR_ARG; }
        const unsigned blocks = (unsigned)std::min<uint64_t>((count + 255) / 256, (uint64_t)sm_count() * 32);
        synth_family_kernel<<<blocks, 256, 0, st>>>(d_bases, first_read, n_reads, read_len, seed, family);
        PG_LAUNCH_CHECK("synth_family_kernel");
    } else {
        set_error("unknown synthetic kind %d", kind);
        return PG_ERR_ARG;
    }
    return PG_OK;
}

}  // namespace pg
