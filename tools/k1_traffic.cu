// tools/k1_traffic.cu -- K1's memory traffic without its hashing: the least time the headline's
// loads and stores take, in today's structure and in pipelined ones.  Evidence for DESIGN.md "K1".
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o k1_traffic k1_traffic.cu
//
// Shape of bench.py's headline: 10 M reads x 150 B in by 1-D TMA bulk loads, 10 M x 129 u32 out by
// bulk stores of whole [tile][129] output tiles, k = 21.  Each lane writes the words K1 would write
// (value: the read's first byte + position) into the staged output tile; there is no murmur3.
//   today:      one-warp CTA per 32-read tile: load -> wait -> write -> store -> wait for the read-out.
//   pipelined:  persistent warps, IN input stages (next tile's load in flight while the current one
//               is written) and OUT output tiles (a store is waited for only before its buffer is reused).
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <algorithm>
#include <vector>
#include <cuda_runtime.h>

#include "../poly_b200/csrc/tma.cuh"

using namespace pg;

#define CK(x)                                                                                   \
    do {                                                                                        \
        cudaError_t e_ = (x);                                                                   \
        if (e_ != cudaSuccess) {                                                                \
            fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_)); \
            exit(1);                                                                            \
        }                                                                                       \
    } while (0)

template <int N>
__device__ __forceinline__ void wait_read() {  // at most N bulk groups still reading shared memory
    asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}

__host__ __device__ constexpr uint32_t stage_bytes(uint32_t tile, uint32_t L) { return (tile * L + 16u + 15u) & ~15u; }

// W warps per CTA, TILE reads per tile (32 / TILE lanes per read), IN input stages, OUT output tiles.
template <int W, int TILE, int IN, int OUT>
__global__ void __launch_bounds__(W * 32)
traffic_kernel(const uint8_t *__restrict__ in, uint32_t *__restrict__ out, uint32_t L, uint32_t nk, uint64_t n_tiles) {
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ __align__(8) uint64_t s_bar[W * IN];
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    const uint32_t in_stage = stage_bytes(TILE, L), in_bytes = TILE * L, out_words = TILE * nk;
    uint8_t *s_in = smem + warp * (IN * in_stage + OUT * out_words * 4u);
    uint32_t *s_out = reinterpret_cast<uint32_t *>(s_in + IN * in_stage);
    uint64_t *bar = s_bar + warp * IN;
    const uint64_t stride = (uint64_t)gridDim.x * W;
    uint64_t t = (uint64_t)blockIdx.x * W + warp;
    if (threadIdx.x == 0) {
        for (int b = 0; b < W * IN; ++b) mbar_init(&s_bar[b], 1);
        fence_mbar_init();
    }
    __syncthreads();
    if (lane == 0)
        for (int j = 0; j + 1 < IN; ++j)
            if (t + j * stride < n_tiles) {
                mbar_expect_tx(&bar[j], in_bytes);
                bulk_g2s(s_in + j * in_stage, in + (t + j * stride) * in_bytes, in_bytes, &bar[j]);
            }
    // the words of my read that K1 gives this lane: all of them, or one half
    const uint32_t half = (nk + 1) / 2;
    const uint32_t beg = TILE == 32 || lane < TILE ? 0u : half;
    const uint32_t cnt = TILE == 32 ? nk : lane < TILE ? half : nk - half;
    for (uint32_t c = 0; t < n_tiles; t += stride, ++c) {
        if (lane == 0) {
            const uint64_t next = t + (IN - 1) * stride;
            const uint32_t sn = (c + IN - 1) % IN;
            if (next < n_tiles) {
                mbar_expect_tx(&bar[sn], in_bytes);
                bulk_g2s(s_in + sn * in_stage, in + next * in_bytes, in_bytes, &bar[sn]);
            }
        }
        mbar_wait(&bar[c % IN], (c / IN) & 1u);
        if (lane == 0) wait_read<OUT - 1>();
        __syncwarp();
        const uint32_t read = lane % TILE;
        const uint32_t v = s_in[(c % IN) * in_stage + read * L];
        uint32_t *o = s_out + (c % OUT) * out_words + read * nk + beg;
        for (uint32_t i = 0; i < cnt; ++i) o[i] = v + beg + i;
        fence_async_smem();
        __syncwarp();
        if (lane == 0) bulk_s2g(out + t * out_words, s_out + (c % OUT) * out_words, out_words * 4u);
    }
    if (lane == 0) wait_read<0>();
}

__global__ void fill_reads(uint8_t *p, size_t n) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        uint32_t x = (uint32_t)(i * 2654435761u) ^ (uint32_t)(i >> 13);
        x ^= x >> 15;
        x *= 0x2c1b3c6du;
        x ^= x >> 12;
        p[i] = "ACGT"[x & 3];
    }
}

int main(int argc, char **argv) {
    const uint64_t N = 10000000;
    const uint32_t L = 150, nk = L - 21;
    const int launches = argc > 1 ? atoi(argv[1]) : 50, warmup = 5;
    int sms;
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    uint8_t *d_in;
    uint32_t *d_out;
    CK(cudaMalloc(&d_in, N * L));
    CK(cudaMalloc(&d_out, N * nk * 4));
    fill_reads<<<4096, 256>>>(d_in, N * L);
    CK(cudaGetLastError());
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    const double bytes = (double)N * L + (double)N * nk * 4;  // algorithmic: every input byte read once, every hash written once
    printf("{\"device\": \"%s\", \"sms\": %d, \"reads\": %llu, \"read_len\": %u, \"words_per_read\": %u, \"bytes_per_launch\": %.0f, \"launches\": %d}\n",
           prop.name, sms, (unsigned long long)N, L, nk, bytes, launches);

    auto run = [&](auto kern, int W, int TILE, int IN, int OUT, bool persistent, const char *name) {
        const uint64_t tiles = N / TILE;
        const size_t smem = (size_t)W * (IN * stage_bytes(TILE, L) + OUT * TILE * nk * 4);
        CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        int per_sm = 0;
        CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, W * 32, smem));
        uint64_t grid = (tiles + W - 1) / W;
        if (persistent) grid = std::min<uint64_t>(grid, (uint64_t)sms * per_sm);
        CK(cudaMemset(d_out, 0, N * nk * 4));
        for (int i = 0; i < warmup; ++i) kern<<<(unsigned)grid, W * 32, smem>>>(d_in, d_out, L, nk, tiles);
        CK(cudaGetLastError());
        CK(cudaDeviceSynchronize());
        std::vector<float> ms(launches);
        for (int i = 0; i < launches; ++i) {
            CK(cudaEventRecord(e0));
            kern<<<(unsigned)grid, W * 32, smem>>>(d_in, d_out, L, nk, tiles);
            CK(cudaEventRecord(e1));
            CK(cudaEventSynchronize(e1));
            CK(cudaEventElapsedTime(&ms[i], e0, e1));
        }
        // the first and last 64 rows hold what the kernel was asked to write
        std::vector<uint32_t> h(64 * nk);
        bool ok = true;
        for (uint64_t r0 : {(uint64_t)0, N - 64}) {
            CK(cudaMemcpy(h.data(), d_out + r0 * nk, h.size() * 4, cudaMemcpyDeviceToHost));
            std::vector<uint8_t> hi(64 * L);
            CK(cudaMemcpy(hi.data(), d_in + r0 * L, hi.size(), cudaMemcpyDeviceToHost));
            for (uint32_t r = 0; r < 64; ++r)
                for (uint32_t i = 0; i < nk; ++i) ok = ok && h[r * nk + i] == hi[r * L] + i;
        }
        std::sort(ms.begin(), ms.end());
        const float med = ms[launches / 2];
        printf("{\"structure\": \"%s\", \"warps_per_cta\": %d, \"reads_per_tile\": %d, \"in_stages\": %d, \"out_tiles\": %d, "
               "\"smem_per_cta\": %zu, \"ctas_per_sm\": %d, \"grid\": %llu, \"ms_median\": %.4f, \"ms_min\": %.4f, \"ms_max\": %.4f, "
               "\"GBps_median\": %.1f, \"output_ok\": %s}\n",
               name, W, TILE, IN, OUT, smem, per_sm, (unsigned long long)grid, med, ms[0], ms[launches - 1], bytes / med / 1e6,
               ok ? "true" : "false");
        fflush(stdout);
        return ok;
    };
    bool ok = true;
    for (int rep = 0; rep < 2; ++rep) {
        ok &= run(traffic_kernel<1, 32, 1, 1>, 1, 32, 1, 1, false, "today");
        ok &= run(traffic_kernel<2, 16, 2, 2>, 2, 16, 2, 2, true, "pipelined");
        ok &= run(traffic_kernel<1, 32, 2, 1>, 1, 32, 2, 1, true, "pipelined");
    }
    CK(cudaFree(d_in));
    CK(cudaFree(d_out));
    return ok ? 0 : 1;
}
