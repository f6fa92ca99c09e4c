// tools/pipe_bench.cu -- measures issue throughput (cycles per warp instruction per SMSP)
// of the integer instructions K1 is made of, on the GPU this runs on.  Evidence for the
// pipe-balancing choices in DESIGN.md ("K1: integer-issue co-limit").
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o pipe_bench pipe_bench.cu
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

#define ITERS 4096
#define ILP 8

template <int OP>
__device__ __forceinline__ uint32_t op(uint32_t x, uint32_t a, uint32_t b) {
    uint32_t r;
    if (OP == 0) r = __funnelshift_l(x, x, 13);                       // SHF.L.W
    else if (OP == 1) r = x ^ a;                                      // LOP3
    else if (OP == 2) r = x * 0xcc9e2d51u;                            // IMAD imm
    else if (OP == 3) r = x * a + b;                                  // IMAD reg
    else if (OP == 4) r = __umulhi(x, a);                             // IMAD.HI.U32 reg
    else if (OP == 5) r = x + a;                                      // IADD3 / IMAD.IADD
    else if (OP == 6) r = __byte_perm(x, a, 0x2103);                  // PRMT
    else if (OP == 7) r = x * 5u + 0xe6546b64u;                       // IMAD reg(5)+imm
    else if (OP == 8) { uint64_t w = (uint64_t)x * a; r = (uint32_t)w + (uint32_t)(w >> 32); }  // IMAD.WIDE + add
    else if (OP == 9) r = (x >> 16) ^ x;                              // SHF + LOP3 (fmix step)
    else if (OP == 10) r = __umulhi(x, a) ^ x;                        // IMAD.HI + LOP3
    else if (OP == 11) r = __funnelshift_l(x ^ a, x ^ a, 13) * 5u + 0xe6546b64u;  // body round: LOP3+SHF+IMAD
    else if (OP == 12) { uint32_t y = x ^ a; r = __umulhi(y, b) * 5u + (y * 40960u + 0xe6546b64u); } // LOP3 + 3 fma
    else r = x;
    return r;
}

template <int OP>
__global__ void bench(uint32_t *out, uint32_t a, uint32_t b, long long *cycles) {
    uint32_t v[ILP];
#pragma unroll
    for (int i = 0; i < ILP; ++i) v[i] = threadIdx.x * 7919u + i * 104729u + a;
    __syncthreads();
    long long t0 = clock64();
#pragma unroll 1
    for (int it = 0; it < ITERS; ++it) {
#pragma unroll
        for (int u = 0; u < 4; ++u)
#pragma unroll
            for (int i = 0; i < ILP; ++i) v[i] = op<OP>(v[i], a, b);
    }
    long long t1 = clock64();
    uint32_t s = 0;
#pragma unroll
    for (int i = 0; i < ILP; ++i) s ^= v[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
    if (threadIdx.x == 0 && blockIdx.x == 0) *cycles = t1 - t0;
}

template <int OP>
void run(const char *name, int n_instr_per_op, int warps_per_smsp) {
    uint32_t *out; long long *cyc, h;
    int threads = 128 * warps_per_smsp, sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    cudaMalloc(&out, (size_t)sms * threads * 4); cudaMalloc(&cyc, 8);
    bench<OP><<<sms, threads>>>(out, 0x10000u, 0x2000u, cyc);
    bench<OP><<<sms, threads>>>(out, 0x10000u, 0x2000u, cyc);
    cudaMemcpy(&h, cyc, 8, cudaMemcpyDeviceToHost);
    double ops = (double)ITERS * 4 * ILP * warps_per_smsp;  // op<> calls per SMSP
    printf("%-34s warps/SMSP=%d  %.3f cyc per op  (%.3f cyc per SASS instr if %d instr/op)\n", name, warps_per_smsp,
           h / ops, h / ops / n_instr_per_op, n_instr_per_op);
    cudaFree(out); cudaFree(cyc);
}

int main() {
    for (int w : {1, 4}) {
        run<0>("SHF.L.W (rotl)", 1, w);
        run<1>("LOP3 (xor reg)", 1, w);
        run<2>("IMAD x*imm", 1, w);
        run<3>("IMAD x*reg+reg", 1, w);
        run<4>("IMAD.HI.U32 x*reg", 1, w);
        run<5>("IADD", 1, w);
        run<6>("PRMT", 1, w);
        run<7>("IMAD x*5+imm", 1, w);
        run<8>("IMAD.WIDE + IADD (rotl via mul)", 2, w);
        run<9>("SHF.R + LOP3 (fmix step)", 2, w);
        run<10>("IMAD.HI + LOP3 (fmix step, fma)", 2, w);
        run<11>("body round LOP3+SHF+IMAD", 3, w);
        run<12>("body round LOP3+IMAD.HI+2 IMAD", 4, w);
    }
    return 0;
}
