// tm.cu -- K5: primers.SantaLucia / MeltingTemp, one thread per primer,
// /root/reference/primers/primers.go:70-105 (and :121-128 for the defaults), with
// transform.ReverseComplement's byte table (transform/transform.go:15-23,78-109) for
// the self-complementarity test.  float64 throughout, accumulated in the reference's
// statement order; this file is compiled with -fmad=false so that no add/multiply pair
// is contracted into an FMA the Go compiler would not emit on amd64.  The three logs of a
// (cp, na, mg) triple are taken once on the host with libm's log (tm_logs), so the kernels
// hold only IEEE + * / and their Tm, dH and dS are bit for bit the host's.  CUDA's double
// log (<= 1 ulp) differs from glibc's in the last bit for some arguments (DESIGN.md, K5), and
// a Tm one ulp off moves DesignPrimers and SimulateSimple when a target sits on a candidate's Tm.
#include <algorithm>

#include "common.cuh"

namespace pg {

namespace {

// nearest-neighbour table primers.go:42-59, indexed [4*ix+iy] with A,C,G,T = 0..3
__constant__ double c_nn_h[16] = {
    /*AA*/ -7.6, /*AC*/ -8.4, /*AG*/ -7.8, /*AT*/ -7.2,
    /*CA*/ -8.5, /*CC*/ -8.0, /*CG*/ -10.6, /*CT*/ -7.8,
    /*GA*/ -8.2, /*GC*/ -9.8, /*GG*/ -8.0, /*GT*/ -8.4,
    /*TA*/ -7.2, /*TC*/ -8.2, /*TG*/ -8.5, /*TT*/ -7.6};
__constant__ double c_nn_s[16] = {
    /*AA*/ -21.3, /*AC*/ -22.4, /*AG*/ -21.0, /*AT*/ -20.4,
    /*CA*/ -22.7, /*CC*/ -19.9, /*CG*/ -27.2, /*CT*/ -21.0,
    /*GA*/ -22.2, /*GC*/ -24.4, /*GG*/ -19.9, /*GT*/ -22.4,
    /*TA*/ -21.3, /*TC*/ -22.2, /*TG*/ -22.7, /*TT*/ -21.3};

__device__ __forceinline__ int nt_index(uint8_t c) {
    return c == 'A' ? 0 : c == 'C' ? 1 : c == 'G' ? 2 : c == 'T' ? 3 : -1;
}
__device__ __forceinline__ uint8_t upper(uint8_t c) {  // strings.ToUpper on ASCII
    return (c >= 'a' && c <= 'z') ? (uint8_t)(c - 32) : c;
}
// complementTable (transform.go:78-109) restricted to upper-case input: other bytes -> 0
__device__ __forceinline__ uint8_t complement_upper(uint8_t c) {
    switch (c) {
        case 'A': return 'T'; case 'B': return 'V'; case 'C': return 'G'; case 'D': return 'H';
        case 'G': return 'C'; case 'H': return 'D'; case 'K': return 'M'; case 'M': return 'K';
        case 'N': return 'N'; case 'R': return 'Y'; case 'S': return 'S'; case 'T': return 'A';
        case 'V': return 'B'; case 'W': return 'W'; case 'Y': return 'R';
        default: return 0;
    }
}

// The logs of primers.go:95 and :103, the reference's own expressions evaluated on the host.
struct TmLogs {
    double salt;  // log(saltConcentration + (magnesiumConcentration * 140))
    double cp1;   // log(primerConcentration / symmetryFactor), symmetryFactor = 1 (self-complementary)
    double cp4;   // symmetryFactor = 4
};
TmLogs tm_logs(double cp, double na, double mg) { return {log(na + (mg * 140)), log(cp / 1), log(cp / 4)}; }
TmLogs melting_temp_logs() { return tm_logs(500e-9, 50e-3, 0.0); }  // MeltingTemp's defaults, primers.go:122-124

// primers.SantaLucia over an accessor get(j) -> j-th byte of the (already upper-cased) sequence;
// statement order of primers.go:70-105.  len >= 1.
template <typename Get>
__device__ __forceinline__ double santalucia_core(Get get, uint64_t len, const TmLogs &lg, double *dh_out,
                                                  double *ds_out) {
    bool pal = true;
    for (uint64_t j = 0; j < len; ++j) pal &= get(j) == complement_upper(get(len - 1 - j));  // primers.go:81
    const double gas_constant = 1.9872;  // primers.go:73
    double dH = 0.0, dS = 0.0, log_cp;
    dH += 0.2;   // primers.go:78
    dS += -5.7;  // primers.go:79
    if (pal) {   // primers.go:81-87
        dH += 0.0;
        dS += -1.4;
        log_cp = lg.cp1;
    } else {
        log_cp = lg.cp4;
    }
    const uint8_t last = get(len - 1);
    if (last == 'A' || last == 'T') {  // primers.go:89-92
        dH += 2.2;
        dS += 6.9;
    }
    dS += (0.368 * (double)(int64_t)(len - 1) * lg.salt);      // primers.go:94-95
    int px = nt_index(get(0));
    for (uint64_t j = 0; j + 1 < len; ++j) {                   // primers.go:97-101
        const int py = nt_index(get(j + 1));
        double H = 0.0, S = 0.0;                               // absent key -> {0,0}
        if (px >= 0 && py >= 0) { H = c_nn_h[4 * px + py]; S = c_nn_s[4 * px + py]; }
        dH += H;
        dS += S;
        px = py;
    }
    if (dh_out) *dh_out = dH;
    if (ds_out) *ds_out = dS;
    return dH * 1000 / (dS + gas_constant * log_cp) - 273.15;  // primers.go:103
}

__global__ void __launch_bounds__(256)
tm_kernel(const uint8_t *__restrict__ bases, const uint64_t *__restrict__ off, uint64_t n,
          TmLogs lg, double *__restrict__ tm, double *__restrict__ dh,
          double *__restrict__ ds, int32_t *__restrict__ status) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t beg = off[i];
    const uint64_t len = off[i + 1] - beg;
    const uint8_t *s = bases + beg;
    if (len == 0) {  // primers.go:89 sequence[len(sequence)-1]
        if (status) status[i] = PG_ITEM_PANIC;
        return;
    }
    bool ascii = true;
    for (uint64_t j = 0; j < len; ++j) ascii &= __ldg(s + j) < 0x80;
    if (!ascii) {
        if (status) status[i] = PG_ITEM_UNSUPPORTED;
        return;
    }
    double dH, dS;
    const double t = santalucia_core([s](uint64_t j) { return upper(__ldg(s + j)); }, len, lg, &dH, &dS);
    if (tm) tm[i] = t;
    if (dh) dh[i] = dH;
    if (ds) ds[i] = dS;
    if (status) status[i] = PG_ITEM_OK;
}

// pcr.DesignPrimersWithOverhangs core, /root/reference/primers/pcr/pcr.go:44-60 (SURVEY 8f.3):
// thread 2g   : forward primer = shortest prefix of >= 15 nt of the upper-cased sequence whose
//               MeltingTemp reaches the target (pcr.go:46-49);
// thread 2g+1 : reverse primer = reverse complement of the shortest such suffix (pcr.go:50-53).
// Every candidate is evaluated from scratch exactly as MeltingTemp would (same summation order).
// The reference slices past the end (panic) when the sequence is shorter than 15 nt or is
// exhausted before the target is reached.
__global__ void __launch_bounds__(256)
design_primers_kernel(const uint8_t *__restrict__ bases, const uint64_t *__restrict__ off, uint64_t n,
                      TmLogs lg, double target, uint32_t *__restrict__ fwd_len, uint32_t *__restrict__ rev_len,
                      int32_t *__restrict__ status) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= 2 * n) return;
    const uint64_t g = t >> 1;
    const bool rev = t & 1;
    const uint64_t beg = off[g], len = off[g + 1] - beg;
    const uint8_t *s = bases + beg;
    uint32_t *out = rev ? rev_len : fwd_len;
    bool ascii = true;
    for (uint64_t j = 0; j < len; ++j) ascii &= __ldg(s + j) < 0x80;
    if (!ascii) {
        out[g] = 0;
        atomicMax(&status[g], PG_ITEM_UNSUPPORTED);
        return;
    }
    for (uint64_t m = 15;; ++m) {
        if (m > len) {  // sequence[0:15+k] / sequence[len-(15+k):] out of range
            out[g] = 0;
            atomicMax(&status[g], PG_ITEM_PANIC);
            return;
        }
        double tm;
        if (!rev)
            tm = santalucia_core([s](uint64_t j) { return upper(__ldg(s + j)); }, m, lg, nullptr, nullptr);
        else  // ReverseComplement(sequence[len-m:]): byte j is the complement of sequence[len-1-j]
            tm = santalucia_core([s, len](uint64_t j) { return complement_upper(upper(__ldg(s + len - 1 - j))); }, m, lg,
                                 nullptr, nullptr);
        if (!(tm < target)) {  // loop runs while MeltingTemp(primer) < targetTm
            out[g] = (uint32_t)m;
            return;
        }
    }
}

// pcr.SimulateSimple's minimal-primer loop, /root/reference/primers/pcr/pcr.go:93-100 (SURVEY 8f.3):
//     for index := minimalPrimerLength (= 7, pcr.go:35); MeltingTemp(primer[len-index:]) < targetTm; index++ {
//         minimalLength = index; if primer[len-index:] == primer { break } }
// i.e. the LONGEST 3' suffix (>= 7 nt) whose Tm is still below the target, 0 when the 7-mer
// already reaches it, len when even the whole primer stays below.  One thread per primer.
constexpr uint64_t PCR_MIN_PRIMER = 7;  // minimalPrimerLength, pcr.go:35 (15 is only designedMinimalPrimerLength, pcr.go:38)
__global__ void __launch_bounds__(256)
minimal_primer_kernel(const uint8_t *__restrict__ bases, const uint64_t *__restrict__ off, uint64_t n, TmLogs lg, double target,
                      uint32_t *__restrict__ min_len, int32_t *__restrict__ status) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t beg = off[i], len = off[i + 1] - beg;
    const uint8_t *s = bases + beg;
    min_len[i] = 0;
    bool ascii = true;
    for (uint64_t j = 0; j < len; ++j) ascii &= __ldg(s + j) < 0x80;
    if (!ascii) { status[i] = PG_ITEM_UNSUPPORTED; return; }
    if (len < PCR_MIN_PRIMER) { status[i] = PG_ITEM_PANIC; return; }  // primer[len(primer)-7:] out of range
    uint32_t minimal = 0;
    for (uint64_t index = PCR_MIN_PRIMER;; ++index) {
        const uint8_t *suffix = s + (len - index);
        const double tm = santalucia_core([suffix](uint64_t j) { return upper(__ldg(suffix + j)); }, index, lg, nullptr, nullptr);
        if (!(tm < target)) break;
        minimal = (uint32_t)index;
        if (index == len) break;
    }
    min_len[i] = minimal;
    status[i] = PG_ITEM_OK;
}

}  // namespace

int launch_minimal_primer(const uint8_t *d_bases, const uint64_t *d_off, uint64_t n, double target,
                          uint32_t *d_min_len, int32_t *d_status, cudaStream_t st) {
    if (n == 0) return PG_OK;
    minimal_primer_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_bases, d_off, n, melting_temp_logs(), target, d_min_len,
                                                                       d_status);
    PG_LAUNCH_CHECK("minimal_primer_kernel");
    return PG_OK;
}

int launch_tm(const uint8_t *d_bases, const uint64_t *d_off, uint64_t n, double cp, double na,
              double mg, double *d_tm, double *d_dh, double *d_ds, int32_t *d_status,
              cudaStream_t st) {
    if (n == 0) return PG_OK;
    tm_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_bases, d_off, n, tm_logs(cp, na, mg), d_tm, d_dh, d_ds,
                                                          d_status);
    PG_LAUNCH_CHECK("tm_kernel");
    return PG_OK;
}

int launch_design_primers(const uint8_t *d_bases, const uint64_t *d_off, uint64_t n, double target,
                          uint32_t *d_fwd, uint32_t *d_rev, int32_t *d_status, cudaStream_t st) {
    if (n == 0) return PG_OK;
    PG_CUDA(cudaMemsetAsync(d_status, 0, n * sizeof(int32_t), st));
    design_primers_kernel<<<(unsigned)((2 * n + 255) / 256), 256, 0, st>>>(d_bases, d_off, n, melting_temp_logs(), target, d_fwd,
                                                                            d_rev, d_status);
    PG_LAUNCH_CHECK("design_primers_kernel");
    return PG_OK;
}

}  // namespace pg
