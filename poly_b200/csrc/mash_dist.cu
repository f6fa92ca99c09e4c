// mash_dist.cu -- Mash distance between grouped sketches (`mash dist`, `mash triangle`): for every query row A and
// reference row B, Mash's compareSketches counts (denom = min(s, |A u B|), common = the shared values among the denom
// smallest values of A u B), the distance -ln(2J / (1 + J)) / k and the binomial p-value (include/poly_b200.h).
//
// Layout: one warp merges one pair at a time.  A CTA of DIST_WARPS warps takes a work item (a tile of up to 32
// reference rows, a chunk of DIST_QCHUNK queries); the tile is staged in shared memory once, and each warp stages
// its current query row in a slot of its own, then merges it against every row of the tile.  Lane t keeps the
// counts of the tile's row t, so after the tile the 32 lanes finish 32 pairs at once (distance, p-value, stores).
// The tile takes up to 32 rows, as many as fit beside the warps' slots in 227 KiB; from s = 3419 not even one row
// does, and that path (SMEM = false) reads both rows from global memory, with the same merge.
//
// Merge of one pair: the merged sequence of A and B (an equal pair A-first) holds each union value once or, when
// shared, twice in a row, so its first min(a + b, 2 s) items already hold min(s, |A u B|) union values.  Lane l
// takes items [l P / 32, (l + 1) P / 32) of those P items, finds where they start by a co-rank binary search, and
// walks them, one shared-memory load per item: u = union values, sh = shared values (a B item equal to the A item
// just before it).  A warp scan of u gives each lane the union rank its items start at; a shared value counts iff
// its union rank is < s, which holds for every shared value of a lane that ends at or below s, none of a lane that
// starts above it, and is decided item by item by a second walk in the one lane that crosses s.
#include <algorithm>
#include <cmath>

#include "common.cuh"

namespace pg {
namespace {

constexpr int DIST_WARPS = 16;
constexpr int DIST_THREADS = DIST_WARPS * 32;
constexpr int DIST_TILE = 32;                         // reference rows per tile: one per lane
constexpr uint64_t DIST_QCHUNK = 4 * DIST_WARPS;      // queries per work item
constexpr size_t DIST_SMEM_BYTES = 227 * 1024;        // the H100's shared memory per CTA (opt-in)

// rows of the tile and the warps' query slots that fit, s words each
inline int dist_tile_rows(int s) {
    const int64_t rows = (int64_t)(DIST_SMEM_BYTES / (4 * (uint64_t)s)) - DIST_WARPS;
    return (int)std::min<int64_t>(DIST_TILE, rows);
}

// the number of A items among the first d items of the merge of A and B (A first on ties)
__device__ __forceinline__ uint32_t co_rank(const uint32_t *A, uint32_t a, const uint32_t *B, uint32_t b, uint32_t d) {
    uint32_t lo = d > b ? d - b : 0, hi = min(d, a);
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (A[mid] <= B[d - mid - 1]) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

// Walks n items of the merge from A[i], B[j]: u = union values, sh = shared values whose union count up to and
// including their A twin (counted from this walk's start) is <= lim.
__device__ __forceinline__ void merge_walk(const uint32_t *A, uint32_t a, const uint32_t *B, uint32_t b, uint32_t i, uint32_t j, uint32_t n,
                                           uint32_t lim, uint32_t &u, uint32_t &sh) {
    u = 0;
    sh = 0;
    uint32_t prev = i > 0 ? A[i - 1] : 0;  // the last A item taken
    bool has_prev = i > 0;
    uint32_t av = i < a ? A[i] : 0, bv = j < b ? B[j] : 0;
    for (uint32_t t = 0; t < n; ++t) {
        const bool take_a = j >= b || (i < a && av <= bv);
        const bool dup = !take_a && has_prev && prev == bv;
        u += dup ? 0u : 1u;
        sh += (dup && u <= lim) ? 1u : 0u;
        if (take_a) { prev = av; has_prev = true; ++i; } else { ++j; }
        const uint32_t idx = take_a ? i : j;
        const uint32_t *src = take_a ? A : B;
        const uint32_t nv = idx < (take_a ? a : b) ? src[idx] : 0u;
        av = take_a ? nv : av;
        bv = take_a ? bv : nv;
    }
}

// (common, denom) of rows A (a values) and B (b values), the same in every lane of the warp
__device__ __forceinline__ void merge_pair(const uint32_t *A, uint32_t a, const uint32_t *B, uint32_t b, uint32_t s, uint32_t lane,
                                           uint32_t &common, uint32_t &denom) {
    const uint64_t P = min((uint64_t)a + b, (uint64_t)2 * s);
    const uint32_t d0 = (uint32_t)(P * lane / 32), d1 = (uint32_t)(P * (lane + 1) / 32);
    const uint32_t i = co_rank(A, a, B, b, d0), j = d0 - i;
    uint32_t u, sh;
    merge_walk(A, a, B, b, i, j, d1 - d0, 0xffffffffu, u, sh);
    uint32_t incl = u;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
        if ((int)lane >= o) incl += v;
    }
    const uint32_t base = incl - u;  // union values before this lane's items
    uint32_t cnt = sh;
    if (base > s) cnt = 0;
    else if (base + u > s) merge_walk(A, a, B, b, i, j, d1 - d0, s - base, u, cnt);  // u is recounted unchanged
    const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
    common = __reduce_add_sync(0xffffffffu, cnt);
    denom = min(total, s);
}

// Continued fraction of the incomplete beta function (modified Lentz)
__device__ double beta_cf(double a, double b, double x) {
    const double tiny = 1e-300, eps = 1e-15;
    const double qab = a + b, qap = a + 1.0, qam = a - 1.0;
    double c = 1.0, d = 1.0 - qab * x / qap;
    if (fabs(d) < tiny) d = tiny;
    d = 1.0 / d;
    double h = d;
    for (int m = 1; m <= (1 << 22); ++m) {
        const double m2 = 2.0 * m;
        double aa = m * (b - m) * x / ((qam + m2) * (a + m2));
        d = 1.0 + aa * d;
        if (fabs(d) < tiny) d = tiny;
        c = 1.0 + aa / c;
        if (fabs(c) < tiny) c = tiny;
        d = 1.0 / d;
        h *= d * c;
        aa = -(a + m) * (qab + m) * x / ((a + m2) * (qap + m2));
        d = 1.0 + aa * d;
        if (fabs(d) < tiny) d = tiny;
        c = 1.0 + aa / c;
        if (fabs(c) < tiny) c = tiny;
        d = 1.0 / d;
        const double del = d * c;
        h *= del;
        if (fabs(del - 1.0) < eps) break;
    }
    return h;
}

__device__ double mash_distance(uint32_t common, uint32_t denom, int k) {
    if (common == denom) return 0.0;
    if (common == 0) return 1.0;
    const double j = (double)common / denom;
    const double d = -log(2.0 * j / (1.0 + j)) / k;
    return d > 1.0 ? 1.0 : d;
}

// Stirling's remainder ln n! - (n + 1/2) ln n + n - ln sqrt(2 pi) of n = 1 .. 15, each the double nearest
//   mpmath (dps 40): loggamma(n + 1) - (n + mpf(1) / 2) * log(n) + n - log(2 * pi) / 2
__constant__ double STIRLERR_SMALL[15] = {
    0.08106146679532726,  0.0413406959554093,    0.02767792568499834,  0.020790672103765093, 0.016644691189821193,
    0.013876128823070748, 0.01189670994589177,   0.010411265261972096, 0.009255462182712733, 0.00833056343336287,
    0.007573675487951841, 0.00694284010720953,   0.006408994188004207, 0.0059513701127588475, 0.005554733551962801};

// Stirling's remainder of an integer n >= 1: the table, then the series 1/12n - 1/360n^3 + 1/1260n^5 - ... cut where
// its next term is below 1e-16
__device__ double stirlerr(double n) {
    if (n <= 15.0) return STIRLERR_SMALL[(int)n - 1];
    const double S0 = 1.0 / 12, S1 = 1.0 / 360, S2 = 1.0 / 1260, S3 = 1.0 / 1680, S4 = 1.0 / 1188;
    const double nn = n * n;
    if (n > 500.0) return (S0 - S1 / nn) / n;
    if (n > 80.0) return (S0 - (S1 - S2 / nn) / nn) / n;
    if (n > 35.0) return (S0 - (S1 - (S2 - S3 / nn) / nn) / nn) / n;
    return (S0 - (S1 - (S2 - (S3 - S4 / nn) / nn) / nn) / nn) / n;
}

// The deviance x ln(x / m) + m - x (x, m > 0), by its series in v = (x - m) / (x + m) when x is near m, where the
// closed form cancels
__device__ double bd0(double x, double m) {
    if (fabs(x - m) < 0.1 * (x + m)) {
        double v = (x - m) / (x + m), s = (x - m) * v, ej = 2.0 * x * v;
        v *= v;
        for (int j = 1; j < 1000; ++j) {
            ej *= v;
            const double s1 = s + ej / (2 * j + 1);
            if (s1 == s) return s1;
            s = s1;
        }
        return s;
    }
    return x * log(x / m) + m - x;
}

// P[Binomial(n, r) = x] for integers 0 <= x <= n, 0 < r < 1, in Loader's saddle-point form: the Stirling remainders
// and the two deviances are each small where the density is not, so no large terms cancel
__device__ double dbinom(uint32_t x, uint32_t n, double r) {
    const double dn = n, dx = x;
    if (x == 0) return exp(dn * log1p(-r));
    if (x == n) return exp(dn * log(r));
    const double lc = stirlerr(dn) - stirlerr(dx) - stirlerr(dn - dx) - bd0(dx, dn * r) - bd0(dn - dx, fma(-dn, r, dn));
    const double lf = 1.8378770664093453 + log(dx) + log1p(-dx / dn);  // ln(2 pi x (n - x) / n); the constant is ln 2 pi
    return exp(lc - 0.5 * lf);
}

// P[Binomial(denom, r) >= common] = I_r(common, denom - common + 1), Mash's pValue.  With a = common and
// b = denom - common + 1 the incomplete beta's prefactor x^a (1 - x)^b / (a B(a, b)) is (1 - r) dbinom(common), and
// with a and b swapped r dbinom(common - 1), which keeps full precision at any denom where log-gamma differences
// would not.
__device__ double mash_p_value(uint32_t common, uint32_t denom, int k, uint64_t len_q, uint64_t len_r) {
    if (common == 0) return 1.0;
    const double four_k = ldexp(1.0, 2 * k);
    const double pq = 1.0 / (1.0 + four_k / (double)len_q), pr = 1.0 / (1.0 + four_k / (double)len_r);
    const double den = pq + pr - pq * pr;
    const double r = den > 0.0 ? pq * pr / den : 0.0;
    if (!(r > 0.0)) return 0.0;
    if (r >= 1.0) return 1.0;
    const double a = common, b = (double)denom - common + 1.0;
    if (r < (a + 1.0) / (a + b + 2.0)) return dbinom(common, denom, r) * beta_cf(a, b, r) * (1.0 - r);
    return 1.0 - r * dbinom(common - 1, denom, r) * beta_cf(b, a, 1.0 - r);
}

// Lane `lane` < nt of the warp finishes pair (q, r0 + lane) of the block with counts (c, d)
template <bool LIST>
__device__ __forceinline__ void finish_pair(const DistArgs &g, uint64_t q, uint64_t r, uint32_t c, uint32_t d, bool need_p) {
    const double dist = mash_distance(c, d, g.k);
    const double p = need_p ? mash_p_value(c, d, g.k, g.q_len[q], g.r_len[r]) : 1.0;
    if (LIST) {
        const uint64_t gq = g.q0 + q;
        if (g.upper && r <= gq) return;
        if (!(dist <= g.max_distance && p <= g.max_p_value)) return;
        const unsigned long long slot = atomicAdd(g.n_pairs, 1ull);
        if (slot >= g.cap) return;
        g.pair_q[slot] = (uint32_t)gq;
        g.pair_r[slot] = (uint32_t)r;
        if (g.common) g.common[slot] = c;
        if (g.denom) g.denom[slot] = d;
        if (g.distance) g.distance[slot] = dist;
        if (g.p_value) g.p_value[slot] = p;
    } else {
        const uint64_t o = q * g.nr + r;
        if (g.common) g.common[o] = c;
        if (g.denom) g.denom[o] = d;
        if (g.distance) g.distance[o] = dist;
        if (g.p_value) g.p_value[o] = p;
    }
}

// copies the first n words of src to dst with the lanes (or threads) [t, n) step `step`
__device__ __forceinline__ void stage_row(uint32_t *dst, const uint32_t *__restrict__ src, uint32_t n, uint32_t t, uint32_t step) {
    for (uint32_t w = t; w < n; w += step) dst[w] = src[w];
}

template <bool SMEM, bool LIST>
__global__ void __launch_bounds__(DIST_THREADS, 1) mash_dist_kernel(const DistArgs g, int tile) {
    extern __shared__ uint32_t sm[];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5, s = (uint32_t)g.s;
    const uint64_t tiles = (g.nr + tile - 1) / tile, chunks = (g.nq + DIST_QCHUNK - 1) / DIST_QCHUNK;
    const bool need_p = g.p_value != nullptr || (LIST && g.max_p_value < 1.0);
    uint32_t *slot = sm + ((size_t)tile + warp) * s;
    for (uint64_t item = blockIdx.x; item < tiles * chunks; item += gridDim.x) {
        const uint64_t r0 = (item % tiles) * tile, qb = (item / tiles) * DIST_QCHUNK;
        const uint32_t nt = (uint32_t)min((uint64_t)tile, g.nr - r0);
        if (SMEM) {
            __syncthreads();  // the previous item's merges are done with the tile
            for (uint32_t t = warp; t < nt; t += DIST_WARPS) stage_row(sm + (size_t)t * s, g.r_rows + (r0 + t) * g.stride, g.r_count[r0 + t], lane, 32);
            __syncthreads();
        }
        const uint64_t qe = min(g.nq, qb + DIST_QCHUNK);
        for (uint64_t q = qb + warp; q < qe; q += DIST_WARPS) {
            const uint32_t a = g.q_count[q];
            const uint32_t *A = g.q_rows + q * g.stride;
            if (SMEM) {
                __syncwarp();  // the warp's previous query is done with its slot
                stage_row(slot, A, a, lane, 32);
                __syncwarp();
                A = slot;
            }
            uint32_t my_c = 0, my_d = 0;
            for (uint32_t t = 0; t < nt; ++t) {
                const uint32_t *B = SMEM ? sm + (size_t)t * s : g.r_rows + (r0 + t) * g.stride;
                uint32_t c, d;
                merge_pair(A, a, B, g.r_count[r0 + t], s, lane, c, d);
                if (lane == t) { my_c = c; my_d = d; }
            }
            if (lane < nt) finish_pair<LIST>(g, q, r0 + lane, my_c, my_d, need_p);
        }
    }
}

template <bool SMEM, bool LIST>
int launch_dist(const DistArgs &g, int tile, size_t smem, cudaStream_t st) {
    const void *fn = (const void *)mash_dist_kernel<SMEM, LIST>;
    const uint64_t items = ((g.nr + tile - 1) / tile) * ((g.nq + DIST_QCHUNK - 1) / DIST_QCHUNK);
    uint64_t blocks = 0;
    if (int rc = resident_blocks(fn, DIST_THREADS, smem, items, &blocks)) return rc;
    mash_dist_kernel<SMEM, LIST><<<(unsigned)blocks, DIST_THREADS, smem, st>>>(g, tile);
    PG_LAUNCH_CHECK("mash_dist_kernel");
    return PG_OK;
}

}  // namespace

int launch_mash_dist(const DistArgs &g, bool list, cudaStream_t st) {
    if (g.nq == 0 || g.nr == 0) return PG_OK;
    const int tile = dist_tile_rows(g.s);
    if (tile >= 1) {
        const size_t smem = ((size_t)tile + DIST_WARPS) * (size_t)g.s * 4;
        return list ? launch_dist<true, true>(g, tile, smem, st) : launch_dist<true, false>(g, tile, smem, st);
    }
    return list ? launch_dist<false, true>(g, DIST_TILE, 0, st) : launch_dist<false, false>(g, DIST_TILE, 0, st);
}

}  // namespace pg
