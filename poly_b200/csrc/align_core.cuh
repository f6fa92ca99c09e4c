// align_core.cuh -- the rules every alignment kernel (sw_score.cu, sw_pairs.cu, sw_align.cu,
// sw_align_long.cu) must apply identically for its outputs to match the reference's
// search/align/align.go: the cell recurrence, the error order, the traceback step and the width of
// the score type; plus the host-side scoring parameters and the device parameter block they upload.
#pragma once
#include <algorithm>
#include <cstring>
#include <initializer_list>
#include <vector>

#include "common.cuh"

namespace pg {

// ---- device ----------------------------------------------------------------------------------

template <typename T>
__device__ __forceinline__ T addmax(T a, T b, T c) {  // max(a + b, c)
    const T x = a + b;
    return x > c ? x : c;
}
template <>
__device__ __forceinline__ int addmax<int>(int a, int b, int c) {
    return __viaddmax_s32(a, b, c);
}

// The score of a row beyond the string: -2^29 / -2^61, below every valid cell.  Near a limit of the
// type, rows beyond the string can wrap: a global alignment's diag + score near the negative limit, or
// a positive gap's running sums near the positive one.  That is harmless only because those rows are
// never read: a row depends on smaller rows alone, the NW result comes from the string's last row, and
// a positive gap masks them out of the SW maximum.
template <typename T>
struct NegBig {
    static constexpr T value = (T)0 - ((T)1 << (sizeof(T) * 8 - 3));
};

// H[i][j] from diag = H[i-1][j-1], sc = S(a_i, b_j), left = H[i][j-1], up = H[i-1][j], in the operand
// order of align.go:132-135 (NW, no zero floor) and align.go:192-196 (SW).
template <typename T, bool GLOBAL>
__device__ __forceinline__ T sw_cell(T diag, T sc, T left, T up, T gap) {
    T v;
    if (GLOBAL) {
        v = addmax<T>(diag, sc, left + gap);
        v = addmax<T>(up, gap, v);
    } else {
        v = addmax<T>(diag, sc, (T)0);
        v = addmax<T>(left, gap, v);
        v = addmax<T>(up, gap, v);
    }
    return v;
}

// The error the reference reports for a pair whose strings are both non-empty, given the first
// index of a bad symbol in a and in b (-1: none): the first failing cell in row-major order, stringA
// outer (align.go:186-191), with Encode(a) tried before Encode(b) (matrix.go:29-36).  Leaves ec, ep
// unchanged when there is no error.  The chain runs on copies and both outputs are stored once, so
// the inlined code stays branch-free (conditional stores through the references would not be).
__host__ __device__ __forceinline__ void first_error(int64_t bad_a, int64_t bad_b, int32_t &ec, int64_t &ep) {
    int32_t c = ec;
    int64_t p = ep;
    if (bad_a == 0) { c = 1; p = 0; }
    else if (bad_b >= 0) { c = 2; p = bad_b; }
    else if (bad_a > 0) { c = 1; p = bad_a; }
    ec = c;
    ep = p;
}

// ---- traceback (align.go:141-160 NW, :209-229 SW) ---------------------------------------------
// "up" is the previous index of stringA ('-' in B), "left" the previous index of stringB.
enum TraceStep { STEP_DIAG, STEP_UP, STEP_LEFT, STEP_STOP };

template <bool GLOBAL>
__device__ __forceinline__ TraceStep trace_step(int h, int h_diag, int h_up, int h_left, int sc, int gap) {
    if (h == h_diag + sc) return STEP_DIAG;             // align.go:146-150 / 215-219
    if (h == h_up + gap) return STEP_UP;                // align.go:151-154 / 220-223
    if (GLOBAL || h == h_left + gap) return STEP_LEFT;  // NW: the plain else of align.go:155-159; SW: 224-228
    return STEP_STOP;                                   // unreachable for a max of the three
}

// The reference builds the strings by prepending: append here, count past the caller's stride.  As in
// first_error, the outputs are stored once from locals.
__device__ __forceinline__ void trace_put(uint8_t *oa, uint8_t *ob, uint64_t stride, uint8_t ca, uint8_t cb, uint32_t &len,
                                          bool &overflow) {
    const uint32_t n = len;
    bool o = overflow;
    if (n < stride) { oa[n] = ca; ob[n] = cb; }
    else o = true;
    len = n + 1;
    overflow = o;
}

// Reverses the stored part of both strings in place and writes the item's length and status.
__device__ __forceinline__ void trace_finish(uint8_t *oa, uint8_t *ob, uint64_t stride, uint32_t len, bool overflow,
                                             uint32_t *out_len, int32_t *status, uint64_t item) {
    const uint32_t n_written = min(len, (uint32_t)stride);
    for (uint32_t x = 0; x < n_written / 2; ++x) {
        uint8_t t1 = oa[x]; oa[x] = oa[n_written - 1 - x]; oa[n_written - 1 - x] = t1;
        t1 = ob[x]; ob[x] = ob[n_written - 1 - x]; ob[n_written - 1 - x] = t1;
    }
    out_len[item] = len;
    status[item] = overflow ? PG_ITEM_UNSUPPORTED : PG_ITEM_OK;
}

// ---- host ------------------------------------------------------------------------------------

// The scoring of one call, as the C ABI passes it: byte -> symbol LUTs of a and b (256 entries, < 0:
// not in the alphabet), the n_a x n_b substitution table with a's symbol on the rows, the gap
// penalty, and local (Smith-Waterman) or global (Needleman-Wunsch) alignment.
struct AlignScoring {
    const int16_t *lut_a, *lut_b;
    const int64_t *table;
    int n_a, n_b;
    int64_t gap;
    int global;

    bool has_null() const { return !lut_a || !lut_b || !table; }
    int check() const {
        if (n_a <= 0 || n_b <= 0 || n_a > 255 || n_b > 255) {
            set_error("alphabet sizes must be in 1..255 (got %d, %d)", n_a, n_b);
            return PG_ERR_ARG;
        }
        return PG_OK;
    }
    int64_t abs_max() const {
        int64_t m = 0;
        for (int i = 0; i < n_a * n_b; ++i) m = std::max<int64_t>(m, table[i] < 0 ? -table[i] : table[i]);
        return m;
    }
};

// Scores take 32-bit arithmetic when score_bound(...) < SCORE32_LIMIT, 64-bit otherwise.
constexpr long double SCORE32_LIMIT = 2.0e9L;

// A bound on every DP value and on the operands of one add, for strings of which the shorter has at
// most short_len symbols and the two together at most sum_len.  NW: a value is the sum of at most sum
// steps of |S| or |gap|, so every value lies within (sum + 2) * max(|S|, |gap|).  SW with gap <= 0: values
// lie in [0, max|S| * short], and one add puts max(|S|, |gap|) on top.  SW with gap > 0: H[i][j] >=
// H[i][j-1] + gap, so values grow with the longer string too and take the NW bound.
inline long double score_bound(int global, int64_t amax, int64_t gap, uint64_t short_len, uint64_t sum_len) {
    const int64_t agap = gap < 0 ? -gap : gap;
    return global || gap > 0 ? (long double)std::max(amax, agap) * (long double)(sum_len + 2)
                             : (long double)amax * (long double)short_len + (long double)std::max(amax, agap);
}

// The packed 2 x int16 score kernel (sw_score.cu) takes a call when it is local with gap <= 0 and every
// DP value stays below 2^14: below 16000 by the bound, and rows beyond a query (-16384 + a value >= 0, or
// a value >= 0 + gap) stay above -2^15.  It holds two queries per thread, so a call needs two of them.
inline bool score_packed16(int global, int64_t gap, long double bound, uint64_t nq) {
    return !global && gap <= 0 && bound < 16000.0L && -gap < 16000 && nq >= 2;
}

// Device copy of the scoring: [lut_row: 256 int16][lut_col: 256 int16][tables in T].
template <typename T>
struct AlignTables {
    const int16_t *lut_row, *lut_col;
    const T *tab;  // the first table; the next one, if any, follows it
};

// Builds and uploads the parameter block.  One table per entry of `a_rows`, in that order: a's
// symbols on its rows when the entry is true, else b's; lut_row is the LUT of the first table's row
// side.  With neg_row each table has one last row of NegBig<T> for the rows beyond a string.  The
// block is copied from pageable memory, which cudaMemcpyAsync stages before it returns, so the host
// vector may go out of scope at once; the copy stays stream-ordered and the host does not wait.
template <typename T>
int upload_tables(const AlignScoring &s, std::initializer_list<bool> a_rows, bool neg_row, StreamScratch &tmp, cudaStream_t st,
                  AlignTables<T> *out) {
    size_t ntab = 0;
    for (bool ar : a_rows) ntab += (size_t)((ar ? s.n_a : s.n_b) + (neg_row ? 1 : 0)) * (ar ? s.n_b : s.n_a);
    std::vector<uint8_t> blob(1024 + ntab * sizeof(T));
    const bool first_a = *a_rows.begin();
    memcpy(blob.data(), first_a ? s.lut_a : s.lut_b, 512);
    memcpy(blob.data() + 512, first_a ? s.lut_b : s.lut_a, 512);
    T *h = reinterpret_cast<T *>(blob.data() + 1024);
    for (bool ar : a_rows) {
        const int rows = ar ? s.n_a : s.n_b, cols = ar ? s.n_b : s.n_a;
        for (int r = 0; r < rows; ++r)
            for (int c = 0; c < cols; ++c) *h++ = (T)(ar ? s.table[(size_t)r * s.n_b + c] : s.table[(size_t)c * s.n_b + r]);
        if (neg_row)
            for (int c = 0; c < cols; ++c) *h++ = NegBig<T>::value;
    }
    uint8_t *d = nullptr;
    PG_CUDA(tmp.alloc(&d, blob.size()));
    PG_CUDA(cudaMemcpyAsync(d, blob.data(), blob.size(), cudaMemcpyHostToDevice, st));
    out->lut_row = reinterpret_cast<const int16_t *>(d);
    out->lut_col = out->lut_row + 256;
    out->tab = reinterpret_cast<const T *>(d + 1024);
    return PG_OK;
}

// Launches kernel with `smem` bytes of dynamic shared memory (raising the kernel's limit through the
// per-device cache when needed) and records it as `name`.
template <typename... P, typename... A>
int launch_smem(void (*kernel)(P...), unsigned grid, unsigned block, size_t smem, cudaStream_t st, const char *name, A... args) {
    int rc = func_smem((const void *)kernel, smem);
    if (rc != PG_OK) return rc;
    kernel<<<grid, block, smem, st>>>(args...);
    PG_LAUNCH_CHECK(name);
    return PG_OK;
}

}  // namespace pg
