// fold.cu -- Zuker minimum free energy and dot-bracket of DNA / RNA (poly's fold package), one CTA per sequence.
//
// The reference fills its V (ends paired) and W (any structure) caches top-down; every cell with j - i >= 4
// is reached, so the fill here goes bottom-up by diagonal, V before W on each, all cells of a diagonal in
// parallel.  A cell keeps its energy and a descriptor (what its inner list is, DESIGN.md "Fold"):
//   NONE        no inner (hairpin, isolated pair, invalid)
//   ONE (r, l)  a stack, bulge or interior loop closing (r, l)
//   MULTI       a multibranch (start, mid, end, helix): inner = L(W[left]) ++ L(W[right])
// where L(W[x]) is what addBranch contributes for W[x].  Each W cell's L list is stored once in an arena
// (at most (j - i + 1) / 5 disjoint branches of >= 5 nt), so lists are read, never rebuilt.
// Float64 throughout, compiled with -fmad=false: every sum is the reference's, in its order.
#include <math.h>

#include <vector>

#include "common.cuh"

namespace pg {

namespace {

struct KeyEnergy {
    const char *key;
    double h, s;
};
struct LenEnergy {
    int len;
    double h, s;
};
#include "fold_tables.inc"

constexpr int kMaxTri = 160;
enum { T_NN, T_IM, T_TM, T_DE };
enum { L_IL, L_BL, L_HL };

// one nucleic-acid kind at the call's temperature: deltaG of every entry (0 where the key is absent, as Go's
// zero value gives), presence bits, and the loop terms for every length (table or Jacobson-Stockmayer)
struct FoldTables {
    double dg[4][625];
    uint8_t has[4][625];
    double loop[3][PG_FOLD_MAX_LEN + 1];
    double mb[4];
    uint32_t tri_key[kMaxTri];
    double tri_dg[kMaxTri];
    int n_tri;
    int rna;
};

constexpr uint64_t KIND_MASK = 3, K_NONE = 0, K_ONE = 1, K_MULTI_W = 2, K_MULTI_V = 3;
constexpr uint64_t HAIRPIN_BIT = 4;  // the description holds "HAIRPIN"
__host__ __device__ inline uint64_t desc(uint64_t kind, int a, int b, int c) {
    return kind | ((uint64_t)a << 8) | ((uint64_t)b << 20) | ((uint64_t)c << 32);
}
__device__ inline int dA(uint64_t d) { return (int)((d >> 8) & 0x7ff); }
__device__ inline int dB(uint64_t d) { return (int)((d >> 20) & 0x7ff); }
__device__ inline int dC(uint64_t d) { return (int)((d >> 32) & 0x7ff); }

__host__ __device__ inline uint64_t cap_of(int d) { return (uint64_t)(d + 1) / 5; }
// arena entries of an n-nt item
__host__ __device__ inline uint64_t arena_entries(int n) {
    uint64_t a = 0;
    for (int d = 0; d < n; ++d) a += (uint64_t)(n - d) * cap_of(d);
    return a;
}
__host__ __device__ inline uint64_t align8(uint64_t x) { return (x + 7) & ~7ull; }

struct Item {
    int n;
    const FoldTables *t;
    uint8_t *code;  // A C G T|U = 0..3
    double *Ve, *We;
    uint64_t *Vd, *Wd;
    uint16_t *Lc;
    uint32_t *arena;
    const uint64_t *doff;  // arena offset of each diagonal (shared memory)
    int *err;
    __device__ uint32_t *L(int i, int j) const { return arena + doff[j - i] + (uint64_t)i * cap_of(j - i); }
    __device__ size_t at(int i, int j) const { return (size_t)i * n + j; }
    __device__ bool comp(int i, int j) const { return code[i] == 3 - code[j]; }
    __device__ int c(int i) const { return i >= 0 && i < n ? code[i] : 4; }
    __device__ int key(int a, int b, int cc, int d) const { return c(a) * 125 + c(b) * 25 + c(cc) * 5 + c(d); }
};

__device__ inline double go_min(double a, double b) {
    if (a == 0 && b == 0) return signbit(a) ? a : b;
    return a < b ? a : b;
}

// fold.go:600-673
__device__ double stack(const Item &it, int start, int ros, int end, int loe) {
    const int n = it.n;
    if (start >= n || ros >= n || end >= n || loe >= n) return 0;
    const int k = it.key(start, ros, end, loe);
    const FoldTables &t = *it.t;
    if (start == -1 || ros == -1 || end == -1 || loe == -1) return t.dg[T_DE][k];
    const double nn = t.has[T_NN][k] ? t.dg[T_NN][k] : t.dg[T_IM][k];
    if ((start > 0 && end < n - 1) || (start == 0 && end == n - 1)) return nn;
    if (start > 0 && end == n - 1) {
        double dG = nn;
        const int kd = it.c(start - 1) * 125 + it.c(start) * 25 + 4 * 5 + it.c(end);
        if (t.has[T_DE][kd]) dG += t.dg[T_DE][kd];
        return dG;
    }
    if (start == 0 && end < n - 1) {
        const int kd = 4 * 125 + it.c(start) * 25 + it.c(end + 1) * 5 + it.c(end);
        if (t.has[T_DE][kd]) {
            double dG = nn;
            dG += t.dg[T_DE][kd];
            return dG;
        }
    }
    return 0;
}

// fold.go:683-731 for a pair that closes (the caller checked the complement)
__device__ double hairpin(const Item &it, int start, int end) {
    const FoldTables &t = *it.t;
    const int len = end - start + 1, hl = len - 2;
    double dG = 0.0;
    if (!t.rna && len <= 6) {
        uint32_t key = (uint32_t)len << 12;
        for (int i = 0; i < len; ++i) key |= (uint32_t)it.code[start + i] << (2 * i);
        for (int i = 0; i < t.n_tri; ++i)
            if (t.tri_key[i] == key) { dG = t.tri_dg[i]; break; }
    }
    dG += t.loop[L_HL][hl];
    const int k = it.key(start, start + 1, end, end - 1);
    if (hl > 3 && t.has[T_TM][k]) dG += t.dg[T_TM][k];
    if (hl == 3 && (it.code[start] == 0 || it.code[end] == 0)) dG += 0.5;
    return dG;
}

// fold.go:285-322
__device__ double bulge(const Item &it, int start, int ros, int end, int loe) {
    const int len = max(ros - start - 1, end - loe - 1);
    double dG = it.t->loop[L_BL][len];
    if (len == 1) {
        if (!it.t->has[T_NN][it.key(start, ros, end, loe)]) atomicOr(it.err, 1);
        dG += stack(it, start, ros, end, loe);
    }
    if (it.code[start] == 0) dG += 0.5;
    if (it.code[ros] == 0) dG += 0.5;
    if (it.code[end] == 0) dG += 0.5;
    if (it.code[loe] == 0) dG += 0.5;
    return dG;
}

// fold.go:534-581 (both sides >= 1 here)
__device__ double internal_loop(const Item &it, int start, int ros, int end, int loe) {
    const int l = ros - start - 1, r = end - loe - 1;
    if (l == 1 && r == 1) {
        const double a = stack(it, start, ros, end, loe);
        const double b = stack(it, ros - 1, ros, loe + 1, loe);
        return a + b;
    }
    double dG = it.t->loop[L_IL][l + r];
    dG += 0.3 * fabs((double)(l - r));
    dG += it.t->dg[T_TM][it.key(start, start + 1, end, end - 1)];
    dG += it.t->dg[T_TM][it.key(ros - 1, ros, loe + 1, loe)];
    return dG;
}

// W energy as the fill reads it: cells with j - i < 4 are invalid (+inf)
__device__ inline double w_energy(const Item &it, int i, int j) { return j - i < 4 ? INFINITY : it.We[it.at(i, j)]; }
__device__ inline uint32_t l_count(const Item &it, int i, int j) { return j - i < 4 ? 0 : it.Lc[it.at(i, j)]; }

// the branches of multibranch(start, mid, end, helix): L(W[l0,l1]) ++ L(W[r0,r1]) (++ (start, end))
struct Branches {
    const uint32_t *lp, *rp;
    int nl, nr, count;
    uint32_t self;
    __device__ uint32_t operator[](int k) const { return k < nl ? lp[k] : k < nl + nr ? rp[k - nl] : self; }
};
__device__ inline int bs(uint32_t b) { return (int)(b >> 16); }
__device__ inline int be(uint32_t b) { return (int)(b & 0xffff); }
__device__ inline uint32_t bpack(int s, int e) { return ((uint32_t)s << 16) | (uint32_t)e; }

__device__ inline Branches branches_of(const Item &it, int start, int mid, int end, bool helix) {
    const int l0 = helix ? start + 1 : start, r1 = helix ? end - 1 : end;
    Branches b;
    b.nl = l_count(it, l0, mid);
    b.nr = l_count(it, mid + 1, r1);
    b.lp = b.nl ? it.L(l0, mid) : nullptr;
    b.rp = b.nr ? it.L(mid + 1, r1) : nullptr;
    b.self = bpack(start, end);
    b.count = b.nl + b.nr + (helix ? 1 : 0);
    return b;
}

// fold.go:359-514: the energy of multibranch(start, mid, end, helix), +inf when it is invalid
__device__ double multibranch(const Item &it, int start, int mid, int end, bool helix) {
    const int l0 = helix ? start + 1 : start, r1 = helix ? end - 1 : end;
    const double le = w_energy(it, l0, mid), re = w_energy(it, mid + 1, r1);
    if (!(isfinite(le) && isfinite(re))) return INFINITY;
    const Branches br = branches_of(it, start, mid, end, helix);
    if (br.nl + br.nr < 2) return INFINITY;
    const int cnt = br.count;
    int unpaired = 0;
    double summed = 0.0;
    for (int index = 0; index < cnt; ++index) {
        const uint32_t cur = br[index], lb = br[abs((index - 1) % cnt)], rb = br[(index + 1) % cnt];
        const int leftStart = bs(cur), leftEnd = be(cur), leftOfEnd = be(lb), rightStart = bs(rb), rightEnd = be(rb);
        int unpairedLeft = 0, unpairedRight = 0;
        double dangling = 0.0;
        if (index == cnt - 1 && !helix) {
        } else if (rb == br.self) {
            unpairedLeft = leftStart - leftOfEnd - 1;
            unpairedRight = rightEnd - leftEnd - 1;
            if (unpairedLeft != 0 && unpairedRight != 0) {
                dangling = stack(it, leftStart - 1, leftStart, leftEnd + 1, leftEnd);
            } else if (unpairedRight != 0) {
                dangling = stack(it, -1, leftStart, leftEnd + 1, leftEnd);
                if (unpairedRight == 1) dangling = go_min(stack(it, rightStart, -1, rightEnd, rightEnd - 1), dangling);
            }
        } else if (cur == br.self) {
            unpairedLeft = leftEnd - leftOfEnd - 1;
            unpairedRight = rightStart - leftStart - 1;
            if (unpairedLeft != 0 && unpairedRight != 0) {
                dangling = stack(it, leftStart - 1, leftStart, leftEnd + 1, leftEnd);
            } else if (unpairedRight != 0) {
                dangling = stack(it, leftStart, leftStart + 1, leftEnd, -1);
                if (unpairedRight == 1) dangling = go_min(stack(it, rightStart - 1, rightStart, -1, rightEnd), dangling);
            }
        } else {
            unpairedLeft = leftStart - leftOfEnd - 1;
            unpairedRight = rightStart - leftEnd - 1;
            if (unpairedLeft != 0 && unpairedRight != 0) {
                dangling = stack(it, leftStart - 1, leftStart, leftEnd + 1, leftEnd);
            } else if (unpairedRight != 0) {
                dangling = stack(it, -1, leftStart, leftEnd + 1, leftEnd);
                if (unpairedRight == 1) dangling = go_min(stack(it, leftStart - 1, leftStart, leftEnd + 1, leftEnd), dangling);
            }
        }
        summed += dangling;
        unpaired += unpairedRight;
        if (unpairedRight < 0) { atomicOr(it.err, 1); return INFINITY; }
        if (cur != br.self) summed += w_energy(it, leftStart, leftEnd);
    }
    const double *mb = it.t->mb;
    double e = mb[0] + mb[1] * (double)cnt + mb[2] * (double)unpaired;
    if (unpaired == 0) e = mb[0] + mb[3];
    return e + summed;
}

// fold.go:139-272 for one cell with end - start >= 4
__device__ void fill_v(const Item &it, int start, int end) {
    const int n = it.n;
    const size_t ix = it.at(start, end);
    if (!it.comp(start, end)) { it.Ve[ix] = INFINITY; it.Vd[ix] = K_NONE; return; }
    bool isolatedOuter = true;
    if (start > 0 && end < n - 1) isolatedOuter = !it.comp(start - 1, end + 1);
    const bool isolatedInner = !it.comp(start + 1, end - 1);
    if (isolatedOuter && isolatedInner) { it.Ve[ix] = 1600; it.Vd[ix] = K_NONE; return; }
    const double e1 = hairpin(it, start, end);
    if (end - start == 4) { it.Ve[ix] = e1; it.Vd[ix] = K_NONE | HAIRPIN_BIT; return; }
    const FoldTables &t = *it.t;
    const bool pairLeftInner = t.has[T_NN][it.key(start, start + 1, end, end - 1)];
    double e2 = INFINITY;
    int e2r = 0, e2l = 0;
    for (int r = start + 1; r < end - 4; ++r) {
        for (int l = r + 4; l < end; ++l) {
            if (!it.comp(r, l)) continue;
            const bool pairInner = pairLeftInner || t.has[T_NN][it.key(r - 1, r, l + 1, l)];
            const bool isStack = r == start + 1 && l == end - 1, bulgeLeft = r > start + 1, bulgeRight = l < end - 1;
            double e;
            if (isStack) e = stack(it, start, r, end, l);
            else if (bulgeLeft && bulgeRight && !pairInner) e = internal_loop(it, start, r, end, l);
            else if (bulgeLeft != bulgeRight) e = bulge(it, start, r, end, l);
            else continue;
            e += it.Ve[it.at(r, l)];
            if (e != -INFINITY && e < e2) { e2 = e; e2r = r; e2l = l; }
        }
    }
    double e3 = INFINITY;
    int e3k = 0;
    if (!isolatedOuter || start == 0 || end == n - 1) {
        for (int k = start + 1; k < end - 1; ++k) {
            const double e = multibranch(it, start, k, end, true);
            if (isfinite(e) && e < e3) { e3 = e; e3k = k; }
        }
    }
    // minimumStructure(e1, e2, e3)
    double m = INFINITY;
    uint64_t d = K_NONE;
    if (e1 != -INFINITY && e1 < m) { m = e1; d = K_NONE | HAIRPIN_BIT; }
    if (e2 != -INFINITY && e2 < m) { m = e2; d = desc(K_ONE, e2r, e2l, 0); }
    if (e3 != -INFINITY && e3 < m) { m = e3; d = desc(K_MULTI_V, start, end, e3k); }
    it.Ve[ix] = m;
    it.Vd[ix] = d;
}

// fold.go:84-122 for one cell with end - start >= 4, then its addBranch list (fold.go:324-343)
__device__ void fill_w(const Item &it, int start, int end) {
    const size_t ix = it.at(start, end);
    double m = INFINITY;
    uint64_t d = K_NONE;
    auto take = [&](double e, uint64_t dd) {
        if (e != -INFINITY && e < m) { m = e; d = dd; }
    };
    take(w_energy(it, start + 1, end), end - start - 1 < 4 ? K_NONE : it.Wd[it.at(start + 1, end)]);
    take(w_energy(it, start, end - 1), end - start - 1 < 4 ? K_NONE : it.Wd[it.at(start, end - 1)]);
    take(it.Ve[ix], it.Vd[ix]);
    double bif = INFINITY;
    int bk = 0;
    for (int k = start + 1; k < end - 1; ++k) {
        const double e = multibranch(it, start, k, end, false);
        if (isfinite(e) && e < bif) { bif = e; bk = k; }
    }
    take(bif, desc(K_MULTI_W, start, end, bk));
    it.We[ix] = m;
    it.Wd[ix] = d;
    // L(W[start, end])
    uint32_t *out = it.L(start, end);
    const uint64_t cap = cap_of(end - start);
    uint32_t cnt = 0;
    const uint64_t kind = d & KIND_MASK;
    if (isfinite(m) && kind == K_ONE) {
        out[cnt++] = bpack(dA(d), dB(d));
    } else if (isfinite(m) && kind != K_NONE) {
        const Branches br = branches_of(it, dA(d), dC(d), dB(d), kind == K_MULTI_V);
        for (int k = 0; k < br.nl + br.nr; ++k) {
            const uint32_t b = br[k];
            const int s = bs(b), e = be(b);
            const uint32_t c = l_count(it, s, e);
            if (!isfinite(w_energy(it, s, e))) continue;
            if (cnt + c > cap) { atomicOr(it.err, 1); break; }
            const uint32_t *src = it.L(s, e);
            for (uint32_t q = 0; q < c; ++q) out[cnt++] = src[q];
        }
    }
    it.Lc[ix] = (uint16_t)cnt;
}

// ---- traceback (fold.go:808-858) ------------------------------------------------------------------------
// A W cell as traceback sees it: the fill's value where the reference computed it, else "never computed"
// (-inf) or "invalid" (+inf) for short cells, by whether a probe of the top-down recursion reached them.
// Only the root's own probe, the W(i +- 1) recursion and W's multibranch count: a short cell is +-inf, so
// it can only equal the structure a shift loop walks when that is the +inf root, and then no V cell with
// j - i >= 4 is finite (W(0, n-1) <= V(i, j)), so no V cell ran its multibranch loop.
__device__ bool w_probed(const Item &it, int a, int b) {
    const int n = it.n, d = b - a;
    if (a == 0 && b == n - 1) return true;
    if (d == 3 && (a >= 1 || b <= n - 2)) return true;                  // W(a-1, b) or W(a, b+1) recursed
    return d >= 1 && ((a + 4 <= n - 1 && b + 2 <= n - 1) || (a >= 2 && b >= 4));  // W's multibranch
}
struct Cell {
    double e;
    uint64_t d;
};
__device__ Cell w_cell(const Item &it, int i, int j) {
    if (i > j) return {-INFINITY, K_NONE};
    if (j - i < 4) return {w_probed(it, i, j) ? INFINITY : -INFINITY, K_NONE};
    return {it.We[it.at(i, j)], it.Wd[it.at(i, j)]};
}
__device__ int inner_len(const Item &it, uint64_t d) {
    switch (d & KIND_MASK) {
        case K_NONE: return 0;
        case K_ONE: return 1;
        default: return branches_of(it, dA(d), dC(d), dB(d), (d & KIND_MASK) == K_MULTI_V).nl +
                        branches_of(it, dA(d), dC(d), dB(d), (d & KIND_MASK) == K_MULTI_V).nr;
    }
}
__device__ uint32_t inner_at(const Item &it, uint64_t d, int k) {
    if ((d & KIND_MASK) == K_ONE) return bpack(dA(d), dB(d));
    return branches_of(it, dA(d), dC(d), dB(d), (d & KIND_MASK) == K_MULTI_V)[k];
}
__device__ bool equal(const Item &it, Cell x, Cell y) {
    const int nx = inner_len(it, x.d), ny = inner_len(it, y.d);
    if (nx != ny) return false;
    for (int k = 0; k < nx; ++k)
        if (inner_at(it, x.d, k) != inner_at(it, y.d, k)) return false;
    return x.e == y.e;
}
// the shift loops; false where the reference indexes out of range
__device__ bool shift(const Item &it, int &start, int &end) {
    const Cell s = w_cell(it, start, end);
    if (s.d & HAIRPIN_BIT) return true;
    for (;;) {
        if (start + 1 >= it.n) return false;
        if (!equal(it, w_cell(it, start + 1, end), s)) break;
        ++start;
    }
    for (;;) {
        if (end - 1 < 0) return false;
        if (!equal(it, w_cell(it, start, end - 1), s)) break;
        --end;
    }
    return true;
}

constexpr int kStack = 256;
constexpr int kThreads = 128;

__global__ void __launch_bounds__(kThreads) fold_zuker_kernel(const uint8_t *__restrict__ seqs, const uint64_t *__restrict__ off,
                                                              uint64_t n_items, const FoldTables *__restrict__ tabs,
                                                              uint8_t *__restrict__ scratch, const uint64_t *__restrict__ scr_off,
                                                              double *__restrict__ mfe, uint8_t *__restrict__ db, uint64_t *__restrict__ db_len,
                                                              int32_t *__restrict__ status) {
    __shared__ uint64_t doff[PG_FOLD_MAX_LEN + 1];
    __shared__ uint32_t stk[kStack];
    __shared__ int s_hi, s_notdna, s_notrna, s_err;
    for (uint64_t item = blockIdx.x; item < n_items; item += gridDim.x) {
        const uint8_t *seq = seqs + off[item];
        const uint64_t len = off[item + 1] - off[item];
        uint8_t *dbo = db + (off[item] - off[0]);
        if (threadIdx.x == 0) { s_hi = 0; s_notdna = 0; s_notrna = 0; s_err = 0; }
        __syncthreads();
        // prepass: strings.ToUpper, then checks.IsDNA / checks.IsRNA (seqfold.go:149-160)
        int hi = 0, nd = 0, nr = 0;
        for (uint64_t i = threadIdx.x; i < len; i += blockDim.x) {
            uint8_t b = seq[i];
            if (b >= 0x80) hi = 1;
            if (b >= 'a' && b <= 'z') b -= 32;
            if (!(b == 'A' || b == 'C' || b == 'G' || b == 'T')) nd = 1;
            if (!(b == 'A' || b == 'C' || b == 'G' || b == 'U')) nr = 1;
        }
        if (hi) atomicOr(&s_hi, 1);
        if (nd) atomicOr(&s_notdna, 1);
        if (nr) atomicOr(&s_notrna, 1);
        __syncthreads();
        int st = PG_ITEM_OK;
        if (s_hi) st = PG_ITEM_UNSUPPORTED;           // ToUpper re-encodes such bytes: the message is not reproduced
        else if (s_notdna && s_notrna) st = PG_ITEM_FOLD_NOT_NUCLEIC;
        else if (len < 2) st = PG_ITEM_PANIC;         // empty cache (seqfold.go:187) or W[1][0] in traceback
        else if (len > PG_FOLD_MAX_LEN) st = PG_ITEM_UNSUPPORTED;
        if (st != PG_ITEM_OK) {
            for (uint64_t i = threadIdx.x; i < len; i += blockDim.x) dbo[i] = '.';  // a deterministic output region
            if (threadIdx.x == 0) { status[item] = st; mfe[item] = 0; db_len[item] = 0; }
            __syncthreads();
            continue;
        }
        const int n = (int)len;
        uint8_t *base = scratch + scr_off[item];
        Item it;
        it.n = n;
        it.t = tabs + (s_notdna ? 1 : 0);
        const uint64_t nn = (uint64_t)n * n;
        it.code = base;
        it.Ve = (double *)(base + align8(n));
        it.We = it.Ve + nn;
        it.Vd = (uint64_t *)(it.We + nn);
        it.Wd = it.Vd + nn;
        it.Lc = (uint16_t *)(it.Wd + nn);
        it.arena = (uint32_t *)(base + align8(n) + 32 * nn + align8(2 * nn));
        it.doff = doff;
        it.err = &s_err;
        for (int i = threadIdx.x; i < n; i += blockDim.x) {
            uint8_t b = seq[i];
            if (b >= 'a' && b <= 'z') b -= 32;
            it.code[i] = b == 'A' ? 0 : b == 'C' ? 1 : b == 'G' ? 2 : 3;
        }
        if (threadIdx.x == 0) {
            uint64_t a = 0;
            for (int d = 0; d < n; ++d) { doff[d] = a; a += (uint64_t)(n - d) * cap_of(d); }
        }
        for (uint64_t x = threadIdx.x; x < nn; x += blockDim.x) {  // never computed V; W as the fill reads it
            it.Ve[x] = -INFINITY; it.Vd[x] = K_NONE; it.We[x] = INFINITY; it.Wd[x] = K_NONE; it.Lc[x] = 0;
        }
        __syncthreads();
        for (int d = 4; d < n; ++d) {
            for (int i = threadIdx.x; i < n - d; i += blockDim.x) fill_v(it, i, i + d);
            __syncthreads();
            for (int i = threadIdx.x; i < n - d; i += blockDim.x) fill_w(it, i, i + d);
            __syncthreads();
        }
        if (threadIdx.x == 0) {
            int rc = s_err ? PG_ITEM_FOLD_INTERNAL : PG_ITEM_OK;
            double sum = 0.0;
            int last = 0, sp = 0;
            for (int i = 0; i < n; ++i) dbo[i] = '.';
            stk[sp++] = bpack(0, n - 1);
            while (rc == PG_ITEM_OK && sp > 0) {
                const uint32_t top = stk[--sp];
                const bool shifted = top >> 31;  // a branch whose shift loops already ran
                int s = (int)((top >> 16) & 0x7fff), e = be(top);
                if (!shifted && !shift(it, s, e)) { rc = PG_ITEM_PANIC; break; }
                for (;;) {
                    const double ve = it.Ve[it.at(s, e)];
                    const uint64_t vd = it.Vd[it.at(s, e)];
                    const uint64_t kind = vd & KIND_MASK;
                    dbo[s] = '(';
                    dbo[e] = ')';
                    last = max(last, e);
                    if (kind == K_NONE) { sum += ve; break; }
                    if (kind == K_ONE) {
                        const int r = dA(vd), l = dB(vd);
                        sum += ve - it.Ve[it.at(r, l)];
                        s = r; e = l;
                        continue;
                    }
                    const Branches br = branches_of(it, dA(vd), dC(vd), dB(vd), kind == K_MULTI_V);
                    const int nb = br.nl + br.nr;
                    if (sp + nb > kStack) { rc = PG_ITEM_FOLD_INTERNAL; break; }
                    double summed = 0.0;
                    for (int k = 0; k < nb; ++k) {
                        int bs0 = bs(br[k]), be0 = be(br[k]);
                        if (!shift(it, bs0, be0)) { rc = PG_ITEM_PANIC; break; }
                        summed += w_cell(it, bs0, be0).e;
                        stk[sp + nb - 1 - k] = 0x80000000u | bpack(bs0, be0);
                    }
                    if (rc != PG_ITEM_OK) break;
                    sp += nb;
                    sum += ve - summed;
                    break;
                }
            }
            if (rc != PG_ITEM_OK)
                for (int i = 0; i < n; ++i) dbo[i] = '.';
            status[item] = rc;
            mfe[item] = rc == PG_ITEM_OK ? sum : 0;
            db_len[item] = rc == PG_ITEM_OK ? (uint64_t)last + 1 : 0;
        }
        __syncthreads();
    }
}

}  // namespace

uint64_t fold_scratch_bytes(uint64_t len) {
    if (len < 2 || len > PG_FOLD_MAX_LEN) return 0;
    const uint64_t nn = len * len;
    return align8(align8(len) + 32 * nn + align8(2 * nn) + 4 * arena_entries((int)len));
}

static int code_of(char c) { return c == 'A' ? 0 : c == 'C' ? 1 : c == 'G' ? 2 : (c == 'T' || c == 'U') ? 3 : c == '.' ? 4 : -1; }

// the two tables (DNA, RNA) at temp degrees Celsius: deltaG = H - T * (S / 1000), T = temp + 273.15
std::vector<uint8_t> fold_tables(double temp) {
    std::vector<uint8_t> out(2 * sizeof(FoldTables));
    const double T = temp + 273.15;
    auto dG = [T](double h, double s) { return h - T * (s / 1000.0); };
    for (int kind = 0; kind < 2; ++kind) {
        FoldTables &t = ((FoldTables *)out.data())[kind];
        memset(&t, 0, sizeof t);
        t.rna = kind;
        const KeyEnergy *keyed[4] = {kind ? k_rna_nearestNeighbors : k_dna_nearestNeighbors, kind ? k_rna_internalMismatches : k_dna_internalMismatches,
                                     kind ? k_rna_terminalMismatches : k_dna_terminalMismatches, kind ? k_rna_danglingEnds : k_dna_danglingEnds};
        for (int x = 0; x < 4; ++x) {
            for (int k = 0; k < 625; ++k) t.dg[x][k] = dG(0, 0);
            for (const KeyEnergy *e = keyed[x]; e->key; ++e) {
                const char *s = e->key;
                if (strlen(s) != 5 || s[2] != '/') continue;  // "init", "sym", ...: never a pair() key
                const int c0 = code_of(s[0]), c1 = code_of(s[1]), c3 = code_of(s[3]), c4 = code_of(s[4]);
                if (c0 < 0 || c1 < 0 || c3 < 0 || c4 < 0) continue;
                const int k = c0 * 125 + c1 * 25 + c3 * 5 + c4;
                t.dg[x][k] = dG(e->h, e->s);
                t.has[x][k] = 1;
            }
        }
        const LenEnergy *loops[3] = {kind ? k_rna_internalLoops : k_dna_internalLoops, kind ? k_rna_bulgeLoops : k_dna_bulgeLoops,
                                     kind ? k_rna_hairpinLoops : k_dna_hairpinLoops};
        for (int x = 0; x < 3; ++x) {
            bool has[PG_FOLD_MAX_LEN + 1] = {};
            double h30 = 0, s30 = 0;
            for (const LenEnergy *e = loops[x]; e->len >= 0; ++e) {
                if (e->len <= PG_FOLD_MAX_LEN) { t.loop[x][e->len] = dG(e->h, e->s); has[e->len] = true; }
                if (e->len == 30) { h30 = e->h; s30 = e->s; }
            }
            for (int len = 0; len <= PG_FOLD_MAX_LEN; ++len) {  // fold.go:762-765, through libm's log
                if (has[len]) continue;
                const double gasConstant = 1.9872e-3;
                t.loop[x][len] = dG(h30, s30) + 2.44 * gasConstant * T * log((double)len / (double)30);
            }
        }
        const double *mb = kind ? k_rna_multibranch : k_dna_multibranch;
        for (int i = 0; i < 4; ++i) t.mb[i] = mb[i];
        for (const KeyEnergy *e = kind ? k_rna_triTetraLoops : k_dna_triTetraLoops; e->key && t.n_tri < kMaxTri; ++e) {
            const int len = (int)strlen(e->key);
            uint32_t key = (uint32_t)len << 12;
            bool ok = len <= 6;
            for (int i = 0; i < len && ok; ++i) {
                const int c = code_of(e->key[i]);
                ok = c >= 0 && c < 4;
                key |= (uint32_t)(ok ? c : 0) << (2 * i);
            }
            if (!ok) continue;
            t.tri_key[t.n_tri] = key;
            t.tri_dg[t.n_tri++] = dG(e->h, e->s);
        }
    }
    return out;
}

int launch_fold_zuker(const uint8_t *d_seqs, const uint64_t *d_off, uint64_t n, const uint8_t *d_tables, uint8_t *d_scratch,
                      const uint64_t *d_scr_off, double *d_mfe, uint8_t *d_db, uint64_t *d_db_len, int32_t *d_status, cudaStream_t st) {
    if (n == 0) return PG_OK;
    const unsigned grid = (unsigned)std::min<uint64_t>(n, 1u << 20);
    fold_zuker_kernel<<<grid, kThreads, 0, st>>>(d_seqs, d_off, n, (const FoldTables *)d_tables, d_scratch, d_scr_off, d_mfe, d_db, d_db_len, d_status);
    PG_LAUNCH_CHECK("fold_zuker_kernel");
    return PG_OK;
}

}  // namespace pg
