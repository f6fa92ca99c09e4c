/* CPU restatement of poly's fold package (fold.go, seqfold.go): Zuker minimum free energy and dot-bracket.
 *
 * TEST INFRASTRUCTURE ONLY.  It keeps the reference's shape on purpose: the top-down memoised recursion
 * over V and W caches that start at defaultStructure (-inf, no inner), the inner lists and descriptions
 * of every structure, addBranch, the Go `%` neighbour quirk and the traceback with its Equal-based shift
 * loops.  So the cells the reference never computes stay "never computed" here by construction.
 * Go panics (index out of range) become FO_PANIC; Go errors become FO_NOT_NUCLEIC or FO_INTERNAL.
 * Built with -ffp-contract=off: every float64 operation is the reference's, in its order.
 * The energy tables come from tests/golden/fold/energies.json through fo_set_table. */
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "parallel.h"
#include "poly_oracle.h"

enum { FO_OK = 0, FO_PANIC = 1, FO_UNSUPPORTED = 2, FO_NOT_NUCLEIC = 3, FO_INTERNAL = 4 };
enum { T_NN, T_IM, T_TM, T_DE, T_TRI, T_IL, T_BL, T_HL, T_COUNT };

#define MAX_KEYS 512
typedef struct {
    int n[T_COUNT];
    char key[T_COUNT][MAX_KEYS][8];
    double h[T_COUNT][MAX_KEYS], s[T_COUNT][MAX_KEYS];
    double mb[4];
    int present;
    short dense[T_COUNT][1296]; /* index + 1 of each "ab/cd" key over ACGTU. (the map's hash, nothing more) */
} Energies;
static int code6(char c) {
    switch (c) {
    case 'A': return 0; case 'C': return 1; case 'G': return 2; case 'T': return 3; case 'U': return 4; case '.': return 5;
    }
    return -1;
}
static int key6(const char *k) {
    if (strlen(k) != 5 || k[2] != '/') return -1;
    int a = code6(k[0]), b = code6(k[1]), c = code6(k[3]), d = code6(k[4]);
    if (a < 0 || b < 0 || c < 0 || d < 0) return -1;
    return ((a * 6 + b) * 6 + c) * 6 + d;
}
static Energies g_tab[2]; /* 0 DNA, 1 RNA */

/* table `t` of kind (0 DNA, 1 RNA): keys are strings (loop tables: decimal lengths) */
void fo_set_table(int kind, int t, int count, const char *keys /* count * 8 bytes */, const double *h, const double *s) {
    Energies *e = &g_tab[kind];
    e->n[t] = count;
    for (int i = 0; i < count; ++i) {
        memcpy(e->key[t][i], keys + 8 * i, 8);
        e->h[t][i] = h[i];
        e->s[t][i] = s[i];
    }
    memset(e->dense[t], 0, sizeof e->dense[t]);
    for (int i = 0; i < count; ++i) {
        int k = key6(e->key[t][i]);
        if (k >= 0) e->dense[t][k] = (short)(i + 1);
    }
    e->present = 1;
}
void fo_set_multibranch(int kind, const double *mb) { memcpy(g_tab[kind].mb, mb, sizeof(g_tab[kind].mb)); }

typedef struct { int start, end; } subsequence;
typedef struct {
    char description[48];
    subsequence *inner;
    int ninner;
    double energy;
} nas;

typedef struct {
    const Energies *en;
    int rna;
    const char *seq;
    int n;
    nas *V, *W; /* n * n */
    double temp;
    int err; /* first Go error (FO_INTERNAL) */
} context;

static const nas defaultStructure = {"", NULL, 0, -INFINITY};
static const nas invalidStructure = {"", NULL, 0, INFINITY};

enum { isolatedBasePairPenalty = 1600, maxLenPreCalulated = 30, minLenForStruct = 4 };
static const double loopsAsymmetryPenalty = 0.3, closingATPenalty = 0.5;

static int equal(nas a, nas b) {
    if (a.ninner != b.ninner) return 0;
    for (int i = 0; i < a.ninner; ++i)
        if (a.inner[i].start != b.inner[i].start || a.inner[i].end != b.inner[i].end) return 0;
    return a.energy == b.energy;
}
static int valid(nas a) { return a.energy != INFINITY && a.energy != -INFINITY; }

/* map lookup: 1 and (h, s) if present */
static int lookup(const context *c, int t, const char *key, double *h, double *s) {
    const Energies *e = c->en;
    int k6 = key6(key);
    if (k6 >= 0) {
        int i = e->dense[t][k6] - 1;
        if (i >= 0) { *h = e->h[t][i]; *s = e->s[t][i]; return 1; }
        *h = 0; *s = 0;
        return 0;
    }
    for (int i = 0; i < e->n[t]; ++i)
        if (strcmp(e->key[t][i], key) == 0) { *h = e->h[t][i]; *s = e->s[t][i]; return 1; }
    *h = 0; *s = 0; /* Go's zero value for a missing key */
    return 0;
}
static int lookup_len(const context *c, int t, int len, double *h, double *s) {
    char k[12];
    snprintf(k, sizeof k, "%d", len);
    return lookup(c, t, k, h, s);
}

static char complement(const context *c, char b) {
    switch (b) {
    case 'A': return c->rna ? 'U' : 'T';
    case 'T': return 'A';
    case 'U': return 'A';
    case 'C': return 'G';
    case 'G': return 'C';
    }
    return ' ';
}

static double deltaG(double h, double s, double temp) { return h - temp * (s / 1000.0); }
static double jacobsonStockmayer(int queryLen, int knownLen, double dGx, double temp) {
    double gasConstant = 1.9872e-3;
    return dGx + 2.44 * gasConstant * temp * log((double)queryLen / (double)knownLen);
}
/* Go's math.Min, whose documented special cases come in this order: Min(x, -Inf) = Min(-Inf, x) = -Inf,
 * Min(x, NaN) = Min(NaN, x) = NaN, Min(-0, +-0) = Min(+-0, -0) = -0 */
static double go_min(double a, double b) {
    if (isinf(a) && a < 0) return a;
    if (isinf(b) && b < 0) return b;
    if (isnan(a) || isnan(b)) return NAN;
    if (a == 0 && b == 0) return signbit(a) ? a : b;
    return a < b ? a : b;
}

static void pair(const char *s, int start, int rightOfStart, int end, int leftOfEnd, char out[6]) {
    out[0] = start >= 0 ? s[start] : '.';
    out[1] = rightOfStart >= 0 ? s[rightOfStart] : '.';
    out[2] = '/';
    out[3] = end >= 0 ? s[end] : '.';
    out[4] = leftOfEnd >= 0 ? s[leftOfEnd] : '.';
    out[5] = 0;
}

static double stack(int start, int rightOfStart, int end, int leftOfEnd, const context *c) {
    int idx[4] = {start, rightOfStart, end, leftOfEnd};
    for (int k = 0; k < 4; ++k)
        if (idx[k] >= c->n) return 0;
    char p[6];
    double h, s;
    pair(c->seq, start, rightOfStart, end, leftOfEnd, p);
    for (int k = 0; k < 4; ++k)
        if (idx[k] == -1) {
            lookup(c, T_DE, p, &h, &s);
            return deltaG(h, s, c->temp);
        }
    if ((start > 0 && end < c->n - 1) || (start == 0 && end == c->n - 1)) {
        if (!lookup(c, T_NN, p, &h, &s)) lookup(c, T_IM, p, &h, &s);
        return deltaG(h, s, c->temp);
    }
    if (start > 0 && end == c->n - 1) {
        if (!lookup(c, T_NN, p, &h, &s)) lookup(c, T_IM, p, &h, &s);
        double dG = deltaG(h, s, c->temp);
        char de[6] = {c->seq[start - 1], c->seq[start], '/', '.', c->seq[end], 0};
        if (lookup(c, T_DE, de, &h, &s)) dG += deltaG(h, s, c->temp);
        return dG;
    }
    if (start == 0 && end < c->n - 1) {
        if (!lookup(c, T_NN, p, &h, &s)) lookup(c, T_IM, p, &h, &s);
        double dG = deltaG(h, s, c->temp);
        char de[6] = {'.', c->seq[start], '/', c->seq[end + 1], c->seq[end], 0};
        if (lookup(c, T_DE, de, &h, &s)) {
            dG += deltaG(h, s, c->temp);
            return dG;
        }
    }
    return 0;
}

static int hairpin(int start, int end, context *c, double *out) {
    if (end - start < minLenForStruct) { *out = INFINITY; return 0; }
    const char *hp = c->seq + start;
    int len = end - start + 1, hairpinLength = len - 2;
    char p[6];
    double h, s;
    pair(c->seq, start, start + 1, end, end - 1, p);
    if (complement(c, hp[0]) != hp[len - 1]) return FO_INTERNAL;
    double dG = 0.0;
    if (!c->rna && len < 8) {
        char k[8];
        memcpy(k, hp, len);
        k[len] = 0;
        if (lookup(c, T_TRI, k, &h, &s)) dG = deltaG(h, s, c->temp);
    }
    if (lookup_len(c, T_HL, hairpinLength, &h, &s)) {
        dG += deltaG(h, s, c->temp);
    } else {
        lookup_len(c, T_HL, maxLenPreCalulated, &h, &s);
        double dGinc = deltaG(h, s, c->temp);
        dG += jacobsonStockmayer(hairpinLength, maxLenPreCalulated, dGinc, c->temp);
    }
    int ok = lookup(c, T_TM, p, &h, &s);
    if (hairpinLength > 3 && ok) dG += deltaG(h, s, c->temp);
    if (hairpinLength == 3 && (hp[0] == 'A' || hp[len - 1] == 'A')) dG += closingATPenalty;
    *out = dG;
    return 0;
}

static int Bulge(int start, int rightOfStart, int end, int leftOfEnd, context *c, double *out) {
    int a = rightOfStart - start - 1, b = end - leftOfEnd - 1;
    int loopLength = a > b ? a : b;
    if (loopLength <= 0) return FO_INTERNAL;
    double dG, h, s;
    if (lookup_len(c, T_BL, loopLength, &h, &s)) {
        dG = deltaG(h, s, c->temp);
    } else {
        lookup_len(c, T_BL, maxLenPreCalulated, &h, &s);
        dG = deltaG(h, s, c->temp);
        dG = jacobsonStockmayer(loopLength, maxLenPreCalulated, dG, c->temp);
    }
    if (loopLength == 1) {
        char p[6];
        pair(c->seq, start, rightOfStart, end, leftOfEnd, p);
        if (!lookup(c, T_NN, p, &h, &s)) return FO_INTERNAL;
        dG += stack(start, rightOfStart, end, leftOfEnd, c);
    }
    int ks[4] = {start, rightOfStart, end, leftOfEnd};
    for (int k = 0; k < 4; ++k)
        if (c->seq[ks[k]] == 'A') dG += closingATPenalty;
    *out = dG;
    return 0;
}

static int internalLoop(int start, int rightOfStart, int end, int leftOfEnd, context *c, double *out) {
    int loopLeftIndex = rightOfStart - start - 1, loopRightIndex = end - leftOfEnd - 1;
    int loopLength = loopLeftIndex + loopRightIndex;
    if (loopLeftIndex < 1 || loopRightIndex < 1) return FO_INTERNAL;
    if (loopLeftIndex == 1 && loopRightIndex == 1) {
        double l = stack(start, rightOfStart, end, leftOfEnd, c);
        double r = stack(rightOfStart - 1, rightOfStart, leftOfEnd + 1, leftOfEnd, c);
        *out = l + r;
        return 0;
    }
    double h, s, dG;
    if (lookup_len(c, T_IL, loopLength, &h, &s)) {
        dG = deltaG(h, s, c->temp);
    } else {
        lookup_len(c, T_IL, maxLenPreCalulated, &h, &s);
        dG = deltaG(h, s, c->temp);
        dG = jacobsonStockmayer(loopLength, maxLenPreCalulated, dG, c->temp);
    }
    double loopAsymmetry = fabs((double)(loopLeftIndex - loopRightIndex));
    dG += loopsAsymmetryPenalty * loopAsymmetry;
    char p[6];
    pair(c->seq, start, start + 1, end, end - 1, p);
    lookup(c, T_TM, p, &h, &s);
    dG += deltaG(h, s, c->temp);
    pair(c->seq, rightOfStart - 1, rightOfStart, leftOfEnd + 1, leftOfEnd, p);
    lookup(c, T_TM, p, &h, &s);
    dG += deltaG(h, s, c->temp);
    *out = dG;
    return 0;
}

static nas *Vc(context *c, int i, int j) { return &c->V[(size_t)i * c->n + j]; }
static nas *Wc(context *c, int i, int j) { return &c->W[(size_t)i * c->n + j]; }

static nas W(int start, int end, context *c);
static nas V(int start, int end, context *c);

typedef struct { subsequence *v; int n, cap; } blist;
static void bpush(blist *b, subsequence s) {
    if (b->n == b->cap) { b->cap = b->cap ? 2 * b->cap : 8; b->v = realloc(b->v, b->cap * sizeof *b->v); }
    b->v[b->n++] = s;
}

static void addBranch(nas structure, blist *branches, context *c) {
    if (!valid(structure) || structure.ninner == 0) return;
    if (structure.ninner == 1) { bpush(branches, structure.inner[0]); return; }
    for (int k = 0; k < structure.ninner; ++k) {
        nas s = W(structure.inner[k].start, structure.inner[k].end, c);
        if (c->err) return;
        addBranch(s, branches, c);
        if (c->err) return;
    }
}

/* the returned inner list is malloc'd (the caller keeps or frees it) */
static nas multibranch(int start, int mid, int end, context *c, int helix) {
    nas left, right;
    if (helix) {
        left = W(start + 1, mid, c);
        if (c->err) return defaultStructure;
        right = W(mid + 1, end - 1, c);
    } else {
        left = W(start, mid, c);
        if (c->err) return defaultStructure;
        right = W(mid + 1, end, c);
    }
    if (c->err) return defaultStructure;
    if (!valid(left) || !valid(right)) return invalidStructure;
    blist br = {0};
    addBranch(left, &br, c);
    if (!c->err) addBranch(right, &br, c);
    if (c->err) { free(br.v); return defaultStructure; }
    if (br.n < 2) { free(br.v); return invalidStructure; }
    if (helix) bpush(&br, (subsequence){start, end});
    int branchCount = br.n, unpaired = 0;
    double summedEnergy = 0.0;
    subsequence cur = {start, end};
    for (int index = 0; index < br.n; ++index) {
        subsequence currentBranch = br.v[index];
        int leftStart = currentBranch.start, leftEnd = currentBranch.end;
        subsequence curBranchLeft = br.v[abs((index - 1) % br.n)];
        int leftOfEnd = curBranchLeft.end;
        subsequence curBranchRight = br.v[abs((index + 1) % br.n)];
        int rightStart = curBranchRight.start, rightEnd = curBranchRight.end;
        int unpairedLeft = 0, unpairedRight = 0;
        double danglingEnergy = 0.0;
        if (index == br.n - 1 && !helix) {
        } else if (curBranchRight.start == cur.start && curBranchRight.end == cur.end) {
            unpairedLeft = leftStart - leftOfEnd - 1;
            unpairedRight = rightEnd - leftEnd - 1;
            if (unpairedLeft != 0 && unpairedRight != 0) {
                danglingEnergy = stack(leftStart - 1, leftStart, leftEnd + 1, leftEnd, c);
            } else if (unpairedRight != 0) {
                danglingEnergy = stack(-1, leftStart, leftEnd + 1, leftEnd, c);
                if (unpairedRight == 1) danglingEnergy = go_min(stack(rightStart, -1, rightEnd, rightEnd - 1, c), danglingEnergy);
            }
        } else if (currentBranch.start == cur.start && currentBranch.end == cur.end) {
            unpairedLeft = leftEnd - leftOfEnd - 1;
            unpairedRight = rightStart - leftStart - 1;
            if (unpairedLeft != 0 && unpairedRight != 0) {
                danglingEnergy = stack(leftStart - 1, leftStart, leftEnd + 1, leftEnd, c);
            } else if (unpairedRight != 0) {
                danglingEnergy = stack(leftStart, leftStart + 1, leftEnd, -1, c);
                if (unpairedRight == 1) danglingEnergy = go_min(stack(rightStart - 1, rightStart, -1, rightEnd, c), danglingEnergy);
            }
        } else {
            unpairedLeft = leftStart - leftOfEnd - 1;
            unpairedRight = rightStart - leftEnd - 1;
            if (unpairedLeft != 0 && unpairedRight != 0) {
                danglingEnergy = stack(leftStart - 1, leftStart, leftEnd + 1, leftEnd, c);
            } else if (unpairedRight != 0) {
                danglingEnergy = stack(-1, leftStart, leftEnd + 1, leftEnd, c);
                if (unpairedRight == 1) danglingEnergy = go_min(stack(leftStart - 1, leftStart, leftEnd + 1, leftEnd, c), danglingEnergy);
            }
        }
        summedEnergy += danglingEnergy;
        unpaired += unpairedRight;
        if (unpairedRight < 0) { c->err = FO_INTERNAL; free(br.v); return defaultStructure; }
        if (!(currentBranch.start == cur.start && currentBranch.end == cur.end)) {
            nas w = W(leftStart, leftEnd, c);
            if (c->err) { free(br.v); return defaultStructure; }
            summedEnergy += w.energy;
        }
    }
    if (unpaired < 0) { c->err = FO_INTERNAL; free(br.v); return defaultStructure; }
    const double *mb = c->en->mb;
    double multibranchEnergy = mb[0] + mb[1] * (double)br.n + mb[2] * (double)unpaired;
    if (unpaired == 0) multibranchEnergy = mb[0] + mb[3];
    double e = multibranchEnergy + summedEnergy;
    if (helix) br.n--;
    nas r;
    snprintf(r.description, sizeof r.description, "BIFURCATION:%dn/%dh", unpaired, branchCount);
    r.inner = br.v;
    r.ninner = br.n;
    r.energy = e;
    return r;
}

static nas minimumStructure(const nas *s, int k) {
    nas m = invalidStructure;
    for (int i = 0; i < k; ++i)
        if (s[i].energy != -INFINITY && s[i].energy < m.energy) m = s[i];
    return m;
}

static nas W(int start, int end, context *c) {
    if (start >= c->n || end < 0 || start < 0 || end >= c->n) { c->err = FO_PANIC; return defaultStructure; }
    if (!equal(*Wc(c, start, end), defaultStructure)) return *Wc(c, start, end);
    if (end - start < minLenForStruct) { *Wc(c, start, end) = invalidStructure; return invalidStructure; }
    nas s[4];
    s[0] = W(start + 1, end, c);
    if (c->err) return defaultStructure;
    s[1] = W(start, end - 1, c);
    if (c->err) return defaultStructure;
    s[2] = V(start, end, c);
    if (c->err) return defaultStructure;
    nas bif = invalidStructure;
    for (int k = start + 1; k < end - 1; ++k) {
        nas t = multibranch(start, k, end, c, 0);
        if (c->err) { free(bif.inner); return defaultStructure; }
        if (valid(t) && t.energy < bif.energy) { free(bif.inner); bif = t; } else free(t.inner);
    }
    s[3] = bif;
    nas m = minimumStructure(s, 4);
    if (m.inner != bif.inner) free(bif.inner);
    *Wc(c, start, end) = m;
    return m;
}

static nas V(int start, int end, context *c) {
    if (!equal(*Vc(c, start, end), defaultStructure)) return *Vc(c, start, end);
    const char *seq = c->seq;
    int n = c->n;
    if (complement(c, seq[start]) != seq[end]) { *Vc(c, start, end) = invalidStructure; return invalidStructure; }
    int isolatedOuter = 1;
    if (start > 0 && end < n - 1) isolatedOuter = complement(c, seq[start - 1]) != seq[end + 1];
    int isolatedInner = complement(c, seq[start + 1]) != seq[end - 1];
    if (isolatedOuter && isolatedInner) {
        nas iso = {"", NULL, 0, isolatedBasePairPenalty};
        *Vc(c, start, end) = iso;
        return iso;
    }
    char paired[6];
    pair(seq, start, start + 1, end, end - 1, paired);
    double hp;
    int rc = hairpin(start, end, c, &hp);
    if (rc) { c->err = rc; return defaultStructure; }
    nas e1 = {"", NULL, 0, hp};
    snprintf(e1.description, sizeof e1.description, "HAIRPIN:%s", paired);
    if (end - start == minLenForStruct) {
        *Vc(c, start, end) = e1;
        *Wc(c, start, end) = e1;
        return e1;
    }
    nas e2 = {"", NULL, 0, INFINITY};
    for (int rightOfStart = start + 1; rightOfStart < end - minLenForStruct; ++rightOfStart) {
        for (int leftOfEnd = rightOfStart + minLenForStruct; leftOfEnd < end; ++leftOfEnd) {
            if (complement(c, seq[rightOfStart]) != seq[leftOfEnd]) continue;
            char p[6], pl[6], pr[6];
            double h, s;
            pair(seq, start, rightOfStart, end, leftOfEnd, p);
            pair(seq, start, start + 1, end, end - 1, pl);
            pair(seq, rightOfStart - 1, rightOfStart, leftOfEnd + 1, leftOfEnd, pr);
            int pairLeftInner = lookup(c, T_NN, pl, &h, &s), pairRightInner = lookup(c, T_NN, pr, &h, &s);
            int pairInner = pairLeftInner || pairRightInner;
            int isStack = rightOfStart == start + 1 && leftOfEnd == end - 1;
            int bulgeLeft = rightOfStart > start + 1, bulgeRight = leftOfEnd < end - 1;
            double e2Test;
            char type[48];
            if (isStack) {
                e2Test = stack(start, rightOfStart, end, leftOfEnd, c);
                snprintf(type, sizeof type, "STACK:%s", p);
                if ((start > 0 && end == n - 1) || (start == 0 && end < n - 1)) snprintf(type, sizeof type, "STACKDanglingEnds:%s", p);
            } else if (bulgeLeft && bulgeRight && !pairInner) {
                if ((rc = internalLoop(start, rightOfStart, end, leftOfEnd, c, &e2Test))) { c->err = rc; free(e2.inner); return defaultStructure; }
                snprintf(type, sizeof type, "INTERIOR_LOOP:%d/%d", rightOfStart - start, end - leftOfEnd);
                if (rightOfStart - start == 2 && end - leftOfEnd == 2)
                    snprintf(type, sizeof type, "STACK:%c%c%c/%c%c%c", seq[start], seq[start + 1], seq[start + 2], seq[end], seq[end - 1], seq[end - 2]);
            } else if (bulgeLeft && !bulgeRight) {
                if ((rc = Bulge(start, rightOfStart, end, leftOfEnd, c, &e2Test))) { c->err = rc; free(e2.inner); return defaultStructure; }
                snprintf(type, sizeof type, "BULGE:%d", rightOfStart - start);
            } else if (!bulgeLeft && bulgeRight) {
                if ((rc = Bulge(start, rightOfStart, end, leftOfEnd, c, &e2Test))) { c->err = rc; free(e2.inner); return defaultStructure; }
                snprintf(type, sizeof type, "BULGE:%d", end - leftOfEnd);
            } else {
                continue;
            }
            nas tv = V(rightOfStart, leftOfEnd, c);
            if (c->err) { free(e2.inner); return defaultStructure; }
            e2Test += tv.energy;
            if (e2Test != -INFINITY && e2Test < e2.energy) {
                if (!e2.inner) e2.inner = malloc(sizeof(subsequence));
                e2.energy = e2Test;
                strcpy(e2.description, type);
                e2.inner[0] = (subsequence){rightOfStart, leftOfEnd};
                e2.ninner = 1;
            }
        }
    }
    nas e3 = invalidStructure;
    if (!isolatedOuter || start == 0 || end == n - 1) {
        for (int k = start + 1; k < end - 1; ++k) {
            nas t = multibranch(start, k, end, c, 1);
            if (c->err) { free(e2.inner); free(e3.inner); return defaultStructure; }
            if (valid(t) && t.energy < e3.energy) { free(e3.inner); e3 = t; } else free(t.inner);
        }
    }
    nas s[3] = {e1, e2, e3};
    nas e = minimumStructure(s, 3);
    if (e.inner != e2.inner) free(e2.inner);
    if (e.inner != e3.inner) free(e3.inner);
    *Vc(c, start, end) = e;
    return e;
}

/* ---- traceback and Result ---------------------------------------------------------------------------- */
typedef struct { nas *v; int n, cap; } slist;
static void spush(slist *l, nas s) {
    if (l->n == l->cap) { l->cap = l->cap ? 2 * l->cap : 16; l->v = realloc(l->v, l->cap * sizeof *l->v); }
    l->v[l->n++] = s;
}
static void trackbackEnergy(slist *l) {
    for (int start = 0; start < l->n - 1; ++start) l->v[start].energy -= l->v[start + 1].energy;
}
static nas one(nas s, int start, int end) {
    nas r = s;
    r.inner = malloc(sizeof(subsequence));
    r.inner[0] = (subsequence){start, end};
    r.ninner = 1;
    return r;
}
static int in_range(context *c, int i, int j) {
    if (i < 0 || i >= c->n || j < 0 || j >= c->n) { c->err = FO_PANIC; return 0; }
    return 1;
}

static slist traceback(int start, int end, context *c) {
    slist out = {0};
    nas structure = *Wc(c, start, end);
    if (!strstr(structure.description, "HAIRPIN")) {
        while (in_range(c, start + 1, end) && equal(*Wc(c, start + 1, end), structure)) start += 1;
        if (c->err) return out;
        while (in_range(c, start, end - 1) && equal(*Wc(c, start, end - 1), structure)) end -= 1;
        if (c->err) return out;
    }
    for (;;) {
        structure = *Vc(c, start, end);
        spush(&out, one(structure, start, end));
        if (structure.ninner == 0) { trackbackEnergy(&out); return out; }
        if (structure.ninner == 1) { start = structure.inner[0].start; end = structure.inner[0].end; continue; }
        double summedEnergy = 0.0;
        trackbackEnergy(&out);
        slist branches = {0};
        for (int k = 0; k < structure.ninner; ++k) {
            slist tb = traceback(structure.inner[k].start, structure.inner[k].end, c);
            if (c->err) { free(tb.v); free(branches.v); return out; }
            if (tb.n > 0 && tb.v[0].ninner > 0) {
                subsequence ss = tb.v[0].inner[0];
                summedEnergy += Wc(c, ss.start, ss.end)->energy;
                for (int t = 0; t < tb.n; ++t) spush(&branches, tb.v[t]);
            }
            free(tb.v);
        }
        out.v[out.n - 1].energy -= summedEnergy;
        for (int t = 0; t < branches.n; ++t) spush(&out, branches.v[t]);
        free(branches.v);
        return out;
    }
}

/* newFoldingContext: status, and on FO_OK a filled context (free with ctx_free) */
static int ctx_new(context *c, const char *raw, int64_t n, double temp, char **upper) {
    memset(c, 0, sizeof *c);
    char *seq = malloc(n + 1);
    *upper = seq;
    for (int64_t i = 0; i < n; ++i) {
        unsigned char b = (unsigned char)raw[i];
        if (b >= 0x80) return FO_UNSUPPORTED; /* strings.ToUpper re-encodes such bytes */
        seq[i] = (b >= 'a' && b <= 'z') ? (char)(b - 32) : (char)b;
    }
    seq[n] = 0;
    int dna = 1, rna = 1;
    for (int64_t i = 0; i < n; ++i) {
        char b = seq[i];
        if (!(b == 'A' || b == 'C' || b == 'T' || b == 'G')) dna = 0;
        if (!(b == 'A' || b == 'C' || b == 'U' || b == 'G')) rna = 0;
    }
    if (!dna && !rna) return FO_NOT_NUCLEIC;
    c->rna = !dna;
    c->en = &g_tab[c->rna];
    c->seq = seq;
    c->n = (int)n;
    c->temp = temp + 273.15;
    c->V = malloc(sizeof(nas) * (n > 0 ? n * n : 1));
    c->W = malloc(sizeof(nas) * (n > 0 ? n * n : 1));
    for (int64_t i = 0; i < n * n; ++i) c->V[i] = c->W[i] = defaultStructure;
    if (n == 0) return FO_PANIC; /* seqfold.go:187 indexes an empty cache */
    W(0, (int)n - 1, c);
    return c->err;
}

static int cmp_ptr(const void *a, const void *b) {
    uintptr_t x = *(const uintptr_t *)a, y = *(const uintptr_t *)b;
    return x < y ? -1 : x > y;
}
static void ctx_free(context *c) { /* inner lists are shared between cells: free each once */
    size_t m = (size_t)c->n * c->n, k = 0;
    uintptr_t *ps = malloc(sizeof(uintptr_t) * (2 * m + 1));
    for (size_t i = 0; i < m; ++i) {
        if (c->V[i].inner) ps[k++] = (uintptr_t)c->V[i].inner;
        if (c->W[i].inner) ps[k++] = (uintptr_t)c->W[i].inner;
    }
    qsort(ps, k, sizeof *ps, cmp_ptr);
    for (size_t i = 0; i < k; ++i)
        if (i == 0 || ps[i] != ps[i - 1]) free((void *)ps[i]);
    free(ps);
    free(c->V);
    free(c->W);
}

/* Zuker + MinimumFreeEnergy + DotBracket.  db needs n bytes.  If `structs` is not NULL it receives a
 * malloc'd text: one line per traceback struct, "<energy %a> <description> <start>,<end>;..." */
int fo_fold(const char *raw, int64_t n, double temp, double *mfe, char *db, int64_t *db_len, char **structs) {
    context c;
    char *upper = NULL;
    int st = ctx_new(&c, raw, n, temp, &upper);
    *mfe = 0;
    *db_len = 0;
    if (structs) *structs = NULL;
    if (st == FO_OK) {
        slist l = traceback(0, (int)n - 1, &c);
        st = c.err;
        if (st == FO_OK) {
            double e = 0.0;
            int last = 0;
            for (int i = 0; i < l.n; ++i) e += l.v[i].energy;
            if (l.n == 0) e = INFINITY;
            for (int i = 0; i < l.n; ++i)
                for (int k = 0; k < l.v[i].ninner; ++k)
                    if (l.v[i].inner[k].end > last) last = l.v[i].inner[k].end;
            int len = l.n ? last + 1 : 0;
            memset(db, '.', len);
            for (int i = 0; i < l.n; ++i)
                if (l.v[i].ninner == 1) { db[l.v[i].inner[0].start] = '('; db[l.v[i].inner[0].end] = ')'; }
            *mfe = e;
            *db_len = len;
            if (structs) {
                size_t cap = 256 + (size_t)l.n * 96, used = 0;
                char *t = malloc(cap);
                t[0] = 0;
                for (int i = 0; i < l.n; ++i) {
                    used += snprintf(t + used, cap - used, "%a %s ", l.v[i].energy, l.v[i].description[0] ? l.v[i].description : "-");
                    for (int k = 0; k < l.v[i].ninner; ++k) used += snprintf(t + used, cap - used, "%d,%d;", l.v[i].inner[k].start, l.v[i].inner[k].end);
                    used += snprintf(t + used, cap - used, "\n");
                }
                *structs = t;
            }
        }
        for (int i = 0; i < l.n; ++i) free(l.v[i].inner);
        free(l.v);
    }
    if (c.V) ctx_free(&c);
    free(upper);
    return st;
}

/* operands of which = 5: an index of fo_probe names one of these */
static const double go_min_operands[] = {-INFINITY, -1.0, -0.0, 0.0, 1.0, INFINITY, NAN};

/* One of the reference's internal functions on a filled context (for the reference tests' pins):
 * which 0 stack(a,b,c,d), 1 Bulge(a,b,c,d), 2 hairpin(a,b), 3 internalLoop(a,b,c,d), 4 W(a,b).energy,
 * 5 go_min(go_min_operands[a], go_min_operands[b]) */
int fo_probe(const char *raw, int64_t n, double temp, int which, int a, int b, int cc, int d, double *out) {
    context c;
    char *upper = NULL;
    int st = ctx_new(&c, raw, n, temp, &upper);
    if (st == FO_OK) {
        switch (which) {
        case 0: *out = stack(a, b, cc, d, &c); break;
        case 1: st = Bulge(a, b, cc, d, &c, out); break;
        case 2: st = hairpin(a, b, &c, out); break;
        case 3: st = internalLoop(a, b, cc, d, &c, out); break;
        case 5: *out = go_min(go_min_operands[a], go_min_operands[b]); break;
        default: *out = W(a, b, &c).energy; st = c.err; break;
        }
    }
    if (c.V) ctx_free(&c);
    free(upper);
    return st;
}

void fo_pair(const char *s, int a, int b, int c, int d, char *out) { pair(s, a, b, c, d, out); }
void fo_free(void *p) { free(p); }

/* ---- batch over threads ------------------------------------------------------------------------------ */
typedef struct {
    const uint8_t *seqs;
    const uint64_t *off;
    double temp;
    double *mfe;
    uint8_t *db;
    uint64_t *db_len;
    int32_t *status;
} Batch;

static void fold_one(void *arg, uint64_t i) {
    Batch *b = arg;
    int64_t len;
    b->status[i] = fo_fold((const char *)b->seqs + b->off[i], (int64_t)(b->off[i + 1] - b->off[i]), b->temp, &b->mfe[i],
                           (char *)b->db + b->off[i] - b->off[0], &len, NULL);
    b->db_len[i] = (uint64_t)len;
}

/* db is laid out like seqs (item i at off[i] - off[0]) */
int fo_fold_batch(const uint8_t *seqs, const uint64_t *off, uint64_t n, double temp, double *mfe, uint8_t *db, uint64_t *db_len, int32_t *status,
                  int threads) {
    Batch b = {seqs, off, temp, mfe, db, db_len, status};
    return po_parallel_for(n, threads, 1, fold_one, &b);
}
