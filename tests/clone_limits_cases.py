"""Seeded clone cases at the edges of the digest and ligation code, shared by test_clone_limits_host.py (CPU)
and test_gpu_clone_limits.py (GPU): a panel of caller-defined enzymes, part families that reach every branch
of the digest kernels (site lengths 1..32 at every offset of the 32-position walk, self-overlapping sites,
forward/reverse ties, extreme skips and overhang lengths, recognition-site corner cases), ligation reactions,
Golden Gate libraries for other enzymes, and an independent plain-Python restatement of clone.CutWithEnzyme
(the reference's clone/clone.go:138-268, restated from the Go, not from oracle/clone_oracle.c) that also
reports which paths a cut took.

An enzyme here is the tuple clone_oracle.cut takes: (forward site, reverse site, skip, overhang length,
recognition site), in the reference's convention (Position = match end + Skip forwards, match start - Skip
in reverse)."""
from __future__ import annotations

import random

import numpy as np

import seqhash_oracle
from clone_util import random_reaction

I32_MIN, I32_MAX = -(1 << 31), (1 << 31) - 1
OK, PANIC, UNSUPPORTED = 0, 1, 2  # clone_oracle's codes and PG_ITEM_*

# Real enzymes, REBASE-like; the exact values do not matter, only that they stay fixed.
PANEL = {
    "BsmBI": (b"CGTCTC", b"GAGACG", 1, 4, b"CGTCTC"),      # another 6-byte Type IIS
    "PaqCI": (b"CACCTGC", b"GCAGGTG", 4, 4, b"CACCTGC"),   # a 7-byte site
    "SapI": (b"GCTCTTC", b"GAAGAGC", 1, 3, b"GCTCTTC"),    # 3-nt overhangs
    "EcoRI": (b"GAATTC", b"GAATTC", -5, 4, b"GAATTC"),     # palindromic, G^AATTC: a negative skip
    "NotI": (b"GCGGCCGC", b"GCGGCCGC", -6, 4, b"GCGGCCGC"),  # palindromic 8-byte site, GC^GGCCGC
    "Bpu10I": (b"CCTNAGC", b"GCTNAGG", 2, 3, b"CCTNAGC"),  # N as a literal matches only an N byte
}

# ---- CutWithEnzyme restated (clone.go:138-268) -------------------------------------------------------------
# transform.complementTable (transform.go:78-109); every other byte maps to 0
_COMPLEMENT = bytearray(256)
for _a, _b in zip(b"ABCDGHKMNRSTVWYabcdghkmnrstvwy", b"TVGHCDMKNYSABWRtvghcdmknysabwr"):
    _COMPLEMENT[_a] = _b


def reverse_complement(s: bytes) -> bytes:
    return bytes(_COMPLEMENT[c] for c in reversed(s))


def is_palindromic(s: bytes) -> bool:
    """checks.IsPalindromic"""
    return s == reverse_complement(s)


class Panic(Exception):
    """A Go slice expression out of range: the reference panics."""


def go_slice(s: bytes, lo: int, hi: int | None = None) -> bytes:
    """s[lo:hi] with Go's bounds rule (0 <= lo <= hi <= len(s)); Python slicing would clamp instead."""
    hi = len(s) if hi is None else hi
    if not 0 <= lo <= hi <= len(s):
        raise Panic(f"slice bounds out of range [{lo}:{hi}] with length {len(s)}")
    return s[lo:hi]


def find_all(s: bytes, pat: bytes):
    """regexp.FindAllStringIndex of a literal: leftmost non-overlapping [start, end) matches"""
    out, i = [], s.find(pat)
    while i >= 0:
        out.append((i, i + len(pat)))
        i = s.find(pat, i + len(pat))
    return out


def cut(part: bytes, circular: bool, directional: bool, enzyme, trace: dict | None = None):
    """(status, [(Sequence, ForwardOverhang, ReverseOverhang), ...]) of CutWithEnzyme.  trace, if given,
    receives the overhangs, the branch taken, the number of forward/reverse ties and of pieces the len > 8
    filter dropped."""
    fsite, rsite, skip, ohl, recog = enzyme
    t = trace if trace is not None else {}
    t.update(branch="none", ties=0, short=0, overhangs=[], palindromic=is_palindromic(recog))
    if any(c >= 0x80 for c in part):  # strings.ToUpper would re-encode it: the library refuses such parts
        t["branch"] = "unsupported"
        return UNSUPPORTED, []
    sequence = (part + part if circular else part).upper()
    palindromic = t["palindromic"]
    forward = [(end + skip, True) for _, end in find_all(sequence, fsite)]
    reverse = [] if palindromic else [(start - skip, False) for start, _ in find_all(sequence, rsite)]
    overhangs = []
    for overhang_set in (forward, reverse):
        if overhang_set and not circular and overhang_set[-1][0] + skip + ohl > len(sequence):
            overhang_set = overhang_set[:-1]
        overhangs += overhang_set
    overhangs.sort(key=lambda o: o[0])  # stable, like sort.SliceStable
    t["overhangs"] = overhangs
    t["ties"] = sum(1 for a, b in zip(overhangs, overhangs[1:]) if a[0] == b[0] and a[1] != b[1])
    try:
        if len(overhangs) == 1 and not directional and not circular:
            P = overhangs[0][0]
            if forward:  # len(forwardOverhangs): the set as found, before the drop
                t["branch"] = "single_forward"
                f1, f2, o = go_slice(sequence, P + ohl), go_slice(sequence, 0, P), go_slice(sequence, P, P + ohl)
                return OK, [(f1, o, b""), (f2, b"", o)]
            t["branch"] = "single_reverse"
            f1, f2, o = go_slice(sequence, P), go_slice(sequence, 0, P - ohl), go_slice(sequence, P - ohl, P)
            return OK, [(f2, b"", o), (f1, o, b"")]
        if len(overhangs) == 2 and not directional and circular:
            t["branch"] = "circular_one"
            P = overhangs[0][0]
            s1, s2, o = go_slice(sequence, P + ohl, len(part)), go_slice(sequence, 0, P), go_slice(sequence, P, P + ohl)
            return OK, [(s1 + s2, o, o)]
        fragments = []
        if len(overhangs) > 1:
            t["branch"] = "pairwise_directional" if directional and not palindromic else "pairwise_all"
            pieces, rssl = [], len(recog) + skip
            for i in range(len(overhangs) - 1):
                cur, nxt = overhangs[i], overhangs[i + 1]
                if directional and not palindromic:
                    if cur[1] and not nxt[1]:
                        pieces.append(go_slice(sequence, cur[0], nxt[0]))
                else:
                    pieces.append(go_slice(sequence, cur[0], nxt[0]))
                if nxt[0] - rssl > len(part):
                    break
            for f in pieces:
                if len(f) > 8:
                    fragments.append((go_slice(f, ohl, len(f) - ohl), go_slice(f, 0, ohl), go_slice(f, len(f) - ohl, len(f))))
                else:
                    t["short"] += 1
        return OK, fragments
    except Panic:
        t["panic"] = True
        return PANIC, []


# ---- part generators -------------------------------------------------------------------------------------
_IUPAC = b"ACGTRYKMSWBDHVN"


def _letters(rng: random.Random, pool: bytes, n: int, mixed_case: bool = False) -> bytes:
    s = bytes(rng.choice(pool) for _ in range(n))
    return bytes(c + 32 if mixed_case and 65 <= c <= 90 and rng.random() < 0.3 else c for c in s)


def occurrences(part: bytes, circular: bool, site: bytes):
    """leftmost non-overlapping starts of site in ToUpper(part) (doubled when circular)"""
    return [s for s, _ in find_all((part + part if circular else part).upper(), site)]


def panel_library(n: int, seed: int):
    """(parts, circular, plants) in the style of clone_util.digest_library for the PANEL enzymes: both sites of
    each planted on disjoint stretches (at both ends, across the origin of circular parts), mixed case, Bpu10I's
    site with its N and with the N replaced (which must not match), lengths from 0 to 4 kbp, NUL and control
    bytes between plants, and a few parts with a byte >= 0x80.  plants[i] lists (position, site) in part i."""
    rng = random.Random(seed)
    sites = [s for e in PANEL.values() for s in (e[0], e[1])] + [b"CCTAAGC", b"GCTTAGG"]
    parts, circ, plants = [], [], []
    for _ in range(n):
        L = int(np.exp(rng.uniform(np.log(8), np.log(4000)))) if rng.random() > 0.05 else rng.randint(0, 8)
        s = bytearray(_letters(rng, b"ACGT", L))
        c = rng.random() < 0.4
        taken, here = [False] * L, []

        def plant(p, site):
            idx = [(p + j) % L for j in range(len(site))]
            if any(taken[x] for x in idx):
                return
            for j, x in enumerate(idx):
                s[x] = site[j]
                taken[x] = True
            here.append((p, site))

        for _ in range(rng.randint(0, 8)):
            site = rng.choice(sites)
            if len(site) > L:
                break
            where = rng.random()
            plant(0 if where < 0.15 else L - len(site) if where < 0.3 else rng.randint(0, L - len(site)), site)
        if c and L > 10 and rng.random() < 0.4:  # across the origin
            site = rng.choice(sites)
            if len(site) < L:
                plant(L - rng.randint(1, len(site) - 1), site)
        free = [x for x in range(L) if not taken[x]]
        if free and rng.random() < 0.3:  # a lower-case stretch
            a = rng.randrange(L)
            b = min(L, a + rng.randint(1, 300))
            s[a:b] = bytes(s[a:b]).lower()
        if free and rng.random() < 0.05:  # NUL and control bytes never match
            for x in rng.sample(free, min(len(free), 4)):
                s[x] = rng.choice([0, 1, 9, 10, 13, 31, 127])
        if free and rng.random() < 0.01:
            s[rng.choice(free)] = 0xC3
        parts.append(bytes(s))
        circ.append(c)
        plants.append(here)
    return parts, circ, plants


def sweep_sites(fl: int, rl: int, seed: int):
    """A forward and a reverse site of fl and rl bytes that match only where they are planted: neither first
    letter occurs anywhere else in either site, or in the filler sweep_parts uses."""
    rng = random.Random(seed)
    while True:
        f0, r0 = rng.sample(b"ACGT", 2)
        body = bytes(c for c in _IUPAC if c not in (f0, r0))
        fsite = bytes([f0]) + _letters(rng, body, fl - 1)
        rsite = bytes([r0]) + _letters(rng, body, rl - 1)
        if not is_palindromic(fsite):
            return fsite, rsite, body


def sweep_parts(fl: int, rl: int, seed: int):
    """(enzyme, parts, circular, starts) for the site-length sweep: starts[i] are the forward and reverse
    match starts expected in ToUpper(part i) (doubled when circular), as sets.  Covers
      - a forward and a reverse match starting at every offset 0..63 of the walk's 32-position steps, linear
        and circular, so each tail lands in the next step's halo;
      - a match ending exactly at the end of a linear part, and one cut short by a byte (no match);
      - parts of every length 0 .. max(fl, rl) + 1 made of a site's prefix and a filler byte;
      - on circular parts, each site across the origin at every split k = 1 .. len - 1."""
    rng = random.Random(seed)
    fsite, rsite, body = sweep_sites(fl, rl, seed)
    enzyme = (fsite, rsite, 1, 4, fsite)

    def fill(n):
        return _letters(rng, body, n, mixed_case=True)

    parts, circ, starts = [], [], []

    def add(p, c, f, r):
        parts.append(p)
        circ.append(c)
        starts.append((set(f), set(r)))

    for o in range(64):
        a, b = 64 + o, 128 + o  # the reverse site one 64-byte block later, at the same offset
        p = fill(a) + fsite + fill(b - a - fl) + rsite + fill(9 + o % 5)
        L = len(p)
        add(p, False, [a], [b])
        add(p, True, [a, a + L], [b, b + L])
    for site, other in ((fsite, False), (rsite, True)):
        pre = fill(40)
        at_end = pre + site
        short = pre + site[:-1]
        add(at_end, False, [] if other else [40], [40] if other else [])
        add(short, False, [], [])
        for k in range(1, len(site)):  # across the origin: site[:k] at the end, site[k:] at the start
            p = site[k:] + fill(30) + site[:k]
            hit = [len(p) - k]
            add(p, True, [] if other else hit, hit if other else [])
    for n in range(max(fl, rl) + 2):  # lengths around the site lengths
        for site, other in ((fsite, False), (rsite, True)):
            p = site[:n] + fill(max(0, n - len(site)))
            hit = [0] if n >= len(site) else []
            add(p, False, [] if other else hit, hit if other else [])
            hit_c = [0, n] if n >= len(site) else []
            add(p, True, [] if other else hit_c, hit_c if other else [])
    return enzyme, parts, circ, starts


SWEEP_LENGTHS = (1, 2, 3, 5, 8, 16, 31, 32)
SWEEP_PAIRS = [(m, m) for m in SWEEP_LENGTHS] + [(32, 1), (1, 32)]

# self-overlapping sites: A^m, (AT)^n, ABA-style overlaps; the runs that hold them are periodic in `unit`
PERIODIC = [(b"A", b"A"), (b"AAA", b"A"), (b"A" * 9, b"A"), (b"ATATAT", b"AT"), (b"AT" * 5, b"AT"), (b"GCGCG", b"GC"),
            (b"GCGCGCGCG", b"GC"), (b"AACAA", b"AAC"), (b"A" * 32, b"A")]
RUN_EXTRA = (31, 32, 33, 63, 64, 65)


def periodic_parts(seed: int):
    """[(enzyme, parts, circular)] for each self-overlapping site: runs of its period whose lengths are
    31, 32, 33, 63, 64 and 65 plus the site length, starting at several offsets of a step, then a lone copy of
    the site and a reverse site, so that the fragment after the run shows which match the greedy rule kept
    last.  Each site comes as a non-palindromic enzyme (both walks) and, where the site's own reverse
    complement equals it, as the palindromic enzyme it is."""
    rng = random.Random(seed)
    out = []
    for site, unit in PERIODIC:
        filler_pool = bytes(c for c in b"ACGT" if c not in site)
        rsite = _letters(rng, filler_pool, 6)
        enzymes = [(site, rsite, 1, 4, b"GGTCTC"), (site, site, 0, 2, b"GGTCTC")]
        if is_palindromic(site):
            enzymes.append((site, rsite, 2, 3, site))
        parts, circ = [], []
        for extra in RUN_EXTRA:
            for lead in (0, 1, 17, 31, 32):
                run = (unit * ((extra + len(site)) // len(unit) + 1))[: extra + len(site)]
                pre = _letters(rng, filler_pool, lead)
                p = pre + run + _letters(rng, filler_pool, 20) + site + _letters(rng, filler_pool, 15) + rsite + _letters(rng, filler_pool, 12)
                parts.append(p)
                circ.append(len(parts) % 3 == 0)
        out.append((site, enzymes, parts, circ))
    return out


def tie_parts(seed: int):
    """[(enzyme, parts, circular)]: forward site == reverse site, a non-palindromic recognition site and
    skip = -fl/2, so every match gives a forward and a reverse overhang at the same position."""
    rng = random.Random(seed)
    out = []
    for site in (b"GT", b"GGATCC"[:4] + b"AG", b"CAGCTGGT", b"ACCTGCAGGTTACAGTCCAGTTCACGTACGTA"[:32]):
        fl = len(site)
        enzyme = (site, site, -(fl // 2), 1 if fl == 2 else 2, b"GGTCTC")
        pool = bytes(c for c in b"ACGT" if c != site[0])
        parts, circ = [], []
        for k in (1, 2, 3):
            for c in (False, True):
                p = _letters(rng, pool, rng.randint(10, 40))
                for _ in range(k):
                    p += site + _letters(rng, pool, rng.randint(12, 50))
                parts.append(p)
                circ.append(c)
        out.append((enzyme, parts, circ))
    return out


SKIP_PART_LENGTHS = (64, 100)


def skip_ohl_enzymes():
    """BsaI's sites with every skip of {-2^31, -fl - 1, -fl, -1, 0, 1, L, 2^31 - 1} (L the part lengths of
    skip_ohl_parts) and every overhang length of {-1, 0, 1, 3, 5, half a fragment +- 1, 2^31 - 1}."""
    fl = 6
    skips = [I32_MIN, -fl - 1, -fl, -1, 0, 1, *SKIP_PART_LENGTHS, I32_MAX]
    ohls = [-1, 0, 1, 3, 5, 9, 10, 11, I32_MAX]  # the F..R pieces at skip 1 are 20 bytes: 10 +- 1
    return [(b"GGTCTC", b"GAGACC", s, o, b"GGTCTC") for s in skips for o in ohls]


def skip_ohl_parts(seed: int):
    """Parts of 64 and 100 bytes (and a few others) with one forward site, one reverse site, a site at each
    end, F..R pairs 20 bytes apart at skip 1, reverse before forward, and three sites: the single-cut linear
    branch both ways, the two-cut circular branch, the pairwise loop and the len > 8 filter."""
    rng = random.Random(seed)
    F, R = b"GGTCTC", b"GAGACC"

    def fill(n):
        while True:
            s = _letters(rng, b"ACGT", n)
            if F not in s and R not in s:
                return s

    parts, circ = [], []
    for L in SKIP_PART_LENGTHS:
        shapes = [fill(20) + F + fill(L - 26), fill(20) + R + fill(L - 26), F + fill(L - 6), fill(L - 6) + F, R + fill(L - 6),
                  fill(L - 6) + R, fill(10) + F + b"A" + fill(20) + b"A" + R + fill(L - 44), fill(8) + R + fill(20) + F + fill(L - 40),
                  fill(5) + F + fill(10) + F + fill(10) + R + fill(L - 43)]
        for p in shapes:
            assert len(p) == L
            for c in (False, True):
                parts.append(p)
                circ.append(c)
    parts += [b"", F, R, F + R, R + F]
    circ += [False, True, False, True, False]
    return parts, circ


def recognition_enzymes():
    """EcoRI's sites under recognition sites that test checks.IsPalindromic's corners: empty (palindromic),
    odd lengths whose middle is its own complement (S, W, N) or not, lower case (the table maps it), one that
    differs from the forward site, letters that complement to 0 (U, Z), and a lower-case forward site (never
    matches: the part is upper-cased, the pattern is not)."""
    F = b"GAATTC"
    recogs = [b"", b"GASTC", b"GAWTC", b"GANTC", b"GAATC", b"gaattc", b"GGTCTC", b"GAUTC", b"UA", b"ZZ", b"GAATTC"]
    out = [(F, F, -5, 4, r) for r in recogs]
    out += [(b"gaattc", F, -5, 4, b"GAATTC"), (F, b"gaattc", 1, 4, b"GGTCTC")]
    return out


def many_matches_parts(seed: int, L: int = 3_000_000):
    """Two circular parts of L bytes for a 1-byte site A: mostly A (millions of starts, few long pieces), and
    A every 10-20 bytes (hundreds of thousands of fragments)."""
    rng = np.random.default_rng(seed)
    mostly = rng.choice(np.frombuffer(b"AAAAAAAAAAAAAACG", np.uint8), L)
    spaced = rng.choice(np.frombuffer(b"CG", np.uint8), L)
    at = np.cumsum(rng.integers(10, 21, L // 10))
    spaced[at[at < L]] = ord("A")
    return [mostly.tobytes(), spaced.tobytes()], [True, True], (b"A", b"T", 2, 3, b"A")


# ---- ligation ---------------------------------------------------------------------------------------------
def ligation_reactions(n: int, seed: int):
    """clone_util.random_reaction, plus fragments with empty overhangs (overhang length 0), sequences seqhash
    rejects (X, J), lower case, and U / Z, which complement to NUL when a fragment is attached
    reverse-complemented."""
    rng = random.Random(seed)
    out = []
    for _ in range(n):
        frags = random_reaction(rng)
        ohs = sorted({x for f in frags for x in f[1:]})
        extra = rng.random()
        if extra < 0.15:
            frags.append((bytes(rng.choice(b"ACGT") for _ in range(rng.randint(0, 8))), b"", rng.choice(ohs + [b""])))
            frags.append((frags[0][0], rng.choice(ohs + [b""]), b""))
        elif extra < 0.3:
            frags.append((b"A" + bytes(rng.choice(b"XJ") for _ in range(rng.randint(1, 3))) + b"A", rng.choice(ohs), rng.choice(ohs)))
        elif extra < 0.4:
            f = frags[rng.randrange(len(frags))]
            frags.append((f[0].lower(), f[1], f[2].lower() if rng.random() < 0.5 else f[2]))
        elif extra < 0.55:
            frags.append((b"AC" + bytes(rng.choice(b"UZ") for _ in range(rng.randint(1, 3))), rng.choice(ohs), rng.choice(ohs)))
        rng.shuffle(frags)
        out.append(frags)
    # AATTAXXA is the first construct whose hash fails: it takes the key "", so AJJA's construct is dropped
    out.append([(b"AXXA", b"AATT", b"AATT"), (b"AJJA", b"AATT", b"AATT")])
    return out


def ligation_paths(fragments):
    """recurseLigate (clone.go:270-324) without hashing, counting the paths it takes: forward and
    reverse-complemented attaches, attaches refused because the seed's overhang is palindromic, closed and
    looping constructs, constructs an early return drops, and constructs whose seqhash fails (key "")."""
    n = dict(forward=0, reverse=0, palindrome_guard=0, clones=0, loops=0, dropped=0, empty_key=0)
    emitted = []

    def rec(seed, used):
        fwd_oh, seq, rev_oh = seed
        if fwd_oh == rev_oh:
            emitted.append([0, True, fwd_oh + seq])
            return
        start = len(emitted)
        used = list(used)
        for nseq, nfwd, nrev in fragments:
            new_seed, how = None, None
            if rev_oh == nfwd:
                new_seed, how = (fwd_oh, seq + rev_oh + nseq, nrev), "forward"
            if rev_oh == reverse_complement(nrev):  # the second test overrides the first
                if rev_oh != reverse_complement(rev_oh):
                    new_seed, how = (fwd_oh, seq + rev_oh + reverse_complement(nseq), reverse_complement(nfwd)), "reverse"
                else:
                    n["palindrome_guard"] += 1
            if new_seed is None:
                continue
            n[how] += 1
            for u in used:
                if u[0] == nseq:
                    for e in emitted[start:]:
                        e[1] = False
                    emitted.append([1, True, u[1] + u[0] + u[2]])
                    return
            used.append((nseq, nfwd, nrev))
            rec(new_seed, used)

    for f in fragments:
        rec((f[1], f[0], f[2]), [])
    for kind, kept, construct in emitted:
        n["clones" if kind == 0 else "loops"] += 1
        n["dropped"] += not kept
        n["empty_key"] += seqhash_oracle.seqhash_string(construct, "DNA", kind == 0, True) is None
    return n


# ---- Golden Gate libraries for other enzymes ----------------------------------------------------------------
def _distinct_overhangs(k: int, length: int, rng: random.Random):
    out = []
    while len(out) < k:
        o = _letters(rng, b"ACGT", length)
        if o == reverse_complement(o) or o in out or reverse_complement(o) in out:
            continue
        out.append(o)
    return out


def type_iis_library(enzyme, positions: int, variants: int, insert_len: int, backbone_len: int, seed: int):
    """clone_util.combinatorial_library for any non-palindromic enzyme with skip >= 0: a circular backbone
    carrying O[positions] -> O[0] and `variants` linear parts O[i] + insert + O[i+1] per position, each between
    the enzyme's two sites and nowhere else.  Returns (parts, variants ** positions)."""
    fsite, rsite, skip, ohl, _ = enzyme
    rng = random.Random(seed)
    O = _distinct_overhangs(positions + 1, ohl, rng)
    gap = b"A" * skip

    def body(n):
        while True:
            s = _letters(rng, b"ACGT", n)
            if all(x not in s for x in (fsite, rsite)):
                return s

    def two_sites(make):
        while True:
            p = make()
            d = p + p[: max(len(fsite), len(rsite)) - 1]  # sites across the origin too
            if len(find_all(d, fsite)) + len(find_all(d, rsite)) == 2:
                return p

    parts = [(two_sites(lambda: fsite + gap + O[positions] + body(backbone_len) + O[0] + gap + rsite + body(30)), True)]
    for i in range(positions):
        for _ in range(variants):
            parts.append((two_sites(lambda: body(12) + fsite + gap + O[i] + body(insert_len) + O[i + 1] + gap + rsite + body(12)), False))
    return parts, variants ** positions


def palindromic_library(enzyme, n_inserts: int, insert_len: int, seed: int):
    """A Golden Gate reaction for a palindromic enzyme that cuts inside its site (EcoRI-like): a circular
    backbone and linear inserts, each between two sites.  Every fragment's ForwardOverhang is the site's own
    overhang, but its ReverseOverhang is the OH bytes before the next cut (the reference's quirk), which end
    in the site's first byte; the bytes before each site come from a small set of palindromic and
    reverse-complementary pairs, and one insert is repeated, so that reverse-complemented attaches, closed
    clones, the palindrome guard and loops all occur."""
    fsite, _, skip, ohl, _ = enzyme
    assert ohl - (len(fsite) + skip) == 3 and fsite[0] == ord("G"), "written for a G^AATTC-like enzyme"
    rng = random.Random(seed)
    # ReverseOverhang = lead + G.  CAA+G and CTT+G are each other's reverse complement (so are CGA+G and
    # CTC+G); CAT+G and CCG+G are palindromic
    leads = [b"CAA", b"CTT", b"CAT", b"CGA", b"CTC", b"CCG"]

    def body(n):
        while True:
            s = _letters(rng, b"ACGT", n)
            if fsite not in s:
                return s

    def insert():
        return body(10) + rng.choice(leads) + fsite + body(insert_len) + rng.choice(leads) + fsite + body(10)

    parts = [(body(6) + rng.choice(leads) + fsite + body(300) + rng.choice(leads) + fsite + body(40), True)]
    inserts = [(insert(), False) for _ in range(n_inserts)]
    parts += inserts + [inserts[0]]
    rng.shuffle(parts)
    return parts
