#!/usr/bin/env python
"""Canonical k-mers (PG_KMER_CANONICAL) against the forward mode on the same bytes: grouped sketches, the sketcher and
the screen add; prints one JSON line (profiles/h100_canonical_n1.json; --out also writes it to a file).

Workloads (those of bench_sketch_groups.py, bench_sketcher.py and bench_screen.py), seeded and generated on the device,
k = 21, s = 1000:
  assemblies: --genomes random genomes of --genome-len bp in --contigs contigs each, min_copies 1, one call;
  samples:    --samples read sets of --reads-per-sample 150 bp reads, 90 % from 3 own 1 Mbp genomes with 1 %
              substitutions, min_copies 2, one call;
  sketcher:   --big-reads 150 bp reads of a --big-genome-len genome (1 % substitutions) in --adds adds to one group,
              min_copies 2, then the row;
  screen_add: --big-reads reads, 90 % from the first 20 assemblies' genomes (1 % substitutions, half of them
              reverse-complemented), the add against the 1 000 assembly sketches of the same mode.
Each leg runs in both modes, alternating, --runs times after --warmup rounds (CUDA events around each call; the grouped
calls synchronise inside); medians and the canonical / forward ratio are reported, with the passes of each grouped call
(pg_launch_count: 2 launches of set-up and 3 per pass; a sketcher add is 3 + 4 per pass).  A separate pass under
torch.profiler splits each leg's kernel time into the walk kernels (groups_walk / screen_walk / the generic kernels)
and the rest.  Parity in the run: canonical rows of --oracle-groups assemblies and one sample, and the canonical screen
of a pool subset, against tests/canonical_oracle.py; the sketcher's canonical row against the one-shot call."""
import argparse
import ctypes as C
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from bench_cluster import gpu_info  # noqa: E402
from bench_sketch_groups import reads_from  # noqa: E402
from poly_b200 import _lib  # noqa: E402

K, S, READ_LEN = 21, 1000, 150
MODES = {"forward": 0, "canonical": _lib.PG_KMER_CANONICAL}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--genomes", type=int, default=1000)
    ap.add_argument("--genome-len", type=int, default=5_000_000)
    ap.add_argument("--contigs", type=int, default=100)
    ap.add_argument("--samples", type=int, default=96)
    ap.add_argument("--reads-per-sample", type=int, default=100_000)
    ap.add_argument("--big-reads", type=int, default=10_000_000)
    ap.add_argument("--big-genome-len", type=int, default=5_000_000)
    ap.add_argument("--adds", type=int, default=10)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--oracle-groups", type=int, default=2)
    ap.add_argument("--oracle-reads", type=int, default=50_000)
    ap.add_argument("--oracle-threads", type=int, default=16)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    L = _lib.lib()
    _lib.check(L.pg_init(0))
    dev = torch.device("cuda", 0)
    st = torch.cuda.current_stream(dev).cuda_stream
    before = gpu_info()
    g = torch.Generator(device=dev)
    g.manual_seed(20261018)
    acgt = torch.tensor(list(b"ACGT"), dtype=torch.uint8, device=dev)
    comp = torch.zeros(256, dtype=torch.uint8, device=dev)
    comp[acgt.long()] = torch.tensor(list(b"TGCA"), dtype=torch.uint8, device=dev)

    # assemblies
    G, GL, NC = args.genomes, args.genome_len, args.contigs
    genomes = acgt[torch.randint(0, 4, (G * GL,), generator=g, device=dev)]
    g_off = torch.arange(G + 1, dtype=torch.int64, device=dev) * GL
    cuts = torch.sort(torch.randint(1, GL, (G, NC - 1), generator=g, device=dev), dim=1).values
    rec = torch.cat([torch.zeros((G, 1), dtype=torch.int64, device=dev), cuts], dim=1) + g_off[:-1, None]
    c_off = torch.cat([rec.reshape(-1), g_off[-1:]]).contiguous()
    c_goff = (torch.arange(G + 1, dtype=torch.int64, device=dev) * NC).contiguous()
    # read sets
    Q, R = args.samples, args.reads_per_sample
    src = acgt[torch.randint(0, 4, (Q * 3 * 1_000_000,), generator=g, device=dev)]
    pool = reads_from(g, acgt, src, 1_000_000, Q * R, lambda i: (i // R) * 3 + torch.randint(0, 3, i.shape, generator=g, device=dev), dev)
    del src
    p_off = torch.arange(Q * R + 1, dtype=torch.int64, device=dev) * READ_LEN
    p_goff = torch.arange(Q + 1, dtype=torch.int64, device=dev) * R
    # the sketcher's read set
    NB = args.big_reads
    big_genome = acgt[torch.randint(0, 4, (args.big_genome_len,), generator=g, device=dev)]
    big = reads_from(g, acgt, big_genome, args.big_genome_len, NB, lambda i: torch.zeros_like(i), dev, random_share=0.0)
    del big_genome
    per_add = -(-NB // args.adds)
    add_off = torch.arange(per_add + 1, dtype=torch.int64, device=dev) * READ_LEN
    # the screen's pool: reads of the first 20 assemblies' genomes, half of them reverse-complemented
    spool = reads_from(g, acgt, genomes, GL, NB, lambda i: torch.randint(0, 20, i.shape, generator=g, device=dev), dev).view(NB, READ_LEN)
    flip = torch.rand(NB, generator=g, device=dev) < 0.5
    spool = torch.where(flip[:, None], comp[spool.flip(1).long()], spool).reshape(-1).contiguous()
    s_off = torch.arange(NB + 1, dtype=torch.int64, device=dev) * READ_LEN

    out = {m: {"a": (torch.empty((G, S), dtype=torch.int32, device=dev), torch.empty(G, dtype=torch.int32, device=dev)),
               "b": (torch.empty((Q, S), dtype=torch.int32, device=dev), torch.empty(Q, dtype=torch.int32, device=dev)),
               "c": (torch.empty((1, S), dtype=torch.int32, device=dev), torch.empty(1, dtype=torch.int32, device=dev))} for m in MODES}
    torch.cuda.synchronize()

    def events(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        n0 = L.pg_launch_count()
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), L.pg_launch_count() - n0

    def groups(bases, off, n, goff, ng, m, mode, key):
        rows, cnt = out[mode][key]
        return lambda: _lib.check(L.pg_mash_sketch_groups_flags_dev(bases.data_ptr(), off.data_ptr(), n, goff.data_ptr(), ng, K, S, m, MODES[mode],
                                                                    rows.data_ptr(), S, cnt.data_ptr(), st))

    def sketcher(mode):
        def run():
            h = C.c_void_p()
            _lib.check(L.pg_mash_sketcher_create_flags(1, K, S, 2, 64 * S, MODES[mode], C.byref(h)))
            goff = torch.tensor([0, per_add], dtype=torch.int64, device=dev)
            for i in range(args.adds):
                n = min(per_add, NB - i * per_add)
                goff[1] = n
                _lib.check(L.pg_mash_sketcher_add_dev(h, big[i * per_add * READ_LEN:].data_ptr(), add_off.data_ptr(), n, goff.data_ptr(), 0, 1, st))
            rows, cnt = out[mode]["c"]
            _lib.check(L.pg_mash_sketcher_rows_dev(h, 0, 1, rows.data_ptr(), S, cnt.data_ptr(), None, None, st))
            torch.cuda.synchronize()
            _lib.check(L.pg_mash_sketcher_free(h))
        return run

    screens = {}

    def screen_add(mode):
        def run():
            _lib.check(L.pg_mash_screen_add_dev(screens[mode], spool.data_ptr(), s_off.data_ptr(), NB, st))
        return run

    legs = {}  # leg-major: each leg runs in both modes back to back, and the assemblies (the screens' sketches) first
    for mode in MODES:
        legs[("assemblies", mode)] = groups(genomes, c_off, G * NC, c_goff, G, 1, mode, "a")
    for mode in MODES:
        legs[("samples", mode)] = groups(pool, p_off, Q * R, p_goff, Q, 2, mode, "b")
    for mode in MODES:
        legs[("sketcher", mode)] = sketcher(mode)
    for mode in MODES:
        legs[("screen_add", mode)] = screen_add(mode)
    t = {key: [] for key in legs}
    launches = {}
    for r in range(args.warmup + args.runs):
        for (leg, mode), fn in legs.items():
            if leg == "screen_add":
                if mode not in screens:  # each mode's screen of its own assembly sketches
                    h = C.c_void_p()
                    _lib.check(L.pg_mash_screen_create_flags_dev(out[mode]["a"][0].data_ptr(), G, S, K, 1, MODES[mode], st, C.byref(h)))
                    screens[mode] = h
                _lib.check(L.pg_mash_screen_reset(screens[mode]))
            ms, launches[(leg, mode)] = events(fn)
            if r >= args.warmup:
                t[(leg, mode)].append(ms)
    med = {key: statistics.median(v) for key, v in t.items()}
    passes = {f"{leg}_{mode}": (launches[(leg, mode)] - 2) // 3 for leg in ("assemblies", "samples") for mode in MODES}
    # a sketcher leg: per add 2 launches of set-up, 4 per pass and the merge, then one rows launch
    passes.update({f"sketcher_{mode}_per_add": round(((launches[("sketcher", mode)] - 1) / args.adds - 3) / 4, 2) for mode in MODES})

    # the screen's results: each source genome's containment and multiplicity in each mode
    res = {}
    for mode in MODES:
        sh = np.zeros(G, np.uint32)
        cont = np.zeros(G, np.float64)
        mult = np.zeros(G, np.uint64)
        _lib.check(L.pg_mash_screen_results(screens[mode], sh.ctypes.data, cont.ctypes.data, mult.ctypes.data))
        res[mode] = (cont, mult)

    # kernel-time split under the profiler, one call of each leg and mode
    split = {}
    from torch.profiler import ProfilerActivity, profile

    for key, fn in legs.items():
        if key[0] == "screen_add":
            _lib.check(L.pg_mash_screen_reset(screens[key[1]]))
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        walk = other = 0.0
        for ev in prof.key_averages():
            us = getattr(ev, "device_time_total", None)
            if us is None:
                us = ev.cuda_time_total
            if not us or ev.key.startswith("Memcpy") or ev.key.startswith("Memset"):
                continue
            if "walk_kernel" in ev.key or "generic_kernel" in ev.key:
                walk += us
            elif "kernel" in ev.key.lower() or "cub" in ev.key.lower() or "thrust" in ev.key.lower():
                other += us
        split[f"{key[0]}_{key[1]}"] = {"walk_ms": round(walk / 1e3, 3), "other_kernels_ms": round(other / 1e3, 3)}
    for h in screens.values():
        _lib.check(L.pg_mash_screen_free(h))

    # parity against the canonical restatement
    import canonical_oracle

    rng = np.random.default_rng(7)
    t0 = time.perf_counter()
    ok_oracle = True
    offs = c_off.cpu().numpy()
    ra, ca = (x.cpu().numpy().view(np.uint32) for x in out["canonical"]["a"])
    for i in sorted(rng.choice(G, args.oracle_groups, replace=False)):
        b = genomes[i * GL:(i + 1) * GL].cpu().numpy()
        o = (offs[i * NC:(i + 1) * NC + 1] - offs[i * NC]).astype(np.uint64)
        want = canonical_oracle.sketch_groups(b, o, [0, NC], K, S, 1, args.oracle_threads)
        ok_oracle &= want[0][0].tobytes() == ra[i].tobytes() and want[1][0] == ca[i]
    rb, cb = (x.cpu().numpy().view(np.uint32) for x in out["canonical"]["b"])
    q = int(rng.integers(0, Q))
    b = pool[q * R * READ_LEN:(q + 1) * R * READ_LEN].cpu().numpy()
    want = canonical_oracle.sketch_groups(b, np.arange(R + 1, dtype=np.uint64) * READ_LEN, [0, R], K, S, 2, args.oracle_threads)
    ok_oracle &= want[0][0].tobytes() == rb[q].tobytes() and want[1][0] == cb[q]
    nr = args.oracle_reads
    refs = np.concatenate([ra[:20], ra[rng.choice(np.arange(20, G), 30, replace=False)]])
    sub = spool[:nr * READ_LEN].cpu().numpy()
    sub_off = np.arange(nr + 1, dtype=np.uint64) * READ_LEN
    h = C.c_void_p()
    _lib.check(L.pg_mash_screen_create_flags(refs.ctypes.data, len(refs), S, K, 1, _lib.PG_KMER_CANONICAL, C.byref(h)))
    _lib.check(L.pg_mash_screen_add(h, sub.ctypes.data, sub_off.ctypes.data, nr))
    got = (np.zeros(len(refs), np.uint32), np.zeros(len(refs), np.float64), np.zeros(len(refs), np.uint64))
    _lib.check(L.pg_mash_screen_results(h, *(x.ctypes.data for x in got)))
    _lib.check(L.pg_mash_screen_free(h))
    want = canonical_oracle.mash_screen(refs, (sub, sub_off), K, args.oracle_threads)
    ok_oracle &= all(x.tobytes() == y.tobytes() for x, y in zip(got, want))
    oracle_s = time.perf_counter() - t0
    # the sketcher's canonical row against the one-shot canonical call over the same reads
    one = (torch.empty((1, S), dtype=torch.int32, device=dev), torch.empty(1, dtype=torch.int32, device=dev))
    b_off = torch.arange(NB + 1, dtype=torch.int64, device=dev) * READ_LEN
    _lib.check(L.pg_mash_sketch_groups_flags_dev(big.data_ptr(), b_off.data_ptr(), NB, torch.tensor([0, NB], dtype=torch.int64, device=dev).data_ptr(),
                                                 1, K, S, 2, _lib.PG_KMER_CANONICAL, one[0].data_ptr(), S, one[1].data_ptr(), st))
    sketcher_equal = bool(torch.equal(one[0], out["canonical"]["c"][0]) and torch.equal(one[1], out["canonical"]["c"][1]))

    src_cont = {m: float(res[m][0][:20].min()) for m in MODES}
    src_mult = {m: float(np.median(res[m][1][:20])) for m in MODES}
    ok = bool(ok_oracle and sketcher_equal and src_cont["canonical"] >= 0.99)
    line = {
        "metric": "mash_canonical",
        "shape": f"k={K}, s={S}; assemblies: {G} x {GL} bp in {NC} contigs, m=1; samples: {Q} x {R} x {READ_LEN} bp, m=2; sketcher: {NB} x "
                 f"{READ_LEN} bp reads of a {args.big_genome_len} bp genome in {args.adds} adds, m=2; screen_add: {NB} x {READ_LEN} bp reads "
                 f"(90% from 20 of the assemblies, half reverse-complemented) against the {G} assembly sketches of the same mode",
        "runs": args.runs, "warmup": args.warmup,
        **{f"{leg}_{mode}_ms": round(v, 3) for (leg, mode), v in med.items()},
        **{f"{leg}_canonical_over_forward": round(med[(leg, "canonical")] / med[(leg, "forward")], 3)
           for leg in ("assemblies", "samples", "sketcher", "screen_add")},
        "passes": passes, "kernel_split": split,
        "screen_sources_min_containment": src_cont, "screen_sources_median_multiplicity": src_mult,
        "all_ms": {f"{leg}_{mode}": [round(x, 3) for x in v] for (leg, mode), v in t.items()},
        "oracle_parity": bool(ok_oracle), "oracle_samples": f"{args.oracle_groups} assemblies, 1 sample, screen of {nr} reads x 50 references",
        "oracle_threads": args.oracle_threads, "oracle_s": round(oracle_s, 3), "sketcher_equals_one_shot": sketcher_equal, "ok": ok,
        **before, "sm_clock_mhz_after": gpu_info().get("sm_clock_mhz"),
    }
    print(json.dumps(line))
    if args.out:
        with open(args.out, "w") as f:
            f.write(json.dumps(line) + "\n")
    if not ok:
        sys.exit(1)


if __name__ == "__main__":
    main()
