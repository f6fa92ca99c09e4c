#!/usr/bin/env python
"""Grouped sketches (pg_mash_sketch_groups_dev): whole assemblies and whole read sets, one sketch per group; prints
one JSON line (profiles/h100_sketch_groups_n1.json; --out also writes it to a file).

Workloads, seeded and generated on the device:
  A, assemblies: --genomes random genomes of --genome-len bp, each cut into --contigs contigs at random points;
     k = 21, s = 1000, min_copies 1, one call.  For comparison, over the same bytes: pg_mash_sketch_batch_dev of the
     genomes as single records (the K2t path), and K1 (pg_mash_sketch_uniform_dev, 150 bp reads) over the first
     --k1-fraction of the bytes (K1's positional output of the whole set would not fit), reported as a rate.
  B, read sets: --samples samples x --reads-per-sample reads of 150 bp, sample q 90 % from its own 3 random 1 Mbp
     genomes with 1 % substitutions and 10 % random reads (the bench_screen_samples workload, one group per
     sample), and one sample of --big-reads reads at about 300x of a 5 Mbp genome with 1 % substitutions; k = 21,
     s = 1000, min_copies 2.  The screen add of the samples' bytes against workload A's sketches is timed for scale.
Legs: --runs times after --warmup rounds, one of each per round, medians reported (CUDA events around each call; the
grouped calls synchronise inside).  Passes come from pg_launch_count(): a call is 2 launches of set-up and 3 per pass.
The share of assemblies finished in pass 1 comes from sketching each genome alone (its own call), whose rows must equal
its row of the batched call.
Parity in the run: --oracle-groups assemblies and 2 samples against tests/sketch_groups_oracle.py, with its host time
on --oracle-threads threads."""
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
from poly_b200 import _lib  # noqa: E402

K, S, READ_LEN = 21, 1000, 150
SETUP_LAUNCHES, PASS_LAUNCHES = 2, 3


def reads_from(g, acgt, genomes, gl, n, sources, dev, random_share=0.1):
    """n reads of READ_LEN bp: a share from random bytes, the rest from genome sources(i) at random positions with
    1 % substitutions."""
    col = torch.arange(READ_LEN, dtype=torch.int64, device=dev)
    out = torch.empty(n * READ_LEN, dtype=torch.uint8, device=dev)
    step = 1 << 20
    for a in range(0, n, step):
        b = min(a + step, n)
        m = b - a
        gi = sources(torch.arange(a, b, device=dev))
        start = torch.randint(0, gl - READ_LEN + 1, (m,), generator=g, device=dev)
        copied = genomes[(gi * gl + start)[:, None] + col]
        sub = torch.rand((m, READ_LEN), generator=g, device=dev) < 0.01
        copied = torch.where(sub, acgt[torch.randint(0, 4, (m, READ_LEN), generator=g, device=dev)], copied)
        rnd = torch.rand(m, generator=g, device=dev) < random_share
        out[a * READ_LEN:b * READ_LEN] = torch.where(rnd[:, None], acgt[torch.randint(0, 4, (m, READ_LEN), generator=g, device=dev)], copied).reshape(-1)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--genomes", type=int, default=1000)
    ap.add_argument("--genome-len", type=int, default=5_000_000)
    ap.add_argument("--contigs", type=int, default=100)
    ap.add_argument("--k1-fraction", type=float, default=0.1)
    ap.add_argument("--samples", type=int, default=96)
    ap.add_argument("--reads-per-sample", type=int, default=100_000)
    ap.add_argument("--big-reads", type=int, default=10_000_000)
    ap.add_argument("--big-genome-len", type=int, default=5_000_000)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--oracle-groups", type=int, default=3)
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

    # A: assemblies
    G, GL, NC = args.genomes, args.genome_len, args.contigs
    genomes = acgt[torch.randint(0, 4, (G * GL,), generator=g, device=dev)]
    g_off = torch.arange(G + 1, dtype=torch.int64, device=dev) * GL
    cuts = torch.sort(torch.randint(1, GL, (G, NC - 1), generator=g, device=dev), dim=1).values
    rec = torch.cat([torch.zeros((G, 1), dtype=torch.int64, device=dev), cuts], dim=1) + g_off[:-1, None]
    c_off = torch.cat([rec.reshape(-1), g_off[-1:]]).contiguous()
    c_goff = (torch.arange(G + 1, dtype=torch.int64, device=dev) * NC).contiguous()
    rows_a = torch.empty((G, S), dtype=torch.int32, device=dev)
    cnt_a = torch.empty(G, dtype=torch.int32, device=dev)
    batch = torch.empty((G, S), dtype=torch.int32, device=dev)
    n_k1 = int(G * GL * args.k1_fraction) // READ_LEN
    k1_out = torch.empty((n_k1, READ_LEN - K), dtype=torch.int32, device=dev)

    # B: read sets
    Q, R = args.samples, args.reads_per_sample
    src_genomes = acgt[torch.randint(0, 4, (Q * 3 * 1_000_000,), generator=g, device=dev)]
    pool = reads_from(g, acgt, src_genomes, 1_000_000, Q * R, lambda i: (i // R) * 3 + torch.randint(0, 3, i.shape, generator=g, device=dev), dev)
    del src_genomes
    p_off = torch.arange(Q * R + 1, dtype=torch.int64, device=dev) * READ_LEN
    p_goff = torch.arange(Q + 1, dtype=torch.int64, device=dev) * R
    big_genome = acgt[torch.randint(0, 4, (args.big_genome_len,), generator=g, device=dev)]
    NB = args.big_reads
    big = reads_from(g, acgt, big_genome, args.big_genome_len, NB, lambda i: torch.zeros_like(i), dev, random_share=0.0)
    b_off = torch.arange(NB + 1, dtype=torch.int64, device=dev) * READ_LEN
    b_goff = torch.tensor([0, NB], dtype=torch.int64, device=dev)
    rows_b = torch.empty((Q, S), dtype=torch.int32, device=dev)
    cnt_b = torch.empty(Q, dtype=torch.int32, device=dev)
    rows_c = torch.empty((1, S), dtype=torch.int32, device=dev)
    cnt_c = torch.empty(1, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()

    def events(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        n0 = L.pg_launch_count()
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), L.pg_launch_count() - n0

    def groups(bases, off, n, goff, ng, m, rows, cnt):
        return lambda: _lib.check(L.pg_mash_sketch_groups_dev(bases.data_ptr(), off.data_ptr(), n, goff.data_ptr(), ng, K, S, m, rows.data_ptr(), S,
                                                              cnt.data_ptr(), st))

    legs = {
        "assemblies": groups(genomes, c_off, G * NC, c_goff, G, 1, rows_a, cnt_a),
        "assemblies_batch_k2t": lambda: _lib.check(L.pg_mash_sketch_batch_dev(genomes.data_ptr(), g_off.data_ptr(), G, GL, K, S, 0, batch.data_ptr(), S,
                                                                              None, None, st)),
        "k1_slice": lambda: _lib.check(L.pg_mash_sketch_uniform_dev(genomes.data_ptr(), n_k1, READ_LEN, K, S, 0, k1_out.data_ptr(), READ_LEN - K, None, st)),
        "samples": groups(pool, p_off, Q * R, p_goff, Q, 2, rows_b, cnt_b),
        "big_sample": groups(big, b_off, NB, b_goff, 1, 2, rows_c, cnt_c),
    }
    t = {key: [] for key in list(legs) + ["screen_add_samples"]}
    launches = {}
    h = C.c_void_p()
    for r in range(args.warmup + args.runs):
        ms = {}
        for key, fn in legs.items():
            ms[key], launches[key] = events(fn)
        if r == 0:  # the screen of workload A's group sketches, for the add over the samples' bytes
            _lib.check(L.pg_mash_screen_create_dev(rows_a.data_ptr(), G, S, K, st, C.byref(h)))
        _lib.check(L.pg_mash_screen_reset(h))
        ms["screen_add_samples"], _ = events(lambda: _lib.check(L.pg_mash_screen_add_dev(h, pool.data_ptr(), p_off.data_ptr(), Q * R, st)))
        if r >= args.warmup:
            for key, v in ms.items():
                t[key].append(v)
    _lib.check(L.pg_mash_screen_free(h))
    passes = {key: (launches[key] - SETUP_LAUNCHES) // PASS_LAUNCHES for key in ("assemblies", "samples", "big_sample")}

    # every genome alone: its passes, and its row against the batched call
    ra, ca = rows_a.cpu().numpy().view(np.uint32), cnt_a.cpu().numpy().view(np.uint32)
    one_rows = torch.empty((1, S), dtype=torch.int32, device=dev)
    one_cnt = torch.empty(1, dtype=torch.int32, device=dev)
    pass1, alone_equal = 0, True
    offs = c_off.cpu().numpy()
    for i in range(G):
        sub_off = c_off[i * NC:(i + 1) * NC + 1]
        _, n_l = events(groups(genomes, sub_off, NC, torch.tensor([0, NC], dtype=torch.int64, device=dev), 1, 1, one_rows, one_cnt))
        pass1 += (n_l - SETUP_LAUNCHES) // PASS_LAUNCHES == 1
        alone_equal &= one_rows.cpu().numpy().view(np.uint32).tobytes() == ra[i].tobytes() and int(one_cnt.item()) == int(ca[i])

    # parity against the restatement
    import sketch_groups_oracle

    rng = np.random.default_rng(7)
    t0 = time.perf_counter()
    oracle_ok = True
    for i in sorted(rng.choice(G, args.oracle_groups, replace=False)):
        b = genomes[i * GL:(i + 1) * GL].cpu().numpy()
        o = offs[i * NC:(i + 1) * NC + 1] - offs[i * NC]
        want = sketch_groups_oracle.sketch_groups(b, o.astype(np.uint64), [0, NC], K, S, 1, args.oracle_threads)
        oracle_ok &= want[0][0].tobytes() == ra[i].tobytes() and want[1][0] == ca[i]
    rb, cb = rows_b.cpu().numpy().view(np.uint32), cnt_b.cpu().numpy().view(np.uint32)
    for q in sorted(rng.choice(Q, 2, replace=False)):
        b = pool[q * R * READ_LEN:(q + 1) * R * READ_LEN].cpu().numpy()
        want = sketch_groups_oracle.sketch_groups(b, np.arange(R + 1, dtype=np.uint64) * READ_LEN, [0, R], K, S, 2, args.oracle_threads)
        oracle_ok &= want[0][0].tobytes() == rb[q].tobytes() and want[1][0] == cb[q]
    oracle_s = time.perf_counter() - t0
    ok = bool(oracle_ok and alone_equal and (ca == S).all() and (cb == S).all() and int(cnt_c.item()) == S)

    med = {key: statistics.median(v) for key, v in t.items()}
    a_bases, b_bases, c_bases = G * GL, Q * R * READ_LEN, NB * READ_LEN
    line = {
        "metric": "mash_sketch_groups",
        "shape": f"A: {G} genomes x {GL} bp in {NC} contigs each, k={K}, s={S}, m=1; B: {Q} samples x {R} x {READ_LEN} bp reads (90% from 3 own "
                 f"1 Mbp genomes, 1% substitutions) and one sample of {NB} x {READ_LEN} bp reads of a {args.big_genome_len} bp genome, m=2",
        "runs": args.runs, "warmup": args.warmup,
        **{f"{key}_ms": round(v, 3) for key, v in med.items()},
        "assemblies_gbases_per_s": round(a_bases / med["assemblies"] / 1e6, 1),
        "assemblies_batch_k2t_gbases_per_s": round(a_bases / med["assemblies_batch_k2t"] / 1e6, 1),
        "k1_slice_gbases_per_s": round(n_k1 * READ_LEN / med["k1_slice"] / 1e6, 1),
        "samples_gbases_per_s": round(b_bases / med["samples"] / 1e6, 1),
        "big_sample_gbases_per_s": round(c_bases / med["big_sample"] / 1e6, 1),
        "screen_add_samples_gbases_per_s": round(b_bases / med["screen_add_samples"] / 1e6, 1),
        "passes": passes, "assemblies_finished_in_pass_1": pass1 / G, "assemblies_alone_equal_batched": bool(alone_equal),
        "all_ms": {key: [round(x, 3) for x in v] for key, v in t.items()},
        "oracle_parity": bool(oracle_ok), "oracle_groups": f"{args.oracle_groups} assemblies + 2 samples", "oracle_threads": args.oracle_threads,
        "oracle_s": round(oracle_s, 3), "ok": ok,
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
