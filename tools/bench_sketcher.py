#!/usr/bin/env python
"""Grouped sketches grown in place (pg_mash_sketcher_add_dev) against the one-shot call (pg_mash_sketch_groups_dev);
prints one JSON line (profiles/h100_sketcher_n1.json; --out also writes it to a file).  k = 21, s = 1000.

Workloads, seeded and generated on the device (tools/bench_sketch_groups.py's generators):
  1. one read set: --big-reads x 150 bp reads at about 300x of a 5 Mbp genome, 1 % substitutions, m = 2: one one-shot
     call against --adds adds of equal parts.
  2. samples: --samples samples x --reads-per-sample reads (the one-shot bench's workload B), m = 2: --adds adds, each
     holding every sample's next share of reads, against one one-shot call.
  3. assemblies: --genomes genomes of --genome-len bp in --contigs contigs, m = 1: --adds adds of whole genomes, and
     --adds adds cut half a genome off the genome boundaries, against one one-shot call.
  4. beyond one call: a random --huge-genome-len bp genome on the device, read at --coverage x with 150 bp reads and
     --subs substitutions per base, generated add by add (--huge-add-reads reads each) and never stored whole; m = 2,
     the default budget (64 s).  Run at 1 % and at 10 % substitutions; an incomplete run is repeated with the budget
     4 times larger until it completes (at most --max-budget-steps times).  Reports the per-add median and the
     total, Gbases/s over the adds, held, complete, and the Mash distance to the genome's own one-shot sketch.
Times are CUDA events around each call (the adds synchronise inside).  Legs 1-3 take medians of --runs after --warmup:
of the one-shot call, and of each add over as many fresh sketchers fed the same adds; leg 4 runs once.  Passes come from pg_launch_count(): an add is 2 launches of set-up, 4 per pass and 1 to build the
new state; a one-shot call is 2 of set-up and 3 per pass.  Rows of complete groups must equal the one-shot rows."""
import argparse
import ctypes as C
import json
import os
import statistics
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_cluster import gpu_info  # noqa: E402
from bench_sketch_groups import reads_from  # noqa: E402
from poly_b200 import _lib, mash  # noqa: E402

K, S, READ_LEN = 21, 1000, 150


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--adds", type=int, default=10)
    ap.add_argument("--big-reads", type=int, default=10_000_000)
    ap.add_argument("--big-genome-len", type=int, default=5_000_000)
    ap.add_argument("--samples", type=int, default=96)
    ap.add_argument("--reads-per-sample", type=int, default=100_000)
    ap.add_argument("--genomes", type=int, default=1000)
    ap.add_argument("--genome-len", type=int, default=5_000_000)
    ap.add_argument("--contigs", type=int, default=100)
    ap.add_argument("--huge-genome-len", type=int, default=3_100_000_000)
    ap.add_argument("--coverage", type=float, default=30.0)
    ap.add_argument("--huge-add-reads", type=int, default=10_000_000)
    ap.add_argument("--subs", default="0.01,0.1")
    ap.add_argument("--max-budget-steps", type=int, default=2)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--skip-huge", action="store_true")
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

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        n0 = L.pg_launch_count()
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), L.pg_launch_count() - n0

    def one_shot(bases, off, n, goff, ng, m):
        rows = torch.empty((ng, S), dtype=torch.int32, device=dev)
        cnt = torch.empty(ng, dtype=torch.int32, device=dev)
        fn = lambda: _lib.check(L.pg_mash_sketch_groups_dev(bases.data_ptr(), off.data_ptr(), n, goff.data_ptr(), ng, K, S, m, rows.data_ptr(), S,
                                                            cnt.data_ptr(), st))
        ms = [timed(fn) for _ in range(args.warmup + args.runs)][args.warmup:]
        return statistics.median(x[0] for x in ms), (ms[0][1] - 2) // 3, rows.cpu().numpy().view(np.uint32), cnt.cpu().numpy().view(np.uint32)

    def run_adds(ng, m, adds, budget=None):
        """adds: (bases, off, n, goff, first, nb) on the device, or a callable making them.  Returns per-add ms,
        passes per add, and the rows (rows, count, complete, held)."""
        sk = mash.Sketcher(ng, K, S, m, budget)
        ms, passes = [], []
        for a in adds:
            bases, off, n, goff, first, nb = a() if callable(a) else a
            t, launches = timed(lambda: _lib.check(L.pg_mash_sketcher_add_dev(sk._h, bases.data_ptr(), off.data_ptr(), n, goff.data_ptr(), first, nb,
                                                                              st)))
            ms.append(t)
            passes.append(max(launches - 3, 0) // 4)
        rows = sk.rows()
        sk.close()
        return ms, passes, rows

    def repeat_adds(ng, m, adds):
        """run_adds --warmup + --runs times: the median of each add over the timed runs, and the last run's rows"""
        runs = [run_adds(ng, m, adds) for _ in range(args.warmup + args.runs)][args.warmup:]
        ms = [statistics.median(r[0][i] for r in runs) for i in range(len(adds))]
        return ms, runs[-1][1], runs[-1][2]

    def compare(rows, want_rows, want_cnt):
        r, c, complete, held = rows
        equal = all(r[i].tobytes() == want_rows[i].tobytes() and c[i] == want_cnt[i] for i in range(len(c)) if complete[i])
        prefix = all(r[i, :c[i]].tobytes() == want_rows[i, :c[i]].tobytes() for i in range(len(c)))
        return {"complete": float(complete.mean()), "complete_rows_equal": bool(equal), "prefix": bool(prefix), "held_max": int(held.max())}

    def add_summary(ms, passes):
        return {"add_ms_median": round(statistics.median(ms), 3), "total_ms": round(sum(ms), 3), "passes_per_add": passes,
                "add_ms": [round(x, 3) for x in ms]}

    line = {"metric": "mash_sketcher", "k": K, "s": S, "adds": args.adds, "runs": args.runs, "warmup": args.warmup}
    ok = True

    # 1. one read set
    NB = args.big_reads
    big_genome = acgt[torch.randint(0, 4, (args.big_genome_len,), generator=g, device=dev)]
    big = reads_from(g, acgt, big_genome, args.big_genome_len, NB, lambda i: torch.zeros_like(i), dev, random_share=0.0)
    b_off = torch.arange(NB + 1, dtype=torch.int64, device=dev) * READ_LEN
    one_ms, one_passes, want_r, want_c = one_shot(big, b_off, NB, torch.tensor([0, NB], dtype=torch.int64, device=dev), 1, 2)
    per = NB // args.adds
    adds = [(big, b_off[i * per:], per if i < args.adds - 1 else NB - i * per, torch.tensor([0, per if i < args.adds - 1 else NB - i * per],
             dtype=torch.int64, device=dev), 0, 1) for i in range(args.adds)]
    ms, passes, rows = repeat_adds(1, 2, adds)
    cmp1 = compare(rows, want_r, want_c)
    ok &= cmp1["complete"] == 1.0 and cmp1["complete_rows_equal"]
    line["read_set"] = {"shape": f"{NB} x {READ_LEN} bp reads of a {args.big_genome_len} bp genome, 1% substitutions, m=2",
                        "one_shot_ms": round(one_ms, 3), "one_shot_passes": one_passes, **add_summary(ms, passes), **cmp1}
    del big, b_off, adds

    # 2. samples, each add holding every sample's next share
    Q, R = args.samples, args.reads_per_sample
    src = acgt[torch.randint(0, 4, (Q * 3 * 1_000_000,), generator=g, device=dev)]
    pool = reads_from(g, acgt, src, 1_000_000, Q * R, lambda i: (i // R) * 3 + torch.randint(0, 3, i.shape, generator=g, device=dev), dev)
    del src
    p_off = torch.arange(Q * R + 1, dtype=torch.int64, device=dev) * READ_LEN
    one_ms, one_passes, want_r, want_c = one_shot(pool, p_off, Q * R, torch.arange(Q + 1, dtype=torch.int64, device=dev) * R, Q, 2)
    share = R // args.adds
    by_add = pool.view(Q, args.adds, share, READ_LEN).transpose(0, 1).contiguous()  # add i: every sample's share i
    a_off = torch.arange(Q * share + 1, dtype=torch.int64, device=dev) * READ_LEN
    a_goff = torch.arange(Q + 1, dtype=torch.int64, device=dev) * share
    adds = [(by_add[i].reshape(-1), a_off, Q * share, a_goff, 0, Q) for i in range(args.adds)]
    ms, passes, rows = repeat_adds(Q, 2, adds)
    cmp2 = compare(rows, want_r, want_c)
    ok &= cmp2["complete"] == 1.0 and cmp2["complete_rows_equal"]
    line["samples"] = {"shape": f"{Q} samples x {R} x {READ_LEN} bp reads, m=2, each add every sample's next {share}", "one_shot_ms": round(one_ms, 3),
                       "one_shot_passes": one_passes, **add_summary(ms, passes), **cmp2}
    del pool, by_add, adds

    # 3. assemblies
    G, GL, NC = args.genomes, args.genome_len, args.contigs
    genomes = acgt[torch.randint(0, 4, (G * GL,), generator=g, device=dev)]
    g_off = torch.arange(G + 1, dtype=torch.int64, device=dev) * GL
    cuts = torch.sort(torch.randint(1, GL, (G, NC - 1), generator=g, device=dev), dim=1).values
    rec = torch.cat([torch.zeros((G, 1), dtype=torch.int64, device=dev), cuts], dim=1) + g_off[:-1, None]
    c_off = torch.cat([rec.reshape(-1), g_off[-1:]]).contiguous()
    one_ms, one_passes, want_r, want_c = one_shot(genomes, c_off, G * NC, torch.arange(G + 1, dtype=torch.int64, device=dev) * NC, G, 1)
    res3 = {"shape": f"{G} genomes x {GL} bp in {NC} contigs, m=1", "one_shot_ms": round(one_ms, 3), "one_shot_passes": one_passes}
    for name, shift in (("whole_genomes", 0), ("cut_inside_genomes", NC // 2)):
        bounds = [0] + [i * G * NC // args.adds + shift for i in range(1, args.adds)] + [G * NC]
        adds = []
        for a, b in zip(bounds[:-1], bounds[1:]):
            first, last = a // NC, (b - 1) // NC
            goff = np.array([0] + [min(max(q * NC, a), b) - a for q in range(first + 1, last + 1)] + [b - a], np.int64)
            adds.append((genomes, c_off[a:], b - a, torch.from_numpy(goff).to(dev), first, last - first + 1))
        ms, passes, rows = repeat_adds(G, 1, adds)
        cmp3 = compare(rows, want_r, want_c)
        ok &= cmp3["complete"] == 1.0 and cmp3["complete_rows_equal"]
        res3[name] = {**add_summary(ms, passes), **cmp3}
    line["assemblies"] = res3
    del genomes, c_off, rec, cuts

    # 4. beyond one call
    if not args.skip_huge:
        HL = args.huge_genome_len
        huge = acgt[torch.randint(0, 4, (HL,), generator=g, device=dev)]
        h_rows = torch.empty((1, S), dtype=torch.int32, device=dev)
        h_cnt = torch.empty(1, dtype=torch.int32, device=dev)
        h_off = torch.tensor([0, HL], dtype=torch.int64, device=dev)
        h_goff = torch.tensor([0, 1], dtype=torch.int64, device=dev)
        _lib.check(L.pg_mash_sketch_groups_dev(huge.data_ptr(), h_off.data_ptr(), 1, h_goff.data_ptr(), 1, K, S, 1, h_rows.data_ptr(), S,
                                               h_cnt.data_ptr(), st))
        torch.cuda.synchronize()
        genome_count = int(h_cnt.item())
        genome_mash = mash.Mash(K, S)
        genome_mash.Sketches[:] = h_rows.cpu().numpy().view(np.uint32)[0]
        n_reads = int(HL * args.coverage) // READ_LEN
        per = args.huge_add_reads
        n_adds = (n_reads + per - 1) // per
        col = torch.arange(READ_LEN, dtype=torch.int64, device=dev)
        code = torch.zeros(256, dtype=torch.int64, device=dev)
        code[acgt.long()] = torch.arange(4, device=dev)
        bases = torch.empty(per * READ_LEN, dtype=torch.uint8, device=dev)
        r_off = torch.arange(per + 1, dtype=torch.int64, device=dev) * READ_LEN

        def make_add(i, sub, gen):
            def f():
                m_ = min(per, n_reads - i * per)
                step = 1 << 20
                for a in range(0, m_, step):
                    b = min(a + step, m_)
                    start = torch.randint(0, HL - READ_LEN + 1, (b - a,), generator=gen, device=dev)
                    r = huge[start[:, None] + col]
                    flip = torch.rand((b - a, READ_LEN), generator=gen, device=dev) < sub
                    alt = acgt[(code[r.long()] + torch.randint(1, 4, r.shape, generator=gen, device=dev)) % 4]  # another base
                    bases[a * READ_LEN:b * READ_LEN] = torch.where(flip, alt, r).reshape(-1)
                torch.cuda.synchronize()
                return bases, r_off, m_, torch.tensor([0, m_], dtype=torch.int64, device=dev), 0, 1
            return f

        huge_res = []
        for sub in (float(x) for x in args.subs.split(",")):
            budget = 64 * S
            for step in range(args.max_budget_steps + 1):
                gen = torch.Generator(device=dev)
                gen.manual_seed(int(sub * 1e6) + 7)
                ms, passes, (r, c, complete, held) = run_adds(1, 2, [make_add(i, sub, gen) for i in range(n_adds)], budget)
                m_ = mash.Mash(K, S)
                m_.Sketches[:] = r[0]
                huge_res.append({"subs": sub, "max_values": budget, "reads": n_reads, "gbases": round(n_reads * READ_LEN / 1e9, 2), "n_adds": n_adds,
                                 "add_ms_median": round(statistics.median(ms), 3), "total_ms": round(sum(ms), 1),
                                 "gbases_per_s": round(n_reads * READ_LEN / sum(ms) / 1e6, 1), "passes_per_add_median": statistics.median(passes),
                                 "passes_per_add_max": max(passes), "held": int(held[0]), "count": int(c[0]), "complete": bool(complete[0]),
                                 "distance_to_genome": round(float(m_.Distance(genome_mash)), 4)})
                print(json.dumps(huge_res[-1]), file=sys.stderr)
                if complete[0]:
                    break
                budget *= 4
        line["beyond_one_call"] = {"shape": f"a {HL} bp random genome, {args.coverage}x of {READ_LEN} bp reads in adds of {per}, m=2",
                                   "genome_sketch_count": genome_count, "runs": huge_res}
        ok &= genome_count == S
        del huge, bases

    line.update({"ok": bool(ok), **before, "sm_clock_mhz_after": gpu_info().get("sm_clock_mhz")})
    print(json.dumps(line))
    if args.out:
        with open(args.out, "w") as f:
            f.write(json.dumps(line) + "\n")
    if not ok:
        sys.exit(1)


if __name__ == "__main__":
    main()
