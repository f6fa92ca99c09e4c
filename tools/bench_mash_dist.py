#!/usr/bin/env python
"""Mash distance between grouped sketches (pg_mash_dist_dev, pg_mash_dist_within_dev); prints one JSON line
(profiles/h100_mash_dist_n1.json; --out also writes it to a file).

Workload, seeded and generated on the device: --species random genomes of --genome-len bp, each the root of a family of
--strains genomes (the root itself, then strains at substitution rates spread evenly over 0.5 .. 5 %), sketched one group
per genome by pg_mash_sketch_groups_dev with k = 21, s = 1 000.  200 kbp genomes keep 32-bit chance collisions between
species rare (about s G / 2^32 = 0.05 shared values per pair) and generation cheap.
Legs, --runs times after --warmup rounds, CUDA-event medians, all outputs kept on the device:
  (a) the first 1 000 sketches against themselves, dense, all four outputs;
  (b) every sketch against every sketch (10 000 x 10 000 = 10^8 pairs by default), dense, all four outputs;
  (c) the triangle of (b) filtered at distance <= --max-distance (pg_mash_dist_within_dev, PG_PAIRS_UPPER).
For scale: pg_mash_distance_block_dev over the same rows (the reference's Similarity / Distance: a different answer),
and the plain restatement (tests/mash_dist_oracle.py) over a slice of --oracle-pairs pairs on one host thread.
Merge steps per pair are min(a + b, 2 s) from the shapes: the items of the merged rows the kernel walks.
Checked in the run: --sample pairs of (b) against the restatement, (c) against (b) filtered on the device, and the
distance of each root to its strains against -ln(1 - rate) within five binomial spreads of J."""
import argparse
import json
import math
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)
from bench_cluster import gpu_info  # noqa: E402
from poly_b200 import _lib, mash  # noqa: E402

K, S = 21, 1000


def make_sketches(args, dev):
    """rows [n, S] int32, count [n] int32 and rates [n] (0 for a root), one species at a time on the device"""
    g = torch.Generator(device=dev)
    g.manual_seed(args.seed)
    acgt = torch.tensor(list(b"ACGT"), dtype=torch.uint8, device=dev)
    P, T, GL = args.species, args.strains, args.genome_len
    rates = [0.0] + list(np.linspace(0.005, 0.05, T - 1))
    rows = torch.empty((P * T, S), dtype=torch.int32, device=dev)
    count = torch.empty(P * T, dtype=torch.int32, device=dev)
    off = torch.arange(T + 1, dtype=torch.int64, device=dev) * GL
    goff = torch.arange(T + 1, dtype=torch.int64, device=dev)
    for p in range(P):
        root = torch.randint(0, 4, (GL,), generator=g, device=dev, dtype=torch.int64)
        prob = torch.tensor(rates, device=dev, dtype=torch.float32)[:, None]
        sub = torch.rand((T, GL), generator=g, device=dev) < prob
        shift = torch.randint(1, 4, (T, GL), generator=g, device=dev, dtype=torch.int64)
        genomes = acgt[torch.where(sub, (root + shift) % 4, root)].contiguous()
        r, c = mash.sketch_groups(genomes.view(-1), off, goff, K, S)
        rows[p * T:(p + 1) * T], count[p * T:(p + 1) * T] = r, c
    torch.cuda.synchronize()
    return rows, count, np.array(rates * P)


def events(fn, runs, warmup):
    for _ in range(warmup):
        fn()
    times = []
    for _ in range(runs):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return statistics.median(times), min(times), max(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--species", type=int, default=100)
    ap.add_argument("--strains", type=int, default=100, help="genomes per species, the root included")
    ap.add_argument("--genome-len", type=int, default=200_000)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--max-distance", type=float, default=0.05)
    ap.add_argument("--sample", type=int, default=2000)
    ap.add_argument("--oracle-pairs", type=int, default=2000)
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--out")
    args = ap.parse_args()
    import mash_dist_oracle as oracle

    L = _lib.lib()
    _lib.check(L.pg_init(0))
    dev = torch.device("cuda:0")
    st = torch.cuda.current_stream(dev).cuda_stream
    info = gpu_info()
    t0 = time.time()
    rows, count, rates = make_sketches(args, dev)
    n = rows.shape[0]
    gen_s = time.time() - t0
    lens = torch.full((n,), args.genome_len, dtype=torch.int64, device=dev)
    assert int(count.min()) == S, "every genome fills its sketch"

    def dense(m):
        out = (torch.empty((m, m), dtype=torch.int32, device=dev), torch.empty((m, m), dtype=torch.int32, device=dev),
               torch.empty((m, m), dtype=torch.float64, device=dev), torch.empty((m, m), dtype=torch.float64, device=dev))

        def run():
            _lib.check(L.pg_mash_dist_dev(rows.data_ptr(), count.data_ptr(), m, rows.data_ptr(), count.data_ptr(), m, S, S, K, lens.data_ptr(),
                                          lens.data_ptr(), *[o.data_ptr() for o in out], st))
        return out, run

    na = min(1000, n)
    _, run_a = dense(na)
    leg_a = events(run_a, args.runs, args.warmup)
    out_b, run_b = dense(n)
    leg_b = events(run_b, args.runs, args.warmup)
    c_b, d_b, dist_b, p_b = out_b

    cap = 1 << 24
    lists = [torch.empty(cap, dtype=dt, device=dev) for dt in (torch.int32, torch.int32, torch.int32, torch.int32, torch.float64, torch.float64)]
    d_n = torch.zeros(1, dtype=torch.int64, device=dev)

    def run_c():
        _lib.check(L.pg_mash_dist_within_dev(rows.data_ptr(), count.data_ptr(), n, rows.data_ptr(), count.data_ptr(), n, S, S, K, lens.data_ptr(),
                                             lens.data_ptr(), args.max_distance, 1.0, _lib.PG_PAIRS_UPPER, *[t.data_ptr() for t in lists], cap,
                                             d_n.data_ptr(), st))
    leg_c = events(run_c, args.runs, args.warmup)
    n_pairs = int(d_n.item())

    same = torch.empty((n, n), dtype=torch.int32, device=dev)
    distr = torch.empty((n, n), dtype=torch.float64, device=dev)
    leg_ref = events(lambda: _lib.check(L.pg_mash_distance_block_dev(rows.data_ptr(), n, S, 0, n, same.data_ptr(), distr.data_ptr(), st)),
                     args.runs, args.warmup)
    del same, distr

    # parity: sampled pairs of (b) against the restatement
    rng = np.random.default_rng(args.seed)
    hrows = rows.cpu().numpy().view(np.uint32)
    hcount = count.cpu().numpy().view(np.uint32)
    qi, ri = rng.integers(0, n, args.sample), rng.integers(0, n, args.sample)
    qi[: args.sample // 4] = ri[: args.sample // 4] // args.strains * args.strains  # roots against members of any family
    ri[: args.sample // 8] = qi[: args.sample // 8] + rng.integers(0, args.strains, args.sample // 8)  # some within one family
    ri = np.minimum(ri, n - 1)
    got = [t[torch.from_numpy(qi).to(dev), torch.from_numpy(ri).to(dev)].cpu().numpy() for t in out_b]
    parity = True
    for x in range(args.sample):
        c, d = oracle.compare(hrows[qi[x], : hcount[qi[x]]].tolist(), hrows[ri[x], : hcount[ri[x]]].tolist(), S)
        wd = oracle.distance(c, d, K)
        wp = oracle.p_value(c, d, K, args.genome_len, args.genome_len)
        ok = (got[0][x] == c and got[1][x] == d and abs(got[2][x] - wd) <= 2 * np.spacing(wd) and
              (abs(got[3][x] - wp) <= 1e-9 * wp if wp >= 1e-290 else got[3][x] <= 1e-280))
        parity &= bool(ok)
    # (c) against (b) filtered on the device
    iu = torch.triu(torch.ones((n, n), dtype=torch.bool, device=dev), 1) & (dist_b <= args.max_distance)
    want_n = int(iu.sum())
    key = lambda q, r: q.to(torch.int64) * n + r.to(torch.int64)
    within_ok = want_n == n_pairs and n_pairs <= cap
    if within_ok:
        wq, wr = torch.nonzero(iu, as_tuple=True)
        within_ok = torch.equal(torch.sort(key(lists[0][:n_pairs], lists[1][:n_pairs]))[0], torch.sort(key(wq, wr))[0])
    del iu
    # distance of each root to its strains against -ln(1 - rate)
    dev_max, dev_sum, tracks = 0.0, 0.0, True
    T = args.strains
    roots = np.arange(0, n, T)
    droot = dist_b[torch.from_numpy(roots).to(dev)].cpu().numpy()
    for sp, rt in enumerate(roots):
        for t in range(1, T):
            rate = rates[rt + t]
            a = (1 - rate) ** K
            j = a / (2 - a)
            bound = 5 * math.sqrt(j * (1 - j) / S) / (K * j * (1 + j))
            e = abs(droot[sp, rt + t] + math.log(1 - rate))
            dev_max, dev_sum = max(dev_max, e / bound), dev_sum + e
            tracks &= e <= bound
    chance = c_b.view(n // T, T, n // T, T)
    between = float(chance.sum(dim=(1, 3)).to(torch.float64).sum() - chance.diagonal(dim1=0, dim2=2).sum().to(torch.float64))
    between_pairs = n * n - (n // T) * T * T

    # the restatement over a slice, on one host thread
    m = int(math.isqrt(args.oracle_pairs))
    t0 = time.perf_counter()
    for x in range(m):
        for y in range(m):
            c, d = oracle.compare(hrows[x, : hcount[x]].tolist(), hrows[y, : hcount[y]].tolist(), S)
            oracle.distance(c, d, K)
            oracle.p_value(c, d, K, args.genome_len, args.genome_len)
    oracle_s = time.perf_counter() - t0

    steps = lambda m_: float(np.minimum(hcount[:m_, None].astype(np.int64) + hcount[None, :m_], 2 * S).mean())
    rec = {
        "tool": "tools/bench_mash_dist.py", **info,
        "shape": f"{args.species} species x {args.strains} genomes of {args.genome_len} bp (root + strains at 0.5-5% substitutions), k={K}, s={S}",
        "generate_and_sketch_s": round(gen_s, 2),
        "a_dense_1k": {"pairs": na * na, "ms_median": round(leg_a[0], 3), "ms_min_max": [round(leg_a[1], 3), round(leg_a[2], 3)],
                       "pairs_per_s": na * na / leg_a[0] * 1e3, "merge_steps_per_pair": steps(na)},
        "b_dense": {"pairs": n * n, "ms_median": round(leg_b[0], 3), "ms_min_max": [round(leg_b[1], 3), round(leg_b[2], 3)],
                    "pairs_per_s": n * n / leg_b[0] * 1e3, "merge_steps_per_pair": steps(n),
                    "merge_steps_per_s": n * n * steps(n) / leg_b[0] * 1e3, "output_bytes": n * n * 24,
                    "output_GB_per_s": n * n * 24 / leg_b[0] / 1e6},
        "c_triangle_within": {"max_distance": args.max_distance, "pairs_listed": n_pairs, "ms_median": round(leg_c[0], 3),
                              "ms_min_max": [round(leg_c[1], 3), round(leg_c[2], 3)], "pairs_per_s": n * n / leg_c[0] * 1e3},
        "reference_distance_block_ms_median": round(leg_ref[0], 3),
        "oracle_host_pairs": m * m, "oracle_host_s": round(oracle_s, 3), "oracle_pairs_per_s": m * m / oracle_s,
        "parity_sample": args.sample, "parity": bool(parity), "within_equals_filtered_dense": bool(within_ok),
        "root_to_strain_tracks_rate": bool(tracks), "root_to_strain_mean_abs_error": dev_sum / (len(roots) * (T - 1)),
        "root_to_strain_max_error_over_bound": dev_max,
        "between_species_mean_common": between / between_pairs,
        "sm_clock_after_mhz": gpu_info().get("sm_clock_mhz"),
    }
    line = json.dumps(rec)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    assert parity and within_ok and tracks, "checks failed"


if __name__ == "__main__":
    main()
