#!/usr/bin/env python
"""Growing the sketch index at the cfg3 shape; prints one JSON line (profiles/h100_index_add_n1.json).

Workload: 100k x 10 kbp family reads (R = 100), k = 31, s = 2000, sketched on the device.  References are the 90 k
reads with i % R < 0.9 R, queries the other 10 k.  Legs, timed alternately `--runs` times after a warm-up:
  (a) create:  pg_mash_index_create_dev over the 90 k references;
  (b) grow:    pg_mash_index_create_dev over the first 80 k, then ten pg_mash_index_add_dev calls of 1 k, each timed;
  (c) add10k:  pg_mash_index_create_dev over the first 80 k (untimed), then one pg_mash_index_add_dev of the last 10 k;
  (d) queries: top-10 pg_mash_index_query_dev and pg_mash_index_query_within_dev at Distance <= 0.7 for the 10 k
               queries, on the index (b) grew and on the index (a) created.
Medians are reported.  Parity: the grown index's answers equal the created index's for all 10 k queries, and its
radius lists equal the CPU oracle's on a sample of queries."""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))  # within_oracle: the parity check only
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_query import gpu_info  # noqa: E402
from poly_b200 import _lib, mash, synth  # noqa: E402


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100_000)
    ap.add_argument("--families", type=int, default=100)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--parity", type=int, default=32)
    ap.add_argument("--base", type=int, default=80_000, help="references of the index that legs (b) and (c) grow")
    ap.add_argument("--batches", type=int, default=10, help="adds of leg (b)")
    ap.add_argument("--max-distance", type=float, default=0.7)
    args = ap.parse_args()
    L = _lib.lib()
    _lib.check(L.pg_init(0))
    dev = torch.device("cuda", 0)
    st = torch.cuda.current_stream(dev).cuda_stream
    n, R, RL, k, s = args.n, args.families, 10_000, 31, 2000
    reads = torch.empty(n * RL, dtype=torch.uint8, device=dev)
    _lib.check(L.pg_synth_reads_dev(reads.data_ptr(), 0, n, RL, synth.SEED_READS, 1, R, st))
    sk = torch.empty((n, s), dtype=torch.int32, device=dev)
    _lib.check(L.pg_mash_sketch_uniform_dev(reads.data_ptr(), n, RL, k, s, 0, sk.data_ptr(), s, None, st))
    del reads
    is_ref = torch.arange(n, device=dev) % R < R - R // 10
    refs, queries = sk[is_ref].contiguous(), sk[~is_ref].contiguous()
    del sk
    nr, nq = refs.shape[0], queries.shape[0]
    base = args.base
    step = (nr - base) // args.batches
    cuts = [base + i * step for i in range(args.batches)] + [nr]
    min_same = mash.min_same_for_distance(args.max_distance, s)

    def create(rows):
        return mash.SketchIndex(rows)

    def grow():
        ix = create(refs[:base])
        ms = []
        for a, b in zip(cuts, cuts[1:]):
            ms.append(timed(lambda: ix.add(refs[a:b]))[1])
        return ix, ms

    def add_all():
        ix = create(refs[:base])
        return ix, timed(lambda: ix.add(refs[base:]))[1]

    cap = 4 << 20
    off = torch.empty(nq + 1, dtype=torch.int64, device=dev)
    lref = torch.empty(cap, dtype=torch.int32, device=dev)
    lsame = torch.empty(cap, dtype=torch.int32, device=dev)
    ldist = torch.empty(cap, dtype=torch.float64, device=dev)
    total = torch.zeros((), dtype=torch.int64, device=dev)
    top = 10
    kref = torch.empty((nq, top), dtype=torch.int32, device=dev)
    ksame = torch.empty((nq, top), dtype=torch.int32, device=dev)
    kdist = torch.empty((nq, top), dtype=torch.float64, device=dev)
    knh = torch.empty(nq, dtype=torch.int32, device=dev)

    def nearest(ix):
        _lib.check(L.pg_mash_index_query_dev(ix._h, queries.data_ptr(), nq, s, top, 1, kref.data_ptr(), ksame.data_ptr(), kdist.data_ptr(),
                                             knh.data_ptr(), st))

    def within(ix):
        _lib.check(L.pg_mash_index_query_within_dev(ix._h, queries.data_ptr(), nq, s, min_same, off.data_ptr(), lref.data_ptr(), lsame.data_ptr(),
                                                    ldist.data_ptr(), cap, total.data_ptr(), st))

    def answers():
        m = int(total.item())
        assert m <= cap, m
        return [x.cpu().numpy().copy() for x in (kref, ksame, kdist, knh, off)] + [x[:m].cpu().numpy().copy() for x in (lref, lsame, ldist)]

    # warm-up of every leg
    ix, _ = timed(lambda: create(refs))
    nearest(ix), within(ix)
    ix.close()
    for leg in (grow, add_all):
        g, _ = leg()
        nearest(g), within(g)
        g.close()
    create_ms, grow_total_ms, add1k_ms, add10k_ms = [], [], [], []
    q = {"nearest_fresh": [], "nearest_grown": [], "within_fresh": [], "within_grown": []}
    parity_fresh = True
    for _ in range(args.runs):
        fresh, t = timed(lambda: create(refs))
        create_ms.append(t)
        (grown, ms), t = timed(grow)
        grow_total_ms.append(t)
        add1k_ms.extend(ms)
        for name, ix in (("fresh", fresh), ("grown", grown)):
            q["nearest_" + name].append(timed(lambda: nearest(ix))[1])
            q["within_" + name].append(timed(lambda: within(ix))[1])
        nearest(fresh), within(fresh)
        want = answers()
        nearest(grown), within(grown)
        got = answers()
        parity_fresh &= all(a.tobytes() == b.tobytes() for a, b in zip(got, want))
        fresh.close()
        grown.close()
        (g10, t10), _ = timed(add_all)
        add10k_ms.append(t10)
        g10.close()
    import within_oracle

    sample = np.sort(np.random.default_rng(0).choice(nq, size=min(args.parity, nq), replace=False))
    h_refs = refs.cpu().numpy().view(np.uint32)
    w_off, w_ref, w_same, w_dist = within_oracle.within(h_refs, queries.cpu().numpy().view(np.uint32)[sample], min_same)
    g_off, g_ref, g_same, g_dist = got[4].view(np.uint64), got[5].view(np.uint32), got[6].view(np.uint32), got[7]
    rows = [np.arange(int(g_off[i]), int(g_off[i + 1])) for i in sample]
    sel = np.concatenate(rows) if rows else np.zeros(0, np.int64)
    s_off = np.zeros(len(sample) + 1, np.uint64)
    s_off[1:] = np.cumsum([len(r) for r in rows])
    parity_oracle = bool(s_off.tobytes() == w_off.tobytes() and g_ref[sel].tobytes() == w_ref.tobytes()
                         and g_same[sel].tobytes() == w_same.tobytes() and g_dist[sel].tobytes() == w_dist.tobytes())
    med = statistics.median
    line = {
        "metric": "index_add", "runs": args.runs, "parity": bool(parity_fresh and parity_oracle),
        "workload": f"cfg3 {n} x {RL} bp family reads R={R}, k={k}, s={s}; refs {nr} ({base} + {args.batches} adds of {step}, or + one add of {nr - base}), "
                    f"queries {nq}, top-{top} and Distance <= {args.max_distance} (min_same {min_same})",
        "create_ms": round(med(create_ms), 2), "add_1k_ms": round(med(add1k_ms), 2), "add_1k_ms_max": round(max(add1k_ms), 2),
        "add_1k_over_create": round(med(add1k_ms) / med(create_ms), 3),
        "create_80k_plus_10_adds_ms": round(med(grow_total_ms), 2), "add_10k_ms": round(med(add10k_ms), 2),
        "add_10k_over_create": round(med(add10k_ms) / med(create_ms), 3),
        **{k_ + "_ms": round(med(v), 2) for k_, v in q.items()},
        "create_ms_all": [round(x, 2) for x in create_ms], "add_1k_ms_all": [round(x, 2) for x in add1k_ms],
        "add_10k_ms_all": [round(x, 2) for x in add10k_ms],
        "parity_grown_vs_created_all_queries": bool(parity_fresh), "parity_vs_oracle": parity_oracle, "parity_queries": int(len(sample)),
        "within_hits": int(len(got[5])), **gpu_info(),
    }
    print(json.dumps(line))


if __name__ == "__main__":
    main()
