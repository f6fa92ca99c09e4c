#!/usr/bin/env python
"""A growing dereplication at the cfg3 shape: pg_mash_dereplicator_add_dev fed in batches, against one
pg_mash_dereplicate_dev over the whole set and against re-dereplicating the growing prefix after each batch (what
a caller without the dereplicator does); prints one JSON line (profiles/h100_derep_add_n1.json).

Workloads: those of tools/bench_derep.py (100k x 10 kbp reads, k = 31, s = 2000, generated and sketched on the
device, sketches resident; the matching count for Distance <= 0.7): families, chain, distinct.  The set is fed as
`--batches` adds of equal size to a fresh dereplicator.
Legs, `--runs` times each after `--warmup` rounds, medians reported:
  adds:    every add of one sequence, timed alone with a host clock (an add ends in a device synchronise);
           per-add median and range over the runs, and the sequence's total.
  oneshot: pg_mash_dereplicate_dev over all n sketches, CUDA events.
  prefix:  pg_mash_dereplicate_dev over rows [0, end) after every batch, CUDA events, summed over the batches.
Both modes run the adds and the one-shot call; the prefix leg runs in the first mode.  Checked in the run: the
concatenated assignments of every add sequence equal the one-shot call's, and the new-representative counts add
up to its count."""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_cluster import gpu_info  # noqa: E402
from bench_derep import S, sketch_workload  # noqa: E402
from poly_b200 import _lib, mash  # noqa: E402


def run_workload(L, kind, args, dev, st):
    import ctypes as C

    n, nb = args.n, args.batches
    min_same = mash.min_same_for_distance(args.max_distance, S)
    sk = sketch_workload(L, kind, n, dev, st)
    edges = [n * b // nb for b in range(nb + 1)]

    def events(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    one_rep = {f: torch.empty(n, dtype=torch.int32, device=dev) for f in (0, 1)}
    one_cnt = torch.zeros(2, dtype=torch.int64, device=dev)

    def oneshot(flags, rows=n, rep=None):
        out = one_rep[flags] if rep is None else rep
        return lambda: _lib.check(L.pg_mash_dereplicate_dev(sk.data_ptr(), rows, S, min_same, flags, out.data_ptr(),
                                                             one_cnt.data_ptr() + 8 * flags, st))

    add_rep = {f: torch.empty(n, dtype=torch.int32, device=dev) for f in (0, 1)}

    def adds(flags):
        """ms of each add of one sequence, and the total of the new representatives"""
        h = C.c_void_p()
        _lib.check(L.pg_mash_dereplicator_create(S, min_same, flags, C.byref(h)))
        ms, total = [], 0
        try:
            for a, b in zip(edges[:-1], edges[1:]):
                first, n_new = C.c_uint64(0), C.c_uint64(0)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                _lib.check(L.pg_mash_dereplicator_add_dev(h, sk[a:].data_ptr(), b - a, S, add_rep[flags][a:].data_ptr(), C.byref(first),
                                                          C.byref(n_new), st))
                ms.append((time.perf_counter() - t0) * 1e3)
                assert first.value == a
                total += n_new.value
        finally:
            _lib.check(L.pg_mash_dereplicator_free(h))
        return ms, total

    scratch = torch.empty(n, dtype=torch.int32, device=dev)

    def prefix():
        return sum(events(oneshot(0, b, scratch)) for b in edges[1:])

    for _ in range(args.warmup):
        for f in (0, 1):
            adds(f)
            events(oneshot(f))
        prefix()
    t = {"add_first": [], "add_nearest": [], "oneshot_first": [], "oneshot_nearest": [], "prefix_first": []}
    totals = {}
    parity = {}
    for _ in range(args.runs):
        for f, mode in ((0, "first"), (1, "nearest")):
            ms, totals[mode] = adds(f)
            t[f"add_{mode}"].append(ms)
            t[f"oneshot_{mode}"].append(events(oneshot(f)))
            parity[mode] = parity.get(mode, True) and bool(torch.equal(add_rep[f], one_rep[f])) and totals[mode] == int(one_cnt[f])
        t["prefix_first"].append(prefix())
    row = {"workload": kind, "min_same": min_same, "batches": nb, "batch_rows": n // nb}
    for mode in ("first", "nearest"):
        per_add = list(zip(*t[f"add_{mode}"]))  # per add index, over the runs
        row[f"n_reps_{mode}"] = totals[mode]
        row[f"add_{mode}_median_ms"] = [round(statistics.median(x), 2) for x in per_add]
        row[f"add_{mode}_range_ms"] = [[round(min(x), 2), round(max(x), 2)] for x in per_add]
        row[f"adds_total_{mode}_ms"] = round(statistics.median(sum(r) for r in t[f"add_{mode}"]), 2)
        row[f"oneshot_{mode}_ms"] = round(statistics.median(t[f"oneshot_{mode}"]), 2)
        row[f"parity_{mode}"] = parity[mode]
    row["prefix_rederep_total_first_ms"] = round(statistics.median(t["prefix_first"]), 2)
    row["all_oneshot_ms"] = {m: [round(x, 2) for x in t[f"oneshot_{m}"]] for m in ("first", "nearest")}
    del sk
    torch.cuda.empty_cache()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100_000)
    ap.add_argument("--batches", type=int, default=10)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--max-distance", type=float, default=0.7)
    ap.add_argument("--workloads", default="families,chain,distinct")
    args = ap.parse_args()
    L = _lib.lib()
    _lib.check(L.pg_init(0))
    dev = torch.device("cuda", 0)
    st = torch.cuda.current_stream(dev).cuda_stream
    before = gpu_info()
    rows = [run_workload(L, kind, args, dev, st) for kind in args.workloads.split(",")]
    ok = all(r["parity_first"] and r["parity_nearest"] for r in rows)
    line = {
        "metric": "mash_dereplicator_add", "shape": f"cfg3 {args.n} x 10000 bp, k=31, s={S}; Distance <= {args.max_distance}; "
                                                   f"{args.batches} adds",
        "runs": args.runs, "warmup": args.warmup, "parity": ok, "workloads": rows, **before,
        "sm_clock_mhz_after": gpu_info().get("sm_clock_mhz"),
    }
    print(json.dumps(line))
    if not ok:
        sys.exit(1)


if __name__ == "__main__":
    main()
