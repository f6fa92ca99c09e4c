#!/usr/bin/env python
"""A growing clustering at the cfg3 shape: pg_mash_clusterer_add_dev fed in batches, against one
pg_mash_cluster_dev over the whole set and against re-clustering the growing prefix after each batch (what a
caller without the clusterer does); prints one JSON line (profiles/h100_cluster_add_n1.json).

Workloads: those of tools/bench_derep.py (100k x 10 kbp reads, k = 31, s = 2000, generated and sketched on the
device, sketches resident; the matching count for Distance <= 0.7): families, chain, distinct.  The set is fed as
`--batches` adds of equal size to a fresh clusterer.
Legs, `--runs` times each after `--warmup` rounds, medians reported:
  adds:    every add of one sequence, timed alone with a host clock (an add ends in a device synchronise);
           per-add median and range over the runs, and the sequence's total.
  oneshot: pg_mash_cluster_dev over all n sketches, CUDA events.
  prefix:  pg_mash_cluster_dev over rows [0, end) after every batch, CUDA events, summed over the batches.
Checked in the run: the labels after the last add equal the one-shot call's, the group counts agree, and the
link counts of the adds add up to its count.  The one-shot time of the families workload is reported next to the
one recorded in profiles/h100_cluster_n1.json, which the shared link kernel must not exceed."""
import argparse
import ctypes as C
import json
import os
import statistics
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_cluster import gpu_info  # noqa: E402
from bench_derep import ROOT, S, sketch_workload  # noqa: E402
from poly_b200 import _lib, mash  # noqa: E402


def run_workload(L, kind, args, dev, st):
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

    one_label = torch.empty(n, dtype=torch.int32, device=dev)
    one_cnt = torch.zeros(2, dtype=torch.int64, device=dev)

    def oneshot(rows=n, label=one_label):
        return lambda: _lib.check(L.pg_mash_cluster_dev(sk.data_ptr(), rows, S, min_same, label.data_ptr(), one_cnt.data_ptr(),
                                                        one_cnt.data_ptr() + 8, st))

    add_label = torch.empty(n, dtype=torch.int32, device=dev)

    def adds():
        """ms of each add of one sequence, the summed links, each add's n_merged, and the final group count"""
        h = C.c_void_p()
        _lib.check(L.pg_mash_clusterer_create(S, min_same, C.byref(h)))
        ms, links, merged, groups = [], 0, [], 0
        try:
            for a, b in zip(edges[:-1], edges[1:]):
                first, ng, nl, nm = (C.c_uint64(0) for _ in range(4))
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                _lib.check(L.pg_mash_clusterer_add_dev(h, sk[a:].data_ptr(), b - a, S, None, C.byref(first), C.byref(ng), C.byref(nl),
                                                       C.byref(nm), st))
                ms.append((time.perf_counter() - t0) * 1e3)
                assert first.value == a
                links += nl.value
                merged.append(nm.value)
                groups = ng.value
            _lib.check(L.pg_mash_clusterer_labels_dev(h, 0, n, add_label.data_ptr(), st))
            torch.cuda.synchronize()
        finally:
            _lib.check(L.pg_mash_clusterer_free(h))
        return ms, links, merged, groups

    scratch = torch.empty(n, dtype=torch.int32, device=dev)

    def prefix():
        return sum(events(oneshot(b, scratch)) for b in edges[1:])

    for _ in range(args.warmup):
        adds()
        events(oneshot())
        prefix()
    t = {"add": [], "oneshot": [], "prefix": []}
    parity = True
    for _ in range(args.runs):
        ms, links, merged, groups = adds()
        t["add"].append(ms)
        t["oneshot"].append(events(oneshot()))
        parity = parity and bool(torch.equal(add_label, one_label)) and links == int(one_cnt[1]) and groups == int(one_cnt[0])
        t["prefix"].append(prefix())
    per_add = list(zip(*t["add"]))  # per add index, over the runs
    row = {
        "workload": kind, "min_same": min_same, "batches": nb, "batch_rows": n // nb, "n_groups": int(one_cnt[0]),
        "n_links": int(one_cnt[1]), "n_merged_per_add": merged,
        "add_median_ms": [round(statistics.median(x), 2) for x in per_add],
        "add_range_ms": [[round(min(x), 2), round(max(x), 2)] for x in per_add],
        "adds_total_ms": round(statistics.median(sum(r) for r in t["add"]), 2),
        "oneshot_ms": round(statistics.median(t["oneshot"]), 2),
        "prefix_recluster_total_ms": round(statistics.median(t["prefix"]), 2),
        "all_oneshot_ms": [round(x, 2) for x in t["oneshot"]], "parity": parity,
    }
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
    with open(os.path.join(ROOT, "profiles", "h100_cluster_n1.json")) as f:
        recorded = json.load(f)
    ok = all(r["parity"] for r in rows)
    line = {
        "metric": "mash_clusterer_add", "shape": f"cfg3 {args.n} x 10000 bp, k=31, s={S}; Distance <= {args.max_distance}; {args.batches} adds",
        "runs": args.runs, "warmup": args.warmup, "parity": ok, "workloads": rows,
        "recorded_oneshot_families_ms": recorded["cluster_ms"], "recorded_on": f"{recorded['gpu']} at {recorded['power_limit_w']:.0f} W",
        **before, "sm_clock_mhz_after": gpu_info().get("sm_clock_mhz"),
    }
    print(json.dumps(line))
    if not ok:
        sys.exit(1)


if __name__ == "__main__":
    main()
