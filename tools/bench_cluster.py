#!/usr/bin/env python
"""Grouping a sketch set at the cfg3 shape: pg_mash_cluster_dev against the pair-list route; prints one JSON
line (profiles/h100_cluster_n1.json).

Workload: 100k x 10 kbp family reads (R = 100), k = 31, s = 2000, generated and sketched on the device, sketches
resident.  Threshold: the matching count for Distance <= 0.7.
  cluster:  pg_mash_cluster_dev -- labels and both counts stay on the device.
  pairs:    the route without it -- pg_mash_distance_sparse_dev (every related pair as an (i, j, same) triple),
            the triples copied to the host, and there a filter by the threshold and scipy's connected
            components over the links that remain (tests/cluster_oracle.py: cluster_pairs, one thread).
  dense:    for scale, pg_mash_distance_block_dev over all rows into a resident n x n buffer: the pass whose
            tiles the other two consume.
The three are timed alternately, `--runs` times each after `--warmup` rounds, medians reported.  Device legs are
timed with CUDA events, host legs with a host clock around work that ends in a synchronise.  Checked in the run:
both routes give identical labels and counts, and the labels are 1 000 groups of 100 (n / R groups of R)."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))  # cluster_oracle: the host half of the pair-list route
from poly_b200 import _lib, mash, synth  # noqa: E402


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True,
                             timeout=30).stdout.strip().split(", ")
        return {"gpu": out[0], "power_limit_w": float(out[1]), "sm_clock_mhz": int(out[2]), "sm_clock_max_mhz": int(out[3])}
    except Exception as e:  # reported, not fatal
        return {"gpu": torch.cuda.get_device_name(0), "nvidia_smi_error": str(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100_000)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--max-distance", type=float, default=0.7)
    args = ap.parse_args()
    import cluster_oracle

    n, RL, k, s, R = args.n, 10_000, 31, 2000, 100
    min_same = mash.min_same_for_distance(args.max_distance, s)
    L = _lib.lib()
    _lib.check(L.pg_init(0))
    dev = torch.device("cuda", 0)
    st = torch.cuda.current_stream(dev).cuda_stream
    reads = torch.empty(n * RL, dtype=torch.uint8, device=dev)
    _lib.check(L.pg_synth_reads_dev(reads.data_ptr(), 0, n, RL, synth.SEED_READS, 1, R, st))
    sk = torch.empty((n, s), dtype=torch.int32, device=dev)
    _lib.check(L.pg_mash_sketch_uniform_dev(reads.data_ptr(), n, RL, k, s, 0, sk.data_ptr(), s, None, st))
    torch.cuda.synchronize()
    del reads

    def events(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    labels = torch.empty(n, dtype=torch.int32, device=dev)
    counts = torch.zeros(2, dtype=torch.int64, device=dev)

    def cluster():
        return events(lambda: _lib.check(L.pg_mash_cluster_dev(sk.data_ptr(), n, s, min_same, labels.data_ptr(), counts.data_ptr(),
                                                               counts.data_ptr() + 8, st)))

    cap = 64 << 20
    pi, pj, ps = (torch.empty(cap, dtype=torch.int32, device=dev) for _ in range(3))
    cnt = torch.zeros(1, dtype=torch.int64, device=dev)

    def pairs():
        sparse_ms = events(lambda: _lib.check(L.pg_mash_distance_sparse_dev(sk.data_ptr(), n, s, 0, n, 1, pi.data_ptr(), pj.data_ptr(), ps.data_ptr(),
                                                                            cap, cnt.data_ptr(), st)))
        t0 = time.perf_counter()
        m = int(cnt.item())
        assert m <= cap, m
        h = [x[:m].cpu().numpy().view(np.uint32) for x in (pi, pj, ps)]  # .cpu() synchronises
        t1 = time.perf_counter()
        res = cluster_oracle.cluster_pairs(h[0], h[1], h[2], n, min_same)
        t2 = time.perf_counter()
        return sparse_ms, (t1 - t0) * 1e3, (t2 - t1) * 1e3, m, res

    same = torch.empty((n, n), dtype=torch.int32, device=dev)

    def dense():
        return events(lambda: _lib.check(L.pg_mash_distance_block_dev(sk.data_ptr(), n, s, 0, n, same.data_ptr(), None, st)))

    before = gpu_info()
    for _ in range(args.warmup):
        cluster()
        pairs()
        dense()
    cluster_ms, sparse_ms, copy_ms, host_ms, dense_ms = [], [], [], [], []
    m = res = None
    for _ in range(args.runs):
        cluster_ms.append(cluster())
        a, b, c, m, res = pairs()
        sparse_ms.append(a)
        copy_ms.append(b)
        host_ms.append(c)
        dense_ms.append(dense())
    got = labels.cpu().numpy().view(np.uint32)
    n_groups, n_links = (int(x) for x in counts.cpu())
    parity = bool(np.array_equal(got, res[0]) and (n_groups, n_links) == res[1:])
    sizes = np.bincount(got, minlength=n)
    families = bool(n_groups == n // R and (sizes[sizes > 0] == R).all() and np.array_equal(got, np.arange(n) // R * R))
    med = statistics.median
    pairs_total = med(sparse_ms) + med(copy_ms) + med(host_ms)
    line = {
        "metric": "mash_cluster", "workload": f"cfg3 {n} x {RL} bp family reads R={R}, k={k}, s={s}; Distance <= {args.max_distance} = min_same {min_same}",
        "cluster_ms": round(med(cluster_ms), 2), "pairs_route_ms": round(pairs_total, 2), "pairs_sparse_ms": round(med(sparse_ms), 2),
        "pairs_copy_ms": round(med(copy_ms), 2), "pairs_host_components_ms": round(med(host_ms), 2), "dense_ms": round(med(dense_ms), 2),
        "speedup_vs_pairs_route": round(pairs_total / med(cluster_ms), 2), "cluster_over_dense": round(med(cluster_ms) / med(dense_ms), 2),
        "triples": m, "triple_bytes": 12 * m, "label_bytes": 4 * n, "n_groups": n_groups, "n_links": n_links,
        "runs": args.runs, "warmup": args.warmup, "cluster_ms_all": [round(x, 2) for x in cluster_ms],
        "pairs_sparse_ms_all": [round(x, 2) for x in sparse_ms], "pairs_copy_ms_all": [round(x, 2) for x in copy_ms],
        "pairs_host_components_ms_all": [round(x, 2) for x in host_ms], "dense_ms_all": [round(x, 2) for x in dense_ms],
        "parity_labels_and_counts": parity, "groups_are_the_families": families, "host_threads": len(os.sched_getaffinity(0)),
        **before, "sm_clock_mhz_after": gpu_info().get("sm_clock_mhz"),
    }
    print(json.dumps(line))
    if not (parity and families):
        sys.exit(1)


if __name__ == "__main__":
    main()
