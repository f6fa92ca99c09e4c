#!/usr/bin/env python
"""Representatives of a sketch set at the cfg3 shape: pg_mash_dereplicate_dev against the pair-list route and
pg_mash_cluster_dev; prints one JSON line (profiles/h100_derep_n1.json).

Workloads: 100k x 10 kbp reads, k = 31, s = 2000, generated and sketched on the device, sketches resident;
threshold: the matching count for Distance <= 0.7.
  families: family reads (R = 100), as in bench_cluster.py: few representatives, most rows never read.
  chain:    10 kbp windows of one synthetic genome at a 5 kbp step: neighbours share half their k-mers and link,
            nothing else does, so every other window is a representative.  The walk's worst practical case.
  distinct: independent reads: nothing links, every sketch is a representative and the mark pass reads the
            whole upper triangle once.
Legs, alternating, `--runs` times each after `--warmup` rounds, medians reported:
  first / nearest: pg_mash_dereplicate_dev in both modes -- assignments and count stay on the device.
  cluster:         pg_mash_cluster_dev on the same sketches, for scale.
  pairs:           the route without it -- pg_mash_distance_sparse_dev (every related pair as an (i, j, same)
                   triple), the triples copied to the host, and there the greedy loop of
                   tests/derep_oracle.py (dereplicate_pairs, one thread), timed per mode.
Device legs are timed with CUDA events, host legs with a host clock around work that ends in a synchronise.
Checked in the run: both routes give identical assignments and counts in both modes.  A separate profiled pass
(one call per mode, after the timed legs) splits the device call into its kernels."""
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
sys.path.insert(0, os.path.join(ROOT, "tests"))  # derep_oracle: the host half of the pair-list route
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_cluster import gpu_info  # noqa: E402
from poly_b200 import _lib, mash, synth  # noqa: E402

RL, K, S, STEP = 10_000, 31, 2000, 5_000


def sketch_workload(L, kind, n, dev, st):
    """[n, S] int32 sketches of the workload on the device."""
    if kind == "chain":  # one genome, windows [STEP i, STEP i + RL)
        genome = torch.empty((n - 1) * STEP + RL, dtype=torch.uint8, device=dev)
        _lib.check(L.pg_synth_reads_dev(genome.data_ptr(), 0, 1, genome.numel(), synth.SEED_READS + 1, 0, 1, st))
        reads = genome.as_strided((n, RL), (STEP, 1)).contiguous()
        del genome
    else:
        reads = torch.empty(n * RL, dtype=torch.uint8, device=dev)
        _lib.check(L.pg_synth_reads_dev(reads.data_ptr(), 0, n, RL, synth.SEED_READS, 1 if kind == "families" else 0, 100, st))
    sk = torch.empty((n, S), dtype=torch.int32, device=dev)
    _lib.check(L.pg_mash_sketch_uniform_dev(reads.data_ptr(), n, RL, K, S, 0, sk.data_ptr(), S, None, st))
    torch.cuda.synchronize()
    return sk


def kernel_split(fn):
    """ms of device time per kernel class over one fn() under torch.profiler."""
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    split = {}
    for ev in prof.key_averages():
        name = ev.key
        dt = getattr(ev, "device_time_total", None)
        if dt is None:
            dt = ev.cuda_time_total
        if dt <= 0:
            continue
        if name.startswith("derep_") or "derep_" in name:
            cls = next(c for c in ("links", "walk", "mark", "finish") if f"derep_{c}" in name)
        elif "emset" in name:
            cls = "memsets"
        elif "emcpy" in name:
            cls = "copies"
        else:
            cls = "join"  # the distance plan and the dense tiles
        split[cls] = split.get(cls, 0.0) + dt / 1e3
    return {k: round(v, 3) for k, v in sorted(split.items())}


def run_workload(L, kind, args, dev, st):
    import derep_oracle

    n = args.n
    min_same = mash.min_same_for_distance(args.max_distance, S)
    sk = sketch_workload(L, kind, n, dev, st)

    def events(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    rep = {f: torch.empty(n, dtype=torch.int32, device=dev) for f in (0, 1)}
    cnt = torch.zeros(2, dtype=torch.int64, device=dev)

    def derep(flags):
        return lambda: _lib.check(L.pg_mash_dereplicate_dev(sk.data_ptr(), n, S, min_same, flags, rep[flags].data_ptr(),
                                                             cnt.data_ptr() + 8 * flags, st))

    labels = torch.empty(n, dtype=torch.int32, device=dev)
    ccnt = torch.zeros(2, dtype=torch.int64, device=dev)

    def cluster():
        _lib.check(L.pg_mash_cluster_dev(sk.data_ptr(), n, S, min_same, labels.data_ptr(), ccnt.data_ptr(), ccnt.data_ptr() + 8, st))

    cap = 64 << 20
    pi, pj, ps = (torch.empty(cap, dtype=torch.int32, device=dev) for _ in range(3))
    pcnt = torch.zeros(1, dtype=torch.int64, device=dev)

    def pairs():
        sparse_ms = events(lambda: _lib.check(L.pg_mash_distance_sparse_dev(sk.data_ptr(), n, S, 0, n, 1, pi.data_ptr(), pj.data_ptr(),
                                                                            ps.data_ptr(), cap, pcnt.data_ptr(), st)))
        t0 = time.perf_counter()
        m = int(pcnt.item())
        assert m <= cap, m
        h = [x[:m].cpu().numpy().view(np.uint32) for x in (pi, pj, ps)]  # .cpu() synchronises
        t1 = time.perf_counter()
        res, host_ms = [], []
        for nearest in (False, True):
            t = time.perf_counter()
            res.append(derep_oracle.dereplicate_pairs(h[0], h[1], h[2], n, min_same, nearest))
            host_ms.append((time.perf_counter() - t) * 1e3)
        return sparse_ms, (t1 - t0) * 1e3, host_ms, m, res

    for _ in range(args.warmup):
        events(derep(0))
        events(derep(1))
        events(cluster)
        pairs()
    t = {k: [] for k in ("first", "nearest", "cluster", "sparse", "copy", "host_first", "host_nearest")}
    m = res = None
    for _ in range(args.runs):
        t["first"].append(events(derep(0)))
        t["nearest"].append(events(derep(1)))
        t["cluster"].append(events(cluster))
        a, b, c, m, res = pairs()
        t["sparse"].append(a)
        t["copy"].append(b)
        t["host_first"].append(c[0])
        t["host_nearest"].append(c[1])
    got = [rep[f].cpu().numpy().view(np.uint32) for f in (0, 1)]
    n_reps = [int(x) for x in cnt.cpu()]
    parity = [bool(np.array_equal(got[f], res[f][0]) and n_reps[f] == res[f][1]) for f in (0, 1)]
    same_reps = bool(np.array_equal(got[0] == np.arange(n), got[1] == np.arange(n)))
    med = {k: statistics.median(v) for k, v in t.items()}
    route = {mode: med["sparse"] + med["copy"] + med[f"host_{mode}"] for mode in ("first", "nearest")}
    split = {mode: kernel_split(derep(f)) for f, mode in ((0, "first"), (1, "nearest"))}
    del sk, pi, pj, ps
    torch.cuda.empty_cache()
    return {
        "workload": kind, "min_same": min_same, "n_reps": n_reps[0], "n_groups_cluster": int(ccnt[0]), "triples": m,
        "derep_first_ms": round(med["first"], 2), "derep_nearest_ms": round(med["nearest"], 2), "cluster_ms": round(med["cluster"], 2),
        "pairs_route_first_ms": round(route["first"], 2), "pairs_route_nearest_ms": round(route["nearest"], 2),
        "pairs_sparse_ms": round(med["sparse"], 2), "pairs_copy_ms": round(med["copy"], 2),
        "pairs_host_first_ms": round(med["host_first"], 2), "pairs_host_nearest_ms": round(med["host_nearest"], 2),
        "speedup_vs_pairs_route_first": round(route["first"] / med["first"], 2),
        "speedup_vs_pairs_route_nearest": round(route["nearest"] / med["nearest"], 2),
        "all_ms": {k: [round(x, 2) for x in v] for k, v in t.items()},
        "kernels_ms_first": split["first"], "kernels_ms_nearest": split["nearest"],
        "parity_first": parity[0], "parity_nearest": parity[1], "modes_share_representatives": same_reps,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100_000)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--max-distance", type=float, default=0.7)
    ap.add_argument("--workloads", default="families,chain,distinct")
    args = ap.parse_args()
    L = _lib.lib()
    _lib.check(L.pg_init(0))
    dev = torch.device("cuda", 0)
    st = torch.cuda.current_stream(dev).cuda_stream
    before = gpu_info()
    rows = [run_workload(L, kind, args, dev, st) for kind in args.workloads.split(",")]
    ok = all(r["parity_first"] and r["parity_nearest"] and r["modes_share_representatives"] for r in rows)
    line = {
        "metric": "mash_dereplicate", "shape": f"cfg3 {args.n} x {RL} bp, k={K}, s={S}; Distance <= {args.max_distance}",
        "runs": args.runs, "warmup": args.warmup, "host_threads": len(os.sched_getaffinity(0)), "parity": ok,
        "workloads": rows, **before, "sm_clock_mhz_after": gpu_info().get("sm_clock_mhz"),
    }
    print(json.dumps(line))
    if not ok:
        sys.exit(1)


if __name__ == "__main__":
    main()
