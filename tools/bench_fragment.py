#!/usr/bin/env python
"""Throughput of poly's synthesis/fragment on the GPU; prints one JSON line (profiles/h100_fragment_n1.json).

Workloads (genes from synth.independent_reads, seeded):
  fragment       100 k x 1.5 kbp, Fragment(min 90, max 110) with the 48 overhangs of the reference's
                 TestFragmentWithOverhangs as excludes (a gene library cut for synthesis)
  with_overhangs the same genes through FragmentWithOverhangs with those 48 as includes
  long           10 k x 10 kbp, Fragment(min 200, max 300) with 20 excludes
  next           NextOverhangs over 100 k sets of 20 overhangs
Per workload: the median wall time of `--runs` calls after one warm-up call (each call ends in a device
synchronise, so the time includes the host-device copies) as items/s and bases/s (sets/s for `next`, whose
sets are flattened into the C ABI's arrays before the timed calls);
parity (status, ends, error numbers, float64 bytes) of a sample against the C restatement
(oracle/fragment_oracle.c); and that restatement on 16 host threads over the sample ("C restatement, not
Go").  The card's name, power limit and SM clock are read in the same run.  This is integer and FP64
latency-bound work: no share of a bandwidth or FLOP roof is claimed."""
import argparse
import json
import os
import random
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))  # fragment_oracle: parity and the CPU arm only
from poly_b200 import _lib, fragment, synth  # noqa: E402


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True,
                             timeout=30).stdout.strip().split(", ")
        return {"gpu": out[0], "power_limit_w": float(out[1]), "sm_clock_mhz": int(out[2]), "sm_clock_max_mhz": int(out[3])}
    except Exception as e:  # reported, not fatal
        return {"nvidia_smi_error": str(e)}


def timed(fn, runs):
    fn()  # warm-up
    times = []
    for _ in range(runs):
        t0 = time.perf_counter()
        out = fn()
        times.append(time.perf_counter() - t0)
    return out, times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--scale", type=float, default=1.0, help="fraction of each workload's item count")
    ap.add_argument("--sample", type=int, default=2000, help="items per parity sample")
    ap.add_argument("--cpu-threads", type=int, default=16)
    ap.add_argument("--only", default="fragment,with_overhangs,long,next")
    ap.add_argument("--out", default="", help="also write the JSON line to this file")
    a = ap.parse_args()
    import fragment_oracle as fo

    _lib.check(_lib.lib().pg_init(0))
    forty_eight = fo.pins()["TestFragmentWithOverhangs"]["include"]
    status_map = {fo.OK: fragment.ITEM_OK, fo.PANIC: fragment.ITEM_PANIC, fo.UNSUPPORTED: fragment.ITEM_UNSUPPORTED, fo.MIN_GT_MAX: fragment.ITEM_MIN_GT_MAX,
                  fo.MIN_LT_12: fragment.ITEM_MIN_LT_12, fo.NO_POSITION: fragment.ITEM_NO_POSITION}
    out = {"bench": "fragment", **gpu_info(), "workloads": {}}
    for name in a.only.split(","):
        if name == "next":
            n = int(100_000 * a.scale)
            rnd = random.Random(20261016)
            al = "ACGT"
            sets = [["".join(rnd.choice(al) for _ in range(4)) for _ in range(20)] for _ in range(n)]
            flat = np.frombuffer("".join(o for s in sets for o in s).encode(), dtype=np.uint8)
            off = np.arange(20 * n + 1, dtype=np.uint64) * np.uint64(4)
            soff = np.arange(n + 1, dtype=np.uint64) * np.uint64(20)
            (cands, nc, eff), times = timed(lambda: fragment.next_overhangs_flat(flat, off, soff), a.runs)
            idx = np.linspace(0, n - 1, num=min(n, a.sample), dtype=np.int64)
            t0 = time.perf_counter()
            w_c, w_n, w_e = fo.next_overhangs_batch([sets[i] for i in idx], threads=a.cpu_threads)
            t_cpu = time.perf_counter() - t0
            bad = sum(1 for k, i in enumerate(idx) if nc[i] != w_n[k] or cands[i, : nc[i]].tobytes() != w_c[k, : nc[i]].tobytes()
                      or eff[i, : nc[i]].tobytes() != w_e[k, : nc[i]].tobytes())
            t = statistics.median(times)
            out["workloads"][name] = {"sets": n, "set_size": 20, "seconds_median": t, "seconds_all": times, "sets_per_s": n / t,
                                      "parity_sample": len(idx), "parity_mismatches": bad,
                                      "cpu_c_restatement_not_go": {"threads": a.cpu_threads, "sets": len(idx), "seconds": t_cpu, "sets_per_s": len(idx) / t_cpu}}
        else:
            n, L, mn, mx = {"fragment": (100_000, 1500, 90, 110), "with_overhangs": (100_000, 1500, 90, 110), "long": (10_000, 10_000, 200, 300)}[name]
            n = max(int(n * a.scale), 1)
            flat = np.ascontiguousarray(synth.independent_reads(n, L), dtype=np.uint8)
            off = np.arange(n + 1, dtype=np.uint64) * np.uint64(L)
            ex, inc = {"fragment": (forty_eight, []), "with_overhangs": ([], forty_eight), "long": (forty_eight[:20], [])}[name]
            res, times = timed(lambda: fragment.fragment_arrays(flat, off, mn, mx, ex, inc), a.runs)
            st, eff, emin, emax, foff, ends = res
            idx = np.linspace(0, n - 1, num=min(n, a.sample), dtype=np.int64)
            seqs = [flat[int(off[i]): int(off[i + 1])].tobytes() for i in idx]
            t0 = time.perf_counter()
            w_st, w_eff, w_emin, w_emax, w_ends = fo.fragment_batch(seqs, mn, mx, ex, inc, threads=a.cpu_threads)
            t_cpu = time.perf_counter() - t0
            bad = 0
            for k, i in enumerate(idx):
                got = [int(x) for x in ends[int(foff[i]): int(foff[i + 1])]]
                if int(st[i]) != status_map[int(w_st[k])] or eff[i].tobytes() != w_eff[k].tobytes() or got != w_ends[k] \
                        or (int(emin[i]), int(emax[i])) != (int(w_emin[k]), int(w_emax[k])):
                    bad += 1
            t = statistics.median(times)
            out["workloads"][name] = {"items": n, "length": L, "min": mn, "max": mx, "n_exclude": len(ex), "n_include": len(inc),
                                      "seconds_median": t, "seconds_all": times, "items_per_s": n / t, "bases_per_s": n * L / t,
                                      "ok_items": int((st == fragment.ITEM_OK).sum()), "fragments": int(foff[-1]),
                                      "parity_sample": len(idx), "parity_mismatches": bad,
                                      "cpu_c_restatement_not_go": {"threads": a.cpu_threads, "items": len(idx), "seconds": t_cpu, "items_per_s": len(idx) / t_cpu}}
        print(name, json.dumps(out["workloads"][name]), file=sys.stderr, flush=True)
    out.update(gpu_info_after=gpu_info())
    print(json.dumps(out))
    if a.out:
        with open(a.out, "w") as f:
            f.write(json.dumps(out) + "\n")
    if any(w["parity_mismatches"] for w in out["workloads"].values()):
        sys.exit(1)


if __name__ == "__main__":
    main()
