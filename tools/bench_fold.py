#!/usr/bin/env python
"""Zuker fold throughput of pg_fold_zuker_batch on five workloads; prints one JSON line
(profiles/h100_fold_n1.json).

Workloads (seeded; the primers from synth.primers, the rest from a NumPy generator):
  primers  1 M x 25-nt DNA   (the hairpin screen over every primer a design proposes)
  oligos   100 k x 60-nt DNA (oligo pools)
  rna      20 k x 100-nt RNA
  long     1 k x 500-nt DNA
  max      4 x 1 024-nt DNA  (the longest supported item: one timed call, no warm-up of its own and no parity
           sample, as one such item takes minutes on the device and longer in the restatement)
Per workload: the median wall time of `--runs` calls after one warm-up call (each call ends in a device
synchronise, so the time includes the host-device copies) as items/s and V-loop candidate checks/s
(the count of (rightOfStart, leftOfEnd) candidates is computed from the shapes: sum over diagonals d >= 5
of (n - d)(d - 5)(d - 4) / 2 per item); parity (MFE bits, dot-bracket, status) of a sample against the
C restatement (tests/fold_oracle.c); and a CPU arm, that C restatement on 16 host threads over a slice
("C restatement, not Go").  The card's name and power limit are read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))  # fold_oracle: parity and the CPU arm only
from poly_b200 import _lib, fold, synth  # noqa: E402


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True,
                             timeout=30).stdout.strip().split(", ")
        return {"gpu": out[0], "power_limit_w": float(out[1]), "sm_clock_mhz": int(out[2]), "sm_clock_max_mhz": int(out[3])}
    except Exception as e:  # reported, not fatal
        return {"nvidia_smi_error": str(e)}


def checks_per_item(n: int) -> int:
    return sum((n - d) * (d - 5) * (d - 4) // 2 for d in range(5, n))


def workload(name, scale):
    rng = np.random.default_rng(20261016)
    if name == "primers":
        n, L, al = int(1_000_000 * scale), 25, None
        flat = synth.primers(n, L)
    else:
        n, L, al = {"oligos": (int(100_000 * scale), 60, b"ACGT"), "rna": (int(20_000 * scale), 100, b"ACGU"),
                    "long": (max(int(1_000 * scale), 1), 500, b"ACGT"), "max": (4, 1024, b"ACGT")}[name]
        flat = np.frombuffer(al, dtype=np.uint8)[rng.integers(0, 4, n * L)]
    return np.ascontiguousarray(flat, dtype=np.uint8), np.arange(n + 1, dtype=np.uint64) * np.uint64(L), n, L


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--scale", type=float, default=1.0, help="fraction of each workload's item count")
    ap.add_argument("--cpu-threads", type=int, default=16)
    ap.add_argument("--only", default="primers,oligos,rna,long,max")
    a = ap.parse_args()
    import fold_oracle

    _lib.check(_lib.lib().pg_init(0))
    out = {"bench": "fold_zuker", "temp_c": 37.0, **gpu_info(), "workloads": {}}
    slices = {"primers": 4096, "oligos": 512, "rna": 128, "long": 16, "max": 0}
    for name in a.only.split(","):
        flat, off, n, L = workload(name, a.scale)
        if L < 1024:
            fold.zuker_arrays(flat[: int(off[min(n, 64)])], off[: min(n, 64) + 1], 37.0)  # warm-up
        times = []
        for _ in range(a.runs if L < 1024 else 1):
            t0 = time.perf_counter()
            mfe, db, dbl, st = fold.zuker_arrays(flat, off, 37.0)
            times.append(time.perf_counter() - t0)
        t = statistics.median(times)
        # parity on a sample spread over the batch
        idx = np.linspace(0, n - 1, num=min(n, slices[name]), dtype=np.int64)
        seqs = [flat[int(off[i]): int(off[i + 1])].tobytes() for i in idx]
        t0 = time.perf_counter()
        w_mfe, w_db, w_st = fold_oracle.fold_batch(seqs, 37.0, threads=a.cpu_threads)
        t_cpu = time.perf_counter() - t0
        bad = 0
        for k, i in enumerate(idx):
            got = db[int(off[i]): int(off[i]) + int(dbl[i])].tobytes()
            if int(st[i]) != int(w_st[k]) or np.float64(mfe[i]).tobytes() != np.float64(w_mfe[k]).tobytes() or got != w_db[k]:
                bad += 1
        checks = checks_per_item(L) * n
        out["workloads"][name] = {
            "items": n, "length": L, "seconds_median": t, "seconds_all": times, "items_per_s": n / t, "v_candidate_checks_per_s": checks / t,
            "parity_sample": len(idx), "parity_mismatches": bad,
            "cpu_c_restatement_not_go": {"threads": a.cpu_threads, "items": len(idx), "seconds": t_cpu, "items_per_s": len(idx) / t_cpu if len(idx) else None},
        }
        print(name, json.dumps(out["workloads"][name]), file=sys.stderr, flush=True)
    print(json.dumps(out))
    if any(w["parity_mismatches"] for w in out["workloads"].values()):
        sys.exit(1)


if __name__ == "__main__":
    main()
