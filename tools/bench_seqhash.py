#!/usr/bin/env python
"""Seqhash throughput of pg_seqhash_batch_dev on four workloads; prints one JSON line
(profiles/h100_seqhash_n1.json).

Workloads (input generated on the device by pg_synth_reads_dev, seeded; (d) from the test fixture):
  a  plasmid library:        1 M x 5 kbp, DNA, circular double-stranded
  b  cfg2 reads:             10 M x 150 bp, DNA, linear double-stranded (single-chunk path)
  c  bacterial chromosomes:  32 x 4 Mbp, DNA, circular double-stranded (BLAKE3 tree, long rotations)
  d  proteins:               tests/golden/fasta/uniprot_1mb_test_head.fasta.gz records replicated to >= 1 GB,
                             PROTEIN, linear single-stranded
Per workload: the median wall time of `--runs` calls (each ends in a device synchronise) as GB/s of input;
kernel times per stage from torch.profiler in a separate, untimed call; parity of a sample of sequences
against the C restatement (oracle/seqhash_oracle.c); and a CPU arm: that C restatement over all
schedulable cores on a prefix of the workload ("C restatement, not Go").  The card's name and power
limit are read in the same run."""
import argparse
import gzip
import json
import os
import re
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))  # seqhash_oracle: parity and the CPU arm only
from poly_b200 import _lib, fasta, seqhash, synth  # noqa: E402


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True,
                             timeout=30).stdout.strip().split(", ")
        return {"gpu": out[0], "power_limit_w": float(out[1]), "sm_clock_mhz": int(out[2]), "sm_clock_max_mhz": int(out[3])}
    except Exception as e:  # reported, not fatal
        return {"gpu": torch.cuda.get_device_name(0), "nvidia_smi_error": str(e)}


def uniform(n, L, dev, st):
    seqs = torch.empty(n * L, dtype=torch.uint8, device=dev)
    _lib.check(_lib.lib().pg_synth_reads_dev(seqs.data_ptr(), 0, n, L, synth.SEED_READS, 0, 0, st))
    return seqs, torch.arange(n + 1, dtype=torch.int64, device=dev) * L, L


def proteins(min_bytes, dev):
    text = gzip.open(os.path.join(ROOT, "tests", "golden", "fasta", "uniprot_1mb_test_head.fasta.gz")).read()
    seq, off, _, _, err = fasta.ingest(text, names=False)
    assert err is None
    reps = -(-min_bytes // len(seq))
    lens = np.diff(off.astype(np.int64))
    all_off = np.zeros(len(lens) * reps + 1, dtype=np.int64)
    np.cumsum(np.tile(lens, reps), out=all_off[1:])
    return torch.from_numpy(np.tile(seq, reps)).to(dev), torch.from_numpy(all_off).to(dev), int(lens.max())


def stage_times(fn):
    """Kernel time per kernel name (ms) over one call, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
        m = re.search(r"((?:seqhash|blake3)_\w+)(<[^>]*>)?", e.key)
        if t and m:
            out[m.group(0)] = round(out.get(m.group(0), 0) + t / 1e3, 3)
    return out


def run(name, seqs, off, max_len, t, circular, ds, runs, parity_n, cpu_bytes, threads, st):
    n = off.numel() - 1
    total = int(off[-1] - off[0])

    def call():
        return seqhash.hash_device(seqs, off, n, max_len, t, circular, ds, st)

    call()  # warm-up
    torch.cuda.synchronize()
    ms = []
    for _ in range(runs):
        t0 = time.perf_counter()
        dig, code, _ = call()
        torch.cuda.synchronize()
        ms.append((time.perf_counter() - t0) * 1e3)
    stages = stage_times(call)
    dig = dig.cpu().numpy()
    code = code.cpu().numpy()
    h_off = off.cpu().numpy().astype(np.uint64)
    rng = np.random.default_rng(0)
    sample = np.unique(np.concatenate([[0, n - 1], rng.choice(n, size=min(parity_n, n), replace=False)]))
    import seqhash_oracle

    ok = True
    for i in sample:
        s = seqs[int(h_off[i]): int(h_off[i + 1])].cpu().numpy().tobytes()
        c, d, _ = seqhash_oracle.seqhash(s, t, circular, ds)
        ok &= c == int(code[i]) and dig[i].tobytes() == (d or bytes(32))
    # CPU arm on a prefix of whole sequences
    m = max(1, min(n, int(np.searchsorted(h_off, cpu_bytes, side="right")) - 1))
    h_seqs = seqs[: int(h_off[m])].cpu().numpy()
    t0 = time.perf_counter()
    c_dig, c_code, _ = seqhash_oracle.seqhash_batch(h_seqs, h_off[: m + 1], t, circular, ds, threads)
    cpu_s = time.perf_counter() - t0
    cpu_ok = bool(np.array_equal(c_dig, dig[:m]) and np.array_equal(c_code, code[:m]))
    med = statistics.median(ms)
    return {
        "workload": name, "n": n, "input_bytes": total, "type": t, "circular": circular, "double_stranded": ds,
        "ms": round(med, 3), "ms_all": [round(x, 3) for x in ms], "gb_per_s": round(total / med / 1e6, 2),
        "kernel_ms": stages, "parity": bool(ok), "parity_sequences": int(len(sample)), "errors": int((code != 0).sum()),
        "cpu_arm": {"impl": "C restatement, not Go", "threads": threads, "sequences": m, "bytes": int(h_off[m]),
                    "s": round(cpu_s, 3), "gb_per_s": round(int(h_off[m]) / cpu_s / 1e9, 3), "matches_gpu": cpu_ok},
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--parity", type=int, default=32)
    ap.add_argument("--cpu-bytes", type=int, default=64 << 20, help="input bytes of each workload the CPU arm hashes")
    ap.add_argument("--scale", type=float, default=1.0, help="fraction of each workload's sequence count (rehearsal)")
    ap.add_argument("--only", default="abcd")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_seqhash needs a CUDA device")
    _lib.check(_lib.lib().pg_init(0))
    dev = torch.device("cuda", 0)
    st = torch.cuda.current_stream(dev).cuda_stream
    threads = len(os.sched_getaffinity(0))
    sc = lambda k: max(1, int(k * args.scale))  # noqa: E731
    rows = []
    for w in args.only:
        if w == "a":
            seqs, off, ml = uniform(sc(1_000_000), 5000, dev, st)
            rows.append(run("a plasmids 1M x 5 kbp", seqs, off, ml, "DNA", True, True, args.runs, args.parity, args.cpu_bytes, threads, st))
        elif w == "b":
            seqs, off, ml = uniform(sc(10_000_000), 150, dev, st)
            rows.append(run("b reads 10M x 150 bp", seqs, off, ml, "DNA", False, True, args.runs, args.parity, args.cpu_bytes, threads, st))
        elif w == "c":
            seqs, off, ml = uniform(sc(32), 4_000_000, dev, st)
            rows.append(run("c chromosomes 32 x 4 Mbp", seqs, off, ml, "DNA", True, True, args.runs, args.parity, args.cpu_bytes, threads, st))
        elif w == "d":
            seqs, off, ml = proteins(int((1 << 30) * args.scale), dev)
            rows.append(run("d uniprot records to >= 1 GB", seqs, off, ml, "PROTEIN", False, False, args.runs, args.parity, args.cpu_bytes,
                            threads, st))
        del seqs, off
        torch.cuda.empty_cache()
    print(json.dumps({"metric": "seqhash", "workloads": rows, "runs": args.runs, "host_threads": threads, **gpu_info()}))


if __name__ == "__main__":
    main()
