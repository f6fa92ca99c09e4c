#!/usr/bin/env python
"""Pair-list alignment scores (pg_sw_score_pairs_dev / pg_nw_score_pairs_dev) on five workloads; prints
one JSON line per workload (profiles/h100_align_pairs_n1.json).

Workloads (inputs generated from seeds; scoring +3 / -3, gap -2 over {-, A, C, G, T}):
  P1  short pairs:        1 M pairs of 150 x 150, family reads (kind 1), each read against the next
                          read of its family; Smith-Waterman and Needleman-Wunsch
  P2  ragged targets:     100 k pairs of a 150 bp read against a target drawn from 1-10 kbp
  P3  index hits:         cfg3-shaped family reads (10 kbp, k = 31, s = 2000); SketchIndex over 9 000
                          references, top-4 for 1 000 queries -> 4 000 pairs of 10 kbp x 10 kbp; only the
                          pair score call is timed
  P4  one long pair:      20 kbp x 20 kbp through the pair kernels and through pg_sw_score_batch_dev with
                          n = 1 (one thread per query), timed alternately
  P5  one template:       10 k queries of 500 bp against one 10 kbp template through both entry points
                          (reported only)
Per workload: cells = sum of len(a) * len(b), the median wall time of `--runs` calls after warm-up (each
ends in a device synchronise) and GCUPS; parity of a sample against the C restatement (oracle/, driven pair by pair
by oracle/pair_oracle.c); and a CPU arm: that C driver on all schedulable cores over a P1 / P3 sample
("C restatement, not Go").
The card's name, power limit and SM clock are read in the same run."""
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
sys.path.insert(0, os.path.join(ROOT, "tests"))  # pair_oracle: parity and the CPU arm only
import pair_oracle  # noqa: E402
from poly_b200 import _lib, align, mash, synth  # noqa: E402

MAT = np.array([[0, 0, 0, 0, 0], [0, 3, -3, -3, -3], [0, -3, 3, -3, -3], [0, -3, -3, 3, -3], [0, -3, -3, -3, 3]], np.int64)
ALPHA = align.NewAlphabet(["-", "A", "C", "G", "T"])
SC = align.NewScoring(align.NewSubstitutionMatrix(ALPHA, ALPHA, MAT), -2)
LUT = ALPHA.byte_lut()


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True,
                             timeout=30).stdout.strip().split(", ")
        return {"gpu": out[0], "power_limit_w": float(out[1]), "sm_clock_mhz": int(out[2]), "sm_clock_max_mhz": int(out[3])}
    except Exception as e:  # reported, not fatal
        return {"gpu": torch.cuda.get_device_name(0), "nvidia_smi_error": str(e)}


def reads(n, L, kind, family, dev, first=0, seed=synth.SEED_READS):
    seqs = torch.empty(max(n * L, 1), dtype=torch.uint8, device=dev)
    _lib.check(_lib.lib().pg_synth_reads_dev(seqs.data_ptr(), first, n, L, seed, kind, family, torch.cuda.current_stream(dev).cuda_stream))
    return seqs, torch.arange(n + 1, dtype=torch.int64, device=dev) * L


class Set:
    """A ragged sequence set on the device, with host copies for the oracle."""

    def __init__(self, seqs, off):
        self.seqs, self.off = seqs, off
        self.h_seqs, self.h_off = seqs.cpu().numpy(), off.cpu().numpy()
        self.max_len = int(np.diff(self.h_off).max()) if len(self.h_off) > 1 else 0

    def get(self, i):
        return bytes(self.h_seqs[int(self.h_off[i]): int(self.h_off[i + 1])])

    def lens(self):
        return np.diff(self.h_off)


def timed(fn, runs, warmup=2):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(runs):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts), ts


def oracle_scores(A, B, pairs, global_alignment, threads):
    """Scores from the C pair driver over the restated po_sw_score / po_nw_score (oracle/pair_oracle.c)."""
    return pair_oracle.scores((A.h_seqs, A.h_off), (B.h_seqs, B.h_off), pairs, LUT, LUT, MAT, -2, global_alignment, threads)[0].tolist()


def pair_run(name, A, B, pairs, global_alignment, runs, parity_n, threads, extra=None):
    d_pairs = torch.from_numpy(pairs.astype(np.int32)).to(A.seqs.device)
    call = lambda: align.pair_scores_device(A.seqs, A.off, A.max_len, B.seqs, B.off, B.max_len, d_pairs, SC, global_alignment)  # noqa: E731
    ms, ts = timed(call, runs)
    score, ec, _ = (x.cpu().numpy() for x in call())
    cells = int((A.lens()[pairs[:, 0]].astype(np.float64) * B.lens()[pairs[:, 1]]).sum())
    idx = np.random.default_rng(1).choice(len(pairs), min(parity_n, len(pairs)), replace=False)
    want = oracle_scores(A, B, pairs[idx], global_alignment, threads)
    rec = {"workload": name, "mode": "NW" if global_alignment else "SW", "pairs": len(pairs), "cells": cells, "median_ms": round(ms, 3),
           "runs_ms": [round(t, 3) for t in ts], "gcups": round(cells / ms / 1e6, 1), "errors": int((ec != 0).sum()),
           "parity_sample": len(idx), "parity_ok": bool(score[idx].tolist() == want and not ec.any())}
    rec.update(extra or {})
    return rec


def cpu_arm(name, A, B, pairs, threads):
    t0 = time.perf_counter()
    oracle_scores(A, B, pairs, False, threads)
    s = time.perf_counter() - t0
    cells = int((A.lens()[pairs[:, 0]].astype(np.float64) * B.lens()[pairs[:, 1]]).sum())
    return {"workload": name, "arm": "cpu", "label": "C restatement, not Go", "threads": threads, "pairs": len(pairs), "cells": cells,
            "seconds": round(s, 3), "gcups": round(cells / s / 1e9, 3)}


def one_template(q, qmax, d_t, tlen, d_score, d_ec, d_ep, st):
    """pg_sw_score_batch_dev: the queries of set q against one template (query = stringA)."""
    _lib.check(_lib.lib().pg_sw_score_batch_dev(q.seqs.data_ptr(), q.off.data_ptr(), q.off.numel() - 1, qmax, d_t.data_ptr(), tlen, 1,
                                                LUT.ctypes.data, LUT.ctypes.data, MAT.ctypes.data, 5, 5, -2, d_score.data_ptr(),
                                                d_ec.data_ptr(), d_ep.data_ptr(), st))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--scale", type=float, default=1.0, help="fraction of the P1-P3, P5 pair counts (rehearsal)")
    ap.add_argument("--only", default="P1,P2,P3,P4,P5,CPU")
    ap.add_argument("--out", default=None, help="also write the records here (JSON list)")
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    st = torch.cuda.current_stream(dev).cuda_stream
    threads = len(os.sched_getaffinity(0))
    info = gpu_info()
    only = set(args.only.split(","))
    recs = []

    def emit(r):
        r.update(info)
        print(json.dumps(r), flush=True)
        recs.append(r)

    # P1: family reads, each against the next read of its family (wrapping inside the family)
    n1, F = int(1_000_000 * args.scale), 100
    P1 = Set(*reads(n1, 150, 1, F, dev))
    i = np.arange(n1)
    p1 = np.stack([i, np.where((i + 1) % F == 0, i + 1 - F, i + 1) % n1], 1)
    if "P1" in only:
        for g in (False, True):
            emit(pair_run("P1", P1, P1, p1, g, args.runs, 2000, threads))
    if "P2" in only:
        n2 = int(100_000 * args.scale)
        R2 = Set(*reads(n2, 150, 0, 0, dev, seed=synth.SEED_READS + 2))
        rng = np.random.default_rng(2)
        tl = rng.integers(1000, 10_001, 1000)
        toff = np.zeros(len(tl) + 1, np.int64)
        np.cumsum(tl, out=toff[1:])
        tseq, _ = reads(1, int(toff[-1]), 0, 0, dev, seed=synth.SEED_READS + 3)
        T2 = Set(tseq, torch.from_numpy(toff).to(dev))
        p2 = np.stack([np.arange(n2), rng.integers(0, len(tl), n2)], 1)
        emit(pair_run("P2", R2, T2, p2, False, args.runs, 300, threads))
    if "P3" in only or "CPU" in only:
        n_ref, n_q, L = int(9000 * args.scale), int(1000 * args.scale), 10_000
        seqs, off = reads(n_ref + n_q, L, 1, F, dev)
        h = seqs.cpu().numpy()
        sk = mash.sketch_uniform(h, n_ref + n_q, L, 31, 2000)
        qi = np.arange(0, n_ref + n_q, 10)[:n_q]
        ri = np.setdiff1d(np.arange(n_ref + n_q), qi)
        ix = mash.SketchIndex(sk[ri])
        ref = np.asarray(ix.nearest(sk[qi], 4)[0]).astype(np.int64)
        assert (ref != 0xFFFFFFFF).all()
        Q = Set(torch.from_numpy(h.reshape(-1, L)[qi].reshape(-1).copy()).to(dev), torch.arange(len(qi) + 1, dtype=torch.int64, device=dev) * L)
        R = Set(torch.from_numpy(h.reshape(-1, L)[ri].reshape(-1).copy()).to(dev), torch.arange(len(ri) + 1, dtype=torch.int64, device=dev) * L)
        p3 = np.stack([np.repeat(np.arange(len(qi)), 4), ref.reshape(-1)], 1)
        if "P3" in only:
            rec = pair_run("P3", Q, R, p3, False, args.runs, 16, threads)
            s3, _, _ = (x.cpu().numpy() for x in align.pair_scores_device(Q.seqs, Q.off, L, R.seqs, R.off, L, torch.from_numpy(p3.astype(np.int32)).to(dev), SC))
            best = ri[p3[np.arange(len(qi)) * 4 + s3.reshape(-1, 4).argmax(1), 1]]
            rec["best_hit_in_family"] = float(((best // F) == (qi // F)).mean())
            emit(rec)
        if "CPU" in only:
            emit(cpu_arm("P1", P1, P1, p1[: 20_000 if args.scale >= 1 else 2000], threads))
            emit(cpu_arm("P3", Q, R, p3[: max(threads, 4)], threads))
    d_sc, d_ec, d_ep = (torch.empty(10_000, dtype=t, device=dev) for t in (torch.int64, torch.int32, torch.int64))
    if "P4" in only:
        a, _ = reads(1, 20_000, 0, 0, dev, seed=synth.SEED_READS + 4)
        b = a.clone()
        b[::97] = ord("A")  # a related pair with substitutions
        A4 = Set(a, torch.tensor([0, 20_000], dtype=torch.int64, device=dev))
        B4 = Set(b, torch.tensor([0, 20_000], dtype=torch.int64, device=dev))
        pairs = torch.zeros((1, 2), dtype=torch.int32, device=dev)
        new = lambda: align.pair_scores_device(A4.seqs, A4.off, 20_000, B4.seqs, B4.off, 20_000, pairs, SC)  # noqa: E731
        old = lambda: one_template(A4, 20_000, b, 20_000, d_sc, d_ec, d_ep, st)  # noqa: E731
        new(); old(); torch.cuda.synchronize()
        tn, to = [], []
        for _ in range(args.runs):  # alternating
            tn.append(timed(new, 1, 0)[0])
            to.append(timed(old, 1, 0)[0])
        s_new = int(new()[0].cpu()[0])
        old(); torch.cuda.synchronize()
        s_old = int(d_sc[0].cpu())
        want = oracle_scores(A4, B4, np.zeros((1, 2), np.int64), False, 1)[0]
        cells = 20_000 * 20_000
        emit({"workload": "P4", "mode": "SW", "pairs": 1, "cells": cells, "pairs_median_ms": round(statistics.median(tn), 3),
              "one_template_median_ms": round(statistics.median(to), 3), "pairs_runs_ms": [round(t, 3) for t in tn],
              "one_template_runs_ms": [round(t, 3) for t in to], "pairs_gcups": round(cells / statistics.median(tn) / 1e6, 2),
              "one_template_gcups": round(cells / statistics.median(to) / 1e6, 3), "speedup": round(statistics.median(to) / statistics.median(tn), 1),
              "parity_ok": s_new == s_old == want})
    if "P5" in only:
        n5 = int(10_000 * args.scale)
        Qs = Set(*reads(n5, 500, 0, 0, dev, seed=synth.SEED_READS + 5))
        t, _ = reads(1, 10_000, 0, 0, dev, seed=synth.SEED_READS + 6)
        T5 = Set(t, torch.tensor([0, 10_000], dtype=torch.int64, device=dev))
        p5 = torch.from_numpy(np.stack([np.arange(n5), np.zeros(n5, np.int64)], 1).astype(np.int32)).to(dev)
        new = lambda: align.pair_scores_device(Qs.seqs, Qs.off, 500, T5.seqs, T5.off, 10_000, p5, SC)  # noqa: E731
        old = lambda: one_template(Qs, 500, t, 10_000, d_sc, d_ec, d_ep, st)  # noqa: E731
        tn, _ = timed(new, args.runs)
        to, _ = timed(old, args.runs)
        s_new = new()[0].cpu().numpy()
        old(); torch.cuda.synchronize()
        s_old = d_sc[:n5].cpu().numpy()
        cells = n5 * 500 * 10_000
        emit({"workload": "P5", "mode": "SW", "pairs": n5, "cells": cells, "pairs_median_ms": round(tn, 3), "one_template_median_ms": round(to, 3),
              "pairs_gcups": round(cells / tn / 1e6, 1), "one_template_gcups": round(cells / to / 1e6, 1), "parity_ok": bool(np.array_equal(s_new, s_old))})
    if args.out:
        with open(args.out, "w") as f:
            json.dump(recs, f, indent=1)
    if not all(r.get("parity_ok", True) for r in recs):
        sys.exit("parity check failed")


if __name__ == "__main__":
    main()
