#!/usr/bin/env python
"""Mash Screen of a multiplexed run, every sample in one pass, against a reference sketch set; prints one JSON line
(profiles/h100_screen_samples_n1.json; --out also writes it to a file).

Workload, seeded and generated on the device:
  references: --genomes random genomes of --genome-len bp, sketched with k = 21, s = 1000 through
              pg_mash_sketch_batch_dev (select regime);
  run:        --samples samples x --reads-per-sample reads of 150 bp; sample q takes 90 % of its reads from its own
              3 source genomes (3q, 3q + 1, 3q + 2) at random positions with 1 % substitutions and 10 % random reads.
              The reads of all samples are interleaved at random, each tagged with its sample id.
Legs, --runs times after --warmup rounds, one of each per round in this order, medians reported (CUDA events unless
noted):
  add_samples:     one pg_mash_screen_add_samples_dev of the whole run after a reset;
  add_single:      one pg_mash_screen_add_dev of the same bytes on a one-sample screen (no ids);
  k1:              pg_mash_sketch_uniform_dev over the same bytes at k = 21, s = 1000;
  results_samples: one pg_mash_screen_results_samples_dev over every sample;
  winners_samples: one pg_mash_screen_winners_samples_dev over every sample;
  per_sample:      one one-sample screen, per sample a reset, a pg_mash_screen_add_dev of that sample's reads
                   (gathered into one contiguous buffer outside the timing) and pg_mash_screen_results_dev; the passes
                   of every sample timed together with a host clock that ends in a synchronise (the reset is a host
                   call, so each pass first waits for the previous one).
Checked in the run: every row of results_samples equals the per-sample passes' results, and three sampled samples'
rows of winners_samples equal a one-sample screen's winners; one sample's 100 k reads against --oracle-refs sampled
references (a screen of every sample fed the whole run) equal the CPU restatement (tests/screen_oracle.py); in every
sample's own row its 3 sources reach containment >= 0.9 and no other reference reaches 0.2.

At 100 k reads a sample covers each of its sources about 4.5 x, so a source's containment is not near 1: a window of
a source is seen by about lambda = (reads per source) x 129 windows / 1 Mbp x 0.99^21 (no substitution in it) = 3.1
reads, and seen at all with probability 1 - exp(-lambda) = 0.956 (source_containment_expected).  The 0.9 bound leaves
room for the sampling of s = 1 000 hashes and of the reads per source."""
import argparse
import ctypes as C
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from bench_cluster import gpu_info  # noqa: E402
from poly_b200 import _lib  # noqa: E402

K, S, READ_LEN, SOURCES = 21, 1000, 150, 3


def make_workload(args, dev, st):
    g = torch.Generator(device=dev)
    g.manual_seed(20261018)
    acgt = torch.tensor(list(b"ACGT"), dtype=torch.uint8, device=dev)
    G, GL, Q, R = args.genomes, args.genome_len, args.samples, args.reads_per_sample
    assert Q * SOURCES <= G
    genomes = acgt[torch.randint(0, 4, (G * GL,), generator=g, device=dev)]
    g_off = torch.arange(G + 1, dtype=torch.int64, device=dev) * GL
    sk = torch.empty((G, S), dtype=torch.int32, device=dev)
    L = _lib.lib()
    _lib.check(L.pg_mash_sketch_batch_dev(genomes.data_ptr(), g_off.data_ptr(), G, GL, K, S, 0, sk.data_ptr(), S, None, None, st))
    n = Q * R
    ids = torch.arange(n, device=dev) // R  # sample-major before the shuffle
    pool = torch.empty(n * READ_LEN, dtype=torch.uint8, device=dev)
    step = 1 << 20
    col = torch.arange(READ_LEN, dtype=torch.int64, device=dev)
    for a in range(0, n, step):
        b = min(a + step, n)
        m = b - a
        rows = acgt[torch.randint(0, 4, (m, READ_LEN), generator=g, device=dev)]
        src = (torch.arange(a, b, device=dev) % R) < R * 9 // 10
        gi = ids[a:b] * SOURCES + torch.randint(0, SOURCES, (m,), generator=g, device=dev)
        start = torch.randint(0, GL - READ_LEN + 1, (m,), generator=g, device=dev)
        copied = genomes[(gi * GL + start)[:, None] + col]
        sub = torch.rand((m, READ_LEN), generator=g, device=dev) < 0.01
        copied = torch.where(sub, acgt[torch.randint(0, 4, (m, READ_LEN), generator=g, device=dev)], copied)
        pool[a * READ_LEN:b * READ_LEN] = torch.where(src[:, None], copied, rows).reshape(-1)
    grouped = pool  # sample q's reads are rows [q R, q R + R): the per-sample passes' contiguous buffers
    perm = torch.randperm(n, generator=g, device=dev)  # interleave the samples
    pool = grouped.view(n, READ_LEN)[perm].reshape(-1).contiguous()
    ids = ids[perm].to(torch.int32).contiguous()
    p_off = torch.arange(n + 1, dtype=torch.int64, device=dev) * READ_LEN
    torch.cuda.synchronize()
    del genomes
    return sk, pool, p_off, ids, grouped


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--genomes", type=int, default=1000)
    ap.add_argument("--genome-len", type=int, default=1_000_000)
    ap.add_argument("--samples", type=int, default=96)
    ap.add_argument("--reads-per-sample", type=int, default=100_000)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--oracle-refs", type=int, default=50)
    ap.add_argument("--oracle-threads", type=int, default=16)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    L = _lib.lib()
    _lib.check(L.pg_init(0))
    dev = torch.device("cuda", 0)
    st = torch.cuda.current_stream(dev).cuda_stream
    before = gpu_info()
    sk, pool, p_off, ids, grouped = make_workload(args, dev, st)
    G, Q, R = args.genomes, args.samples, args.reads_per_sample
    n = Q * R
    k1_out = torch.empty((n, READ_LEN - K), dtype=torch.int32, device=dev)
    tab = [torch.empty((Q, G), dtype=t, device=dev) for t in (torch.int32, torch.float64, torch.int64)]
    win = [torch.empty((Q, G), dtype=t, device=dev) for t in (torch.int32, torch.float64, torch.int64)]
    one = [torch.empty((Q, G), dtype=t, device=dev) for t in (torch.int32, torch.float64, torch.int64)]  # the per-sample rows
    s_off = torch.arange(R + 1, dtype=torch.int64, device=dev) * READ_LEN

    def events(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    def create(samples):
        h = C.c_void_p()
        _lib.check(L.pg_mash_screen_create_samples_dev(sk.data_ptr(), G, S, K, samples, st, C.byref(h)))
        return h

    def per_sample(h1):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for q in range(Q):
            torch.cuda.synchronize()  # the reset below runs on the library's stream
            _lib.check(L.pg_mash_screen_reset(h1))
            _lib.check(L.pg_mash_screen_add_dev(h1, grouped.data_ptr() + q * R * READ_LEN, s_off.data_ptr(), R, st))
            _lib.check(L.pg_mash_screen_results_dev(h1, one[0][q].data_ptr(), one[1][q].data_ptr(), one[2][q].data_ptr(), st))
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3

    t = {key: [] for key in ("add_samples", "add_single", "k1", "results_samples", "winners_samples", "per_sample")}
    hq, h1 = create(Q), create(1)
    try:
        for r in range(args.warmup + args.runs):
            _lib.check(L.pg_mash_screen_reset(hq))
            _lib.check(L.pg_mash_screen_reset(h1))
            ms = {
                "add_samples": events(lambda: _lib.check(L.pg_mash_screen_add_samples_dev(hq, pool.data_ptr(), p_off.data_ptr(), ids.data_ptr(), n, st))),
                "add_single": events(lambda: _lib.check(L.pg_mash_screen_add_dev(h1, pool.data_ptr(), p_off.data_ptr(), n, st))),
                "k1": events(lambda: _lib.check(L.pg_mash_sketch_uniform_dev(pool.data_ptr(), n, READ_LEN, K, S, 0, k1_out.data_ptr(), READ_LEN - K, None,
                                                                             st))),
                "results_samples": events(lambda: _lib.check(L.pg_mash_screen_results_samples_dev(hq, 0, Q, *(x.data_ptr() for x in tab), st))),
                "winners_samples": events(lambda: _lib.check(L.pg_mash_screen_winners_samples_dev(hq, 0, Q, *(x.data_ptr() for x in win), st))),
                "per_sample": per_sample(h1),
            }
            if r >= args.warmup:
                for key, v in ms.items():
                    t[key].append(v)
    finally:
        torch.cuda.synchronize()
        _lib.check(L.pg_mash_screen_free(hq))
        _lib.check(L.pg_mash_screen_free(h1))

    def host(ts):
        return ts[0].cpu().numpy().view(np.uint32), ts[1].cpu().numpy(), ts[2].cpu().numpy().view(np.uint64)

    res, won, rows_one = host(tab), host(win), host(one)
    same = lambda a, b: all(x.tobytes() == y.tobytes() for x, y in zip(a, b))  # noqa: E731
    # every sample's rows against the per-sample passes (results), three sampled samples against one-sample winners
    rows_parity = same(res, rows_one)
    rng = np.random.default_rng(7)
    picked = sorted(int(x) for x in rng.choice(Q, min(3, Q), replace=False))
    win_parity = True
    for q in picked:
        h = create(1)
        try:
            _lib.check(L.pg_mash_screen_add_dev(h, grouped.data_ptr() + q * R * READ_LEN, s_off.data_ptr(), R, st))
            w1 = [torch.empty(G, dtype=x.dtype, device=dev) for x in win]
            _lib.check(L.pg_mash_screen_winners_dev(h, *(x.data_ptr() for x in w1), st))
            torch.cuda.synchronize()
        finally:
            _lib.check(L.pg_mash_screen_free(h))
        win_parity &= same(host(w1), tuple(x[q] for x in won))
    src = np.arange(Q)[:, None] * SOURCES + np.arange(SOURCES)
    own = np.zeros((Q, G), bool)
    own[np.arange(Q)[:, None], src] = True
    src_min = float(res[1][own].min())
    other_max = float(res[1][~own].max())
    lam = R * 9 / 10 / SOURCES * (READ_LEN - K) / args.genome_len * 0.99 ** K

    # one sample's reads against sampled references: the screen of every sample fed the whole run, against the oracle
    import screen_oracle

    qo = picked[0]
    pick = np.sort(np.concatenate([src[qo], rng.choice(np.setdiff1d(np.arange(G), src[qo]), args.oracle_refs - SOURCES, replace=False)]))
    sk_sub = np.ascontiguousarray(sk.cpu().numpy().view(np.uint32)[pick])
    sub_bases = grouped[qo * R * READ_LEN:(qo + 1) * R * READ_LEN].cpu().numpy()
    sub_off = np.arange(R + 1, dtype=np.uint64) * READ_LEN
    t0 = time.perf_counter()
    want = screen_oracle.mash_screen(sk_sub, (sub_bases, sub_off), K, nthreads=args.oracle_threads)
    oracle_s = time.perf_counter() - t0
    d_sub = torch.from_numpy(sk_sub.view(np.int32)).to(dev)
    h = C.c_void_p()
    _lib.check(L.pg_mash_screen_create_samples_dev(d_sub.data_ptr(), len(pick), S, K, Q, st, C.byref(h)))
    try:
        _lib.check(L.pg_mash_screen_add_samples_dev(h, pool.data_ptr(), p_off.data_ptr(), ids.data_ptr(), n, st))
        torch.cuda.synchronize()
        got = np.zeros(len(pick), np.uint32), np.zeros(len(pick), np.float64), np.zeros(len(pick), np.uint64)
        _lib.check(L.pg_mash_screen_results_samples(h, qo, 1, *(x.ctypes.data for x in got)))
    finally:
        _lib.check(L.pg_mash_screen_free(h))
    oracle_parity = same(got, want) and int(want[0].sum()) > 0
    ok = rows_parity and win_parity and oracle_parity and src_min >= 0.9 and other_max < 0.2

    med = {key: statistics.median(v) for key, v in t.items()}
    bases = n * READ_LEN
    line = {
        "metric": "mash_screen_samples",
        "shape": f"{G} x {args.genome_len} bp references, k={K}, s={S}; run of {Q} samples x {R} x {READ_LEN} bp reads, interleaved "
                 f"(each sample 90% from its own {SOURCES} references, 1% substitutions)",
        "runs": args.runs, "warmup": args.warmup,
        **{f"{key}_ms": round(v, 3) for key, v in med.items()},
        "add_samples_gbases_per_s": round(bases / med["add_samples"] / 1e6, 1),
        "add_samples_over_add_single": round(med["add_samples"] / med["add_single"], 3),
        "add_samples_over_k1": round(med["add_samples"] / med["k1"], 3), "add_single_over_k1": round(med["add_single"] / med["k1"], 3),
        "one_pass_ms": round(med["add_samples"] + med["results_samples"], 3),
        "per_sample_over_one_pass": round(med["per_sample"] / (med["add_samples"] + med["results_samples"]), 2),
        "all_ms": {key: [round(x, 3) for x in v] for key, v in t.items()},
        "source_containment_min": src_min, "source_containment_expected": round(1 - float(np.exp(-lam)), 4),
        "source_containment_median": float(np.median(res[1][own])), "other_containment_max": other_max, "rows_equal_per_sample_passes": rows_parity, "winners_rows_equal_one_sample": win_parity,
        "winners_checked_samples": picked, "oracle_parity": oracle_parity, "oracle_sample": qo, "oracle_refs": len(pick), "oracle_reads": R,
        "oracle_threads": args.oracle_threads, "oracle_s": round(oracle_s, 3), "ok": ok,
        **before, "sm_clock_mhz_after": gpu_info().get("sm_clock_mhz"),
    }
    print(json.dumps(line))
    if args.out:
        with open(args.out, "w") as f:
            f.write(json.dumps(line) + "\n")
    if not ok:
        sys.exit(1)


if __name__ == "__main__":
    main()
