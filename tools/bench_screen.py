#!/usr/bin/env python
"""Mash Screen of a metagenome-shaped pool against a reference sketch set; prints one JSON line
(profiles/h100_screen_n1.json; --out also writes it to a file).

Workload, seeded and generated on the device:
  references: --genomes random genomes of --genome-len bp, sketched with k = 21, s = 1000 through
              pg_mash_sketch_batch_dev (select regime: each sketch is its genome's bottom 1000 hashes);
  pool:       --reads reads of 150 bp (the cfg2 shape): 90 % drawn from the first 20 genomes at random positions
              with 1 % substitutions, 10 % random.
Legs, --runs times after --warmup rounds, medians reported, the add and K1 legs alternating:
  create:  pg_mash_screen_create_dev over the sketches (host clock; create synchronises);
  add:     one pg_mash_screen_add_dev of the whole pool after a reset, CUDA events; Gbases/s of pool;
  results: pg_mash_screen_results_dev, CUDA events;
  k1:      pg_mash_sketch_uniform_dev over the same pool bytes at k = 21, s = 1000 (the headline K1, which hashes the
           same windows), CUDA events.
Checked in the run: the 20 source genomes have containment >= 0.99, and a screen of
the first --oracle-reads reads against --oracle-refs sampled references equals the CPU restatement (tests/screen_oracle.py) in
shared, multiplicity and containment bytes; that call (window hashes by the C oracle on 16 host threads, counting in
NumPy on one) is timed for scale.  The other
genomes' containment is reported, not checked: with 32-bit hashes each of their values is also the hash of some pool
window with probability about 1 - exp(-windows / 2^32), which their multiplicity (near 1, against the sources'
coverage) tells apart."""
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

K, S, READ_LEN, SOURCES = 21, 1000, 150, 20


def make_workload(args, dev, st):
    g = torch.Generator(device=dev)
    g.manual_seed(20260101)
    acgt = torch.tensor(list(b"ACGT"), dtype=torch.uint8, device=dev)
    G, GL = args.genomes, args.genome_len
    genomes = acgt[torch.randint(0, 4, (G * GL,), generator=g, device=dev)]
    g_off = torch.arange(G + 1, dtype=torch.int64, device=dev) * GL
    sk = torch.empty((G, S), dtype=torch.int32, device=dev)
    L = _lib.lib()
    _lib.check(L.pg_mash_sketch_batch_dev(genomes.data_ptr(), g_off.data_ptr(), G, GL, K, S, 0, sk.data_ptr(), S, None, None, st))
    n = args.reads
    n_src = n * 9 // 10
    pool = torch.empty(n * READ_LEN, dtype=torch.uint8, device=dev)
    step = 1 << 20
    col = torch.arange(READ_LEN, dtype=torch.int64, device=dev)
    for a in range(0, n, step):
        b = min(a + step, n)
        m = b - a
        rows = acgt[torch.randint(0, 4, (m, READ_LEN), generator=g, device=dev)]
        src = torch.arange(a, b, device=dev) < n_src
        if bool(src.any()):
            gi = torch.randint(0, SOURCES, (m,), generator=g, device=dev)
            start = torch.randint(0, GL - READ_LEN + 1, (m,), generator=g, device=dev)
            idx = (gi * GL + start)[:, None] + col
            copied = genomes[idx]
            sub = torch.rand((m, READ_LEN), generator=g, device=dev) < 0.01
            copied = torch.where(sub, acgt[torch.randint(0, 4, (m, READ_LEN), generator=g, device=dev)], copied)
            rows = torch.where(src[:, None], copied, rows)
        pool[a * READ_LEN:b * READ_LEN] = rows.reshape(-1)
    # shuffle the reads so source and random reads interleave
    perm = torch.randperm(n, generator=g, device=dev)
    pool = pool.view(n, READ_LEN)[perm].reshape(-1).contiguous()
    p_off = torch.arange(n + 1, dtype=torch.int64, device=dev) * READ_LEN
    torch.cuda.synchronize()
    del genomes
    return sk, pool, p_off


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--genomes", type=int, default=1000)
    ap.add_argument("--genome-len", type=int, default=1_000_000)
    ap.add_argument("--reads", type=int, default=10_000_000)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--oracle-reads", type=int, default=100_000)
    ap.add_argument("--oracle-refs", type=int, default=50)
    ap.add_argument("--oracle-threads", type=int, default=16)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    L = _lib.lib()
    _lib.check(L.pg_init(0))
    dev = torch.device("cuda", 0)
    st = torch.cuda.current_stream(dev).cuda_stream
    before = gpu_info()
    sk, pool, p_off = make_workload(args, dev, st)
    G, n = args.genomes, args.reads
    k1_out = torch.empty((n, READ_LEN - K), dtype=torch.int32, device=dev)
    shared = torch.empty(G, dtype=torch.int32, device=dev)
    cont = torch.empty(G, dtype=torch.float64, device=dev)
    mult = torch.empty(G, dtype=torch.int64, device=dev)

    def events(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    def create():
        h = C.c_void_p()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        _lib.check(L.pg_mash_screen_create_dev(sk.data_ptr(), G, S, K, st, C.byref(h)))
        return h, (time.perf_counter() - t0) * 1e3

    t = {"create": [], "add": [], "results": [], "k1": []}
    h, _ = create()
    try:
        for r in range(args.warmup + args.runs):
            h2, ms_create = create()
            _lib.check(L.pg_mash_screen_free(h2))
            _lib.check(L.pg_mash_screen_reset(h))
            ms_add = events(lambda: _lib.check(L.pg_mash_screen_add_dev(h, pool.data_ptr(), p_off.data_ptr(), n, st)))
            ms_k1 = events(lambda: _lib.check(L.pg_mash_sketch_uniform_dev(pool.data_ptr(), n, READ_LEN, K, S, 0, k1_out.data_ptr(), READ_LEN - K,
                                                                             None, st)))
            ms_res = events(lambda: _lib.check(L.pg_mash_screen_results_dev(h, shared.data_ptr(), cont.data_ptr(), mult.data_ptr(), st)))
            if r >= args.warmup:
                for key, v in (("create", ms_create), ("add", ms_add), ("k1", ms_k1), ("results", ms_res)):
                    t[key].append(v)
    finally:
        _lib.check(L.pg_mash_screen_free(h))
    c = cont.cpu().numpy()
    src_min = float(c[:SOURCES].min())
    other = c[SOURCES:] if G > SOURCES else np.zeros(1)
    m = mult.cpu().numpy().view(np.uint64)

    # parity on a sub-pool and sampled references, against the CPU oracle on host threads
    import screen_oracle

    rng = np.random.default_rng(7)
    pick = np.sort(np.concatenate([np.arange(min(5, G)), rng.choice(np.arange(min(5, G), G), min(args.oracle_refs, G) - min(5, G), replace=False)]))
    sk_sub = sk.cpu().numpy().view(np.uint32)[pick]
    nr = min(args.oracle_reads, n)
    sub_bases = pool[: nr * READ_LEN].cpu().numpy()
    sub_off = np.arange(nr + 1, dtype=np.uint64) * READ_LEN
    t0 = time.perf_counter()
    want = screen_oracle.mash_screen(sk_sub, (sub_bases, sub_off), K, nthreads=args.oracle_threads)
    oracle_s = time.perf_counter() - t0
    hs = C.c_void_p()
    _lib.check(L.pg_mash_screen_create(sk_sub.ctypes.data, len(pick), S, K, C.byref(hs)))
    try:
        _lib.check(L.pg_mash_screen_add(hs, sub_bases.ctypes.data, sub_off.ctypes.data, nr))
        got = np.zeros(len(pick), np.uint32), np.zeros(len(pick), np.float64), np.zeros(len(pick), np.uint64)
        _lib.check(L.pg_mash_screen_results(hs, *(x.ctypes.data for x in got)))
    finally:
        _lib.check(L.pg_mash_screen_free(hs))
    parity = all(g.tobytes() == w.tobytes() for g, w in zip(got, want)) and int(want[0].sum()) > 0
    ok = parity and src_min >= 0.99

    bases = n * READ_LEN
    add_ms, k1_ms = statistics.median(t["add"]), statistics.median(t["k1"])
    line = {
        "metric": "mash_screen", "shape": f"{G} x {args.genome_len} bp references, k={K}, s={S}; pool {n} x {READ_LEN} bp "
                                          f"(90% from {SOURCES} references, 1% substitutions)",
        "runs": args.runs, "warmup": args.warmup,
        "create_ms": round(statistics.median(t["create"]), 3), "add_ms": round(add_ms, 3), "results_ms": round(statistics.median(t["results"]), 3),
        "k1_ms": round(k1_ms, 3), "add_gbases_per_s": round(bases / add_ms / 1e6, 1), "k1_gbases_per_s": round(bases / k1_ms / 1e6, 1),
        "add_over_k1": round(add_ms / k1_ms, 3), "windows": n * (READ_LEN - K),
        "all_ms": {key: [round(x, 3) for x in v] for key, v in t.items()},
        "source_containment_min": src_min, "other_containment_median": float(np.median(other)), "other_containment_max": float(other.max()),
        "source_multiplicity_median": int(np.median(m[:SOURCES])), "other_multiplicity_max": int(m[SOURCES:].max()) if G > SOURCES else 0,
        "oracle_parity": parity, "oracle_refs": len(pick), "oracle_reads": nr, "oracle_threads": args.oracle_threads,
        "oracle_s": round(oracle_s, 3), "ok": ok,
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
