#!/usr/bin/env python
"""Mash Screen's winner-take-all against a reference set of strain families; prints one JSON line
(profiles/h100_screen_winners_n1.json; --out also writes it to a file).

Workload, seeded and generated on the device:
  references: --species random genomes of --genome-len bp, each with --strains strains at substitution rates spread
              evenly over 0.2 .. 5 % (row species * strains + strain), sketched with k = 21, s = 1000 through
              pg_mash_sketch_batch_dev (select regime);
  pool:       --reads reads of 150 bp: 90 % drawn from one strain of each of the first 20 species (species i's strain
              i mod strains, so the sources span the rates) with 1 % substitutions, 10 % random.
Legs, --runs times after --warmup rounds, CUDA-event medians:
  add:      one pg_mash_screen_add_dev of the whole pool after a reset (for scale);
  results:  pg_mash_screen_results_dev;
  winners:  pg_mash_screen_winners_dev.
Scale leg: --scale-n synthetic rows of s = 1000 words in families of 10 that share 80 % of their words (the
family's base row; the other 20 % are each row's own), every word a window hash of the pool, so 10^8 keys at the
default; the whole pool is added once, then results_dev and winners_dev alternate.
Checked in the run: each source strain is its species' top reference under winners; the references at containment
>= 0.5 under results and under winners are counted and reported (expected: about the strains near each source
before, one per present species after); winners never exceeds results for any row of either set; and a screen of
the first --oracle-reads reads against every strain of species 0, 1 and the last one equals the CPU restatement
(tests/screen_winners_oracle.py) in shared, multiplicity and containment bytes."""
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
    g.manual_seed(20261018)
    acgt = torch.tensor(list(b"ACGT"), dtype=torch.uint8, device=dev)
    P, T, GL = args.species, args.strains, args.genome_len
    rates = torch.linspace(0.002, 0.05, T, device=dev)
    sk = torch.empty((P * T, S), dtype=torch.int32, device=dev)
    src = torch.empty((SOURCES, GL), dtype=torch.uint8, device=dev)
    off = torch.arange(T + 1, dtype=torch.int64, device=dev) * GL
    L = _lib.lib()
    for p in range(P):  # one species at a time: its root and strains
        root = torch.randint(0, 4, (GL,), generator=g, device=dev)
        sub = torch.rand((T, GL), generator=g, device=dev) < rates[:, None]
        shift = torch.randint(1, 4, (T, GL), generator=g, device=dev)
        strains = acgt[torch.where(sub, (root + shift) % 4, root)].contiguous()  # a substitution is a different base
        _lib.check(L.pg_mash_sketch_batch_dev(strains.data_ptr(), off.data_ptr(), T, GL, K, S, 0, sk[p * T:].data_ptr(), S, None, None, st))
        if p < SOURCES:
            src[p] = strains[p % T]
        torch.cuda.synchronize()
    n = args.reads
    n_src = n * 9 // 10
    pool = torch.empty(n * READ_LEN, dtype=torch.uint8, device=dev)
    step = 1 << 20
    col = torch.arange(READ_LEN, dtype=torch.int64, device=dev)
    for a in range(0, n, step):
        b = min(a + step, n)
        m = b - a
        rows = acgt[torch.randint(0, 4, (m, READ_LEN), generator=g, device=dev)]
        is_src = torch.arange(a, b, device=dev) < n_src
        if bool(is_src.any()):
            gi = torch.randint(0, SOURCES, (m,), generator=g, device=dev)
            start = torch.randint(0, GL - READ_LEN + 1, (m,), generator=g, device=dev)
            copied = src.view(-1)[(gi * GL + start)[:, None] + col]
            sub = torch.rand((m, READ_LEN), generator=g, device=dev) < 0.01
            copied = torch.where(sub, acgt[torch.randint(0, 4, (m, READ_LEN), generator=g, device=dev)], copied)
            rows = torch.where(is_src[:, None], copied, rows)
        pool[a * READ_LEN:b * READ_LEN] = rows.reshape(-1)
    perm = torch.randperm(n, generator=g, device=dev)  # source and random reads interleave
    pool = pool.view(n, READ_LEN)[perm].reshape(-1).contiguous()
    p_off = torch.arange(n + 1, dtype=torch.int64, device=dev) * READ_LEN
    torch.cuda.synchronize()
    return sk, pool, p_off, g


def scale_rows(args, pool, g, dev, st):
    """--scale-n rows in families of 10: 80 % of each row is its family's base row, 20 % its own; every word is a
    window hash of the pool's first reads (K1 writes each window's hash when s exceeds the windows)."""
    L = _lib.lib()
    nr = 1 << 20
    w = READ_LEN - K
    hashes = torch.empty((nr, w), dtype=torch.int32, device=dev)
    _lib.check(L.pg_mash_sketch_uniform_dev(pool.data_ptr(), nr, READ_LEN, K, S, 0, hashes.data_ptr(), w, None, st))
    hashes = hashes.view(-1)
    n = args.scale_n
    fam = torch.randint(0, hashes.numel(), (n // 10, S), generator=g, device=dev)
    rows = fam.repeat_interleave(10, dim=0)
    own = torch.rand((n, S), generator=g, device=dev) < 0.2
    rows = torch.where(own, torch.randint(0, hashes.numel(), (n, S), generator=g, device=dev), rows)
    out = hashes[rows].contiguous()
    torch.cuda.synchronize()
    return out


def events(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--species", type=int, default=50)
    ap.add_argument("--strains", type=int, default=20)
    ap.add_argument("--genome-len", type=int, default=1_000_000)
    ap.add_argument("--reads", type=int, default=10_000_000)
    ap.add_argument("--scale-n", type=int, default=100_000)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--oracle-reads", type=int, default=100_000)
    ap.add_argument("--oracle-threads", type=int, default=16)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert args.species >= SOURCES + 1 and args.scale_n % 10 == 0
    L = _lib.lib()
    _lib.check(L.pg_init(0))
    dev = torch.device("cuda", 0)
    st = torch.cuda.current_stream(dev).cuda_stream
    before = gpu_info()
    sk, pool, p_off, g = make_workload(args, dev, st)
    P, T, n = args.species, args.strains, args.reads
    G = P * T

    def outs(rows):
        return (torch.empty(rows, dtype=torch.int32, device=dev), torch.empty(rows, dtype=torch.float64, device=dev),
                torch.empty(rows, dtype=torch.int64, device=dev))

    def host(d):
        return d[0].cpu().numpy().view(np.uint32), d[1].cpu().numpy(), d[2].cpu().numpy().view(np.uint64)

    res, win = outs(G), outs(G)
    t = {"add": [], "results": [], "winners": []}
    h = C.c_void_p()
    _lib.check(L.pg_mash_screen_create_dev(sk.data_ptr(), G, S, K, st, C.byref(h)))
    try:
        for r in range(args.warmup + args.runs):
            _lib.check(L.pg_mash_screen_reset(h))
            ms_add = events(lambda: _lib.check(L.pg_mash_screen_add_dev(h, pool.data_ptr(), p_off.data_ptr(), n, st)))
            ms_res = events(lambda: _lib.check(L.pg_mash_screen_results_dev(h, *(x.data_ptr() for x in res), st)))
            ms_win = events(lambda: _lib.check(L.pg_mash_screen_winners_dev(h, *(x.data_ptr() for x in win), st)))
            if r >= args.warmup:
                for key, v in (("add", ms_add), ("results", ms_res), ("winners", ms_win)):
                    t[key].append(v)
    finally:
        _lib.check(L.pg_mash_screen_free(h))
    first, got = host(res), host(win)
    tops = [int(np.argmax(got[1][p * T:(p + 1) * T])) for p in range(SOURCES)]
    sources_on_top = tops == [p % T for p in range(SOURCES)]
    src_rows = [p * T + p % T for p in range(SOURCES)]
    present_before = int((first[1] >= 0.5).sum())
    present_after = int((got[1] >= 0.5).sum())
    species_after = sorted({int(i) // T for i in np.nonzero(got[1] >= 0.5)[0]})
    never_more = bool((got[0] <= first[0]).all())

    # scale: 10^8 keys in families of 10
    rows = scale_rows(args, pool, g, dev, st)
    sres, swin = outs(args.scale_n), outs(args.scale_n)
    ts = {"results": [], "winners": []}
    _lib.check(L.pg_mash_screen_create_dev(rows.data_ptr(), args.scale_n, S, K, st, C.byref(h)))
    try:
        _lib.check(L.pg_mash_screen_add_dev(h, pool.data_ptr(), p_off.data_ptr(), n, st))
        for r in range(args.warmup + args.runs):
            ms_res = events(lambda: _lib.check(L.pg_mash_screen_results_dev(h, *(x.data_ptr() for x in sres), st)))
            ms_win = events(lambda: _lib.check(L.pg_mash_screen_winners_dev(h, *(x.data_ptr() for x in swin), st)))
            if r >= args.warmup:
                ts["results"].append(ms_res)
                ts["winners"].append(ms_win)
    finally:
        _lib.check(L.pg_mash_screen_free(h))
    del rows
    s_first, s_got = host(sres), host(swin)
    scale_never_more = bool((s_got[0] <= s_first[0]).all())

    # parity on a sub-pool: every strain of species 0, 1 (present) and the last (absent), against the CPU restatement
    import screen_winners_oracle

    pick = np.concatenate([np.arange(T), np.arange(T, 2 * T), np.arange(G - T, G)])
    sk_sub = np.ascontiguousarray(sk.cpu().numpy().view(np.uint32)[pick])
    nr = min(args.oracle_reads, n)
    sub_bases = pool[: nr * READ_LEN].cpu().numpy()
    sub_off = np.arange(nr + 1, dtype=np.uint64) * READ_LEN
    t0 = time.perf_counter()
    want = screen_winners_oracle.mash_screen_winners(sk_sub, (sub_bases, sub_off), K, nthreads=args.oracle_threads)
    oracle_s = time.perf_counter() - t0
    hs = C.c_void_p()
    _lib.check(L.pg_mash_screen_create(sk_sub.ctypes.data, len(pick), S, K, C.byref(hs)))
    try:
        _lib.check(L.pg_mash_screen_add(hs, sub_bases.ctypes.data, sub_off.ctypes.data, nr))
        sub = np.zeros(len(pick), np.uint32), np.zeros(len(pick), np.float64), np.zeros(len(pick), np.uint64)
        _lib.check(L.pg_mash_screen_winners(hs, *(x.ctypes.data for x in sub)))
    finally:
        _lib.check(L.pg_mash_screen_free(hs))
    parity = all(a.tobytes() == b.tobytes() for a, b in zip(sub, want)) and int(want[0].sum()) > 0
    ok = parity and sources_on_top and never_more and scale_never_more and species_after == list(range(SOURCES))

    med = {key: statistics.median(v) for key, v in t.items()}
    line = {
        "metric": "mash_screen_winners",
        "shape": f"{P} species x {T} strains ({G} references) of {args.genome_len} bp, strains at 0.2-5% substitutions, k={K}, s={S}; "
                 f"pool {n} x {READ_LEN} bp (90% from one strain of each of {SOURCES} species, 1% substitutions)",
        "runs": args.runs, "warmup": args.warmup,
        "add_ms": round(med["add"], 3), "results_ms": round(med["results"], 3), "winners_ms": round(med["winners"], 3),
        "winners_over_results": round(med["winners"] / med["results"], 3),
        "scale_shape": f"{args.scale_n} x {S} synthetic words ({args.scale_n * S} keys), families of 10 sharing 80% of their words",
        "scale_results_ms": round(statistics.median(ts["results"]), 3), "scale_winners_ms": round(statistics.median(ts["winners"]), 3),
        "scale_winners_over_results": round(statistics.median(ts["winners"]) / statistics.median(ts["results"]), 3),
        "all_ms": {key: [round(x, 3) for x in v] for key, v in t.items()},
        "scale_all_ms": {key: [round(x, 3) for x in v] for key, v in ts.items()},
        "sources_on_top": sources_on_top,
        "source_containment_min_results": float(first[1][src_rows].min()), "source_containment_min_winners": float(got[1][src_rows].min()),
        "refs_at_containment_0.5_results": present_before, "refs_at_containment_0.5_winners": present_after,
        "species_at_containment_0.5_winners": len(species_after),
        "sibling_containment_max_winners": float(np.delete(got[1], src_rows).max()),
        "winners_never_exceed_results": never_more and scale_never_more,
        "scale_shared_sum_results": int(s_first[0].astype(np.uint64).sum()), "scale_shared_sum_winners": int(s_got[0].astype(np.uint64).sum()),
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
