#!/usr/bin/env python
"""Radius queries of the sketch index at the cfg3 shape; prints one JSON line (profiles/h100_index_within_n1.json).

Workloads: 100k x 10 kbp family reads, k = 31, s = 2000, sketched on the device.  References are the reads with
i % R < 0.9 R, queries the other 10 %; the cut is Distance <= 0.7 (min_same 600).
  (a) R = 100: about 90 references per query's family;
  (b) R = 2000: about 1 800 references per query's family, beyond what the top-k query returns.
Legs, per workload:
  build:   pg_mash_index_create_dev, timed once after a warm-up;
  within:  pg_mash_index_query_within_dev on the 10k queries, into lists sized up front, then a device sync;
  sparse:  the route without the radius query -- pg_mash_distance_sparse_dev over the query rows of [refs; queries]
           (which rebuilds the inverted index over every sketch), then on the device with torch: keep query x
           reference pairs with same >= min_same, sort by (query, ref), build the offsets.
within and sparse are timed alternately, `--runs` times each after a warm-up; medians reported.
Parity: every query's lists equal the sparse route's, and a sample of queries equals the CPU oracle."""
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
sys.path.insert(0, os.path.join(ROOT, "tests"))  # within_oracle: the parity check only
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_query import gpu_info  # noqa: E402
from poly_b200 import _lib, mash, synth  # noqa: E402


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, (time.perf_counter() - t0) * 1e3


def workload(L, dev, n, R, runs, parity_n, max_distance):
    RL, k, s = 10_000, 31, 2000
    st = torch.cuda.current_stream(dev).cuda_stream
    reads = torch.empty(n * RL, dtype=torch.uint8, device=dev)
    _lib.check(L.pg_synth_reads_dev(reads.data_ptr(), 0, n, RL, synth.SEED_READS, 1, R, st))
    sk = torch.empty((n, s), dtype=torch.int32, device=dev)
    _lib.check(L.pg_mash_sketch_uniform_dev(reads.data_ptr(), n, RL, k, s, 0, sk.data_ptr(), s, None, st))
    del reads
    is_ref = torch.arange(n, device=dev) % R < R - R // 10
    refs, queries = sk[is_ref].contiguous(), sk[~is_ref].contiguous()
    nr, nq = refs.shape[0], queries.shape[0]
    cat = torch.cat([refs, queries]).contiguous()
    del sk
    min_same = mash.min_same_for_distance(max_distance, s)

    cap = 32 << 20  # list and triple capacity: about 2e7 query-row triples at R = 2000
    off = torch.empty(nq + 1, dtype=torch.int64, device=dev)
    ref = torch.empty(cap, dtype=torch.int32, device=dev)
    same = torch.empty(cap, dtype=torch.int32, device=dev)
    dist = torch.empty(cap, dtype=torch.float64, device=dev)
    total = torch.zeros((), dtype=torch.int64, device=dev)

    def within(ix):
        _lib.check(L.pg_mash_index_query_within_dev(ix._h, queries.data_ptr(), nq, s, min_same, off.data_ptr(), ref.data_ptr(), same.data_ptr(),
                                                    dist.data_ptr(), cap, total.data_ptr(), st))

    pi = torch.empty(cap, dtype=torch.int32, device=dev)
    pj = torch.empty(cap, dtype=torch.int32, device=dev)
    ps = torch.empty(cap, dtype=torch.int32, device=dev)
    cnt = torch.zeros((), dtype=torch.int64, device=dev)

    def sparse():
        _lib.check(L.pg_mash_distance_sparse_dev(cat.data_ptr(), nr + nq, s, nr, nr + nq, 0, pi.data_ptr(), pj.data_ptr(), ps.data_ptr(), cap,
                                                  cnt.data_ptr(), st))
        m = int(cnt.item())
        assert m <= cap, m
        i, j, c = pi[:m].long() - nr, pj[:m].long(), ps[:m]
        keep = (j < nr) & (c >= min_same)                       # query x reference pairs within the cut
        i, j, c = i[keep], j[keep], c[keep]
        key, order = torch.sort((i << 32) | j)                  # query, then reference ascending
        o = torch.zeros(nq + 1, dtype=torch.int64, device=dev)
        o[1:] = torch.cumsum(torch.bincount(key >> 32, minlength=nq), 0)
        return o, (key & 0xFFFFFFFF).to(torch.int32), c[order]

    ix, _ = timed(lambda: mash.SketchIndex(refs))  # warm-up of every leg
    timed(lambda: within(ix))
    timed(sparse)
    ix.close()
    ix, build_ms = timed(lambda: mash.SketchIndex(refs))
    within_ms, sparse_ms = [], []
    base = None
    for _ in range(runs):
        within_ms.append(timed(lambda: within(ix))[1])
        base, t = timed(sparse)
        sparse_ms.append(t)
    ix.close()
    m = int(total.item())
    assert m <= cap, m
    got = (off.cpu().numpy().view(np.uint64), ref[:m].cpu().numpy().view(np.uint32), same[:m].cpu().numpy().view(np.uint32),
           dist[:m].cpu().numpy())
    b_off, b_ref, b_same = (x.cpu().numpy() for x in base)
    want_dist = 1 - b_same.astype(np.float64) / np.float64(s)  # mash.go:134,139
    sparse_parity = bool(np.array_equal(got[0].astype(np.int64), b_off) and np.array_equal(got[1], b_ref.view(np.uint32))
                         and np.array_equal(got[2], b_same.view(np.uint32)) and got[3].tobytes() == want_dist.tobytes())
    import within_oracle

    sample = np.sort(np.random.default_rng(0).choice(nq, size=min(parity_n, nq), replace=False))
    h_refs = refs.cpu().numpy().view(np.uint32)
    h_q = queries.cpu().numpy().view(np.uint32)[sample]
    t0 = time.perf_counter()
    w_off, w_ref, w_same, w_dist = within_oracle.within(h_refs, h_q, min_same)
    oracle_s = time.perf_counter() - t0
    rows = [np.arange(int(got[0][q]), int(got[0][q + 1])) for q in sample]
    sel = np.concatenate(rows) if rows else np.zeros(0, np.int64)
    g_off = np.zeros(len(sample) + 1, np.uint64)
    g_off[1:] = np.cumsum([len(r) for r in rows])
    oracle_parity = bool(g_off.tobytes() == w_off.tobytes() and got[1][sel].tobytes() == w_ref.tobytes()
                         and got[2][sel].tobytes() == w_same.tobytes() and got[3][sel].tobytes() == w_dist.tobytes())
    lens = np.diff(got[0].astype(np.int64))
    med_w, med_s = statistics.median(within_ms), statistics.median(sparse_ms)
    return {
        "workload": f"cfg3 {n} x {RL} bp family reads R={R}, k={k}, s={s}; refs {nr}, queries {nq}, Distance <= {max_distance} (min_same {min_same})",
        "hits": m, "hits_per_query_min": int(lens.min()), "hits_per_query_median": float(np.median(lens)), "hits_per_query_max": int(lens.max()),
        "index_build_ms": round(build_ms, 2), "within_ms": round(med_w, 2), "sparse_route_ms": round(med_s, 2),
        "speedup_vs_sparse": round(med_s / med_w, 2), "within_ms_all": [round(x, 2) for x in within_ms],
        "sparse_route_ms_all": [round(x, 2) for x in sparse_ms], "parity_vs_sparse_all_queries": sparse_parity,
        "parity_vs_oracle": oracle_parity, "parity_queries": int(len(sample)), "oracle_s": round(oracle_s, 1),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100_000)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--parity", type=int, default=32)
    ap.add_argument("--families", type=int, nargs="+", default=[100, 2000])
    ap.add_argument("--max-distance", type=float, default=0.7)
    args = ap.parse_args()
    L = _lib.lib()
    _lib.check(L.pg_init(0))
    dev = torch.device("cuda", 0)
    res = []
    for R in args.families:
        res.append(workload(L, dev, args.n, R, args.runs, args.parity, args.max_distance))
        torch.cuda.empty_cache()
    line = {
        "metric": "index_within", "runs": args.runs,
        "parity": all(r["parity_vs_sparse_all_queries"] and r["parity_vs_oracle"] for r in res),
        "workloads": res, **gpu_info(),
    }
    print(json.dumps(line))


if __name__ == "__main__":
    main()
