#!/usr/bin/env python
"""Top-k query throughput of the sketch index at the cfg3 shape; prints one JSON line
(profiles/h100_index_query_n1.json).

Workload: 100k x 10 kbp family reads (R = 100), k = 31, s = 2000, sketched on the device.  References are the
90k reads with i % 100 < 90, queries the other 10k; top_k = 10, min_same = 1.
  index:    pg_mash_index_create_dev once (timed as the build), then pg_mash_index_query_dev on the 10k batch.
  sparse:   the same question without the index -- pg_mash_distance_sparse_dev over the query rows of the
            concatenated [refs; queries] set (which rebuilds the inverted index over all 100k sketches), then a
            device-side ranking of the (i, j, same) triples with torch: drop query x query pairs, sort by
            (query, -same, ref), keep the first 10 of each query.
The two are timed alternately, `--runs` times each, medians reported.  Parity: the index's results for 64
sampled queries equal the brute-force oracle ranking, and all 10k equal the sparse route's ranking."""
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
sys.path.insert(0, os.path.join(ROOT, "tests"))  # index_oracle: the parity check only
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
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--parity", type=int, default=64)
    args = ap.parse_args()
    n, RL, k, s, R, top_k = args.n, 10_000, 31, 2000, 100, 10
    L = _lib.lib()
    _lib.check(L.pg_init(0))
    dev = torch.device("cuda", 0)
    st = torch.cuda.current_stream(dev).cuda_stream
    reads = torch.empty(n * RL, dtype=torch.uint8, device=dev)
    _lib.check(L.pg_synth_reads_dev(reads.data_ptr(), 0, n, RL, synth.SEED_READS, 1, R, st))
    sk = torch.empty((n, s), dtype=torch.int32, device=dev)
    _lib.check(L.pg_mash_sketch_uniform_dev(reads.data_ptr(), n, RL, k, s, 0, sk.data_ptr(), s, None, st))
    del reads
    idx = torch.arange(n, device=dev)
    is_ref = idx % R < R - R // 10
    refs, queries = sk[is_ref].contiguous(), sk[~is_ref].contiguous()
    nr, nq = refs.shape[0], queries.shape[0]
    cat = torch.cat([refs, queries]).contiguous()
    del sk
    torch.cuda.synchronize()

    def build():
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ix = mash.SketchIndex(refs)
        torch.cuda.synchronize()
        return ix, (time.perf_counter() - t0) * 1e3

    def query(ix):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = ix.nearest(queries, top_k, min_same=1)
        torch.cuda.synchronize()
        return res, (time.perf_counter() - t0) * 1e3

    cap = 64 << 20
    pi = torch.empty(cap, dtype=torch.int32, device=dev)
    pj = torch.empty(cap, dtype=torch.int32, device=dev)
    ps = torch.empty(cap, dtype=torch.int32, device=dev)
    cnt = torch.zeros(1, dtype=torch.int64, device=dev)

    def sparse():
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        _lib.check(L.pg_mash_distance_sparse_dev(cat.data_ptr(), nr + nq, s, nr, nr + nq, 0, pi.data_ptr(), pj.data_ptr(), ps.data_ptr(), cap,
                                                  cnt.data_ptr(), st))
        m = int(cnt.item())
        assert m <= cap, m
        i, j, c = pi[:m].long() - nr, pj[:m].long(), ps[:m].long()
        keep = j < nr                                           # query x reference pairs only
        i, j, c = i[keep], j[keep], c[keep]
        key = (i << 40) | ((s - c) << 20) | j                   # query, same descending, ref ascending
        key, _ = torch.sort(key)
        qi = key >> 40
        first = torch.searchsorted(key, qi << 40)               # start of each query's group
        sel = (torch.arange(len(key), device=dev) - first) < top_k
        key = key[sel]
        qi, rank_pos = key >> 40, (torch.arange(len(key), device=dev) - torch.searchsorted(key, (key >> 40) << 40))
        ref = torch.full((nq, top_k), -1, dtype=torch.int64, device=dev)
        same = torch.zeros((nq, top_k), dtype=torch.int64, device=dev)
        ref[qi, rank_pos] = key & ((1 << 20) - 1)
        same[qi, rank_pos] = s - ((key >> 20) & ((1 << 20) - 1))
        torch.cuda.synchronize()
        return (ref, same), (time.perf_counter() - t0) * 1e3

    # warm-up of every shape
    ix, _ = build()
    query(ix)
    sparse()
    ix.close()
    build_ms, query_ms, sparse_ms = [], [], []
    res = base = None
    for _ in range(args.runs):
        ix, b = build()
        build_ms.append(b)
        res, q = query(ix)
        query_ms.append(q)
        ix.close()
        base, t = sparse()
        sparse_ms.append(t)
    ref, same, dist, nh = (x.cpu().numpy().view(np.uint32) if x.dtype == torch.int32 else x.cpu().numpy() for x in res)
    b_ref = base[0].cpu().numpy().astype(np.int64)
    b_same = base[1].cpu().numpy().astype(np.int64)
    ref_i64 = np.where(ref == mash.NO_REF, -1, ref.astype(np.int64))
    sparse_parity = bool(np.array_equal(ref_i64, b_ref) and np.array_equal(same.astype(np.int64), b_same))
    # oracle parity on sampled queries
    import index_oracle

    rng = np.random.default_rng(0)
    sample = np.sort(rng.choice(nq, size=min(args.parity, nq), replace=False))
    h_refs = refs.cpu().numpy().view(np.uint32)
    h_q = queries.cpu().numpy().view(np.uint32)[sample]
    t0 = time.perf_counter()
    want = index_oracle.nearest(h_refs, h_q, top_k, 1)
    oracle_s = time.perf_counter() - t0
    got = (ref[sample], same[sample], dist[sample], nh[sample])
    parity = all(np.asarray(g).tobytes() == np.ascontiguousarray(w).tobytes() for g, w in zip(got, want))
    med_q = statistics.median(query_ms)
    line = {
        "metric": "index_query", "workload": f"cfg3 {n} x {RL} bp family reads R={R}, k={k}, s={s}; refs {nr}, queries {nq}, top_k={top_k}, min_same=1",
        "index_build_ms": round(statistics.median(build_ms), 2), "query_ms": round(med_q, 2), "queries_per_s": round(nq / (med_q / 1e3), 1),
        "sparse_rank_ms": round(statistics.median(sparse_ms), 2), "speedup_vs_sparse": round(statistics.median(sparse_ms) / med_q, 2),
        "runs": args.runs, "build_ms_all": [round(x, 2) for x in build_ms], "query_ms_all": [round(x, 2) for x in query_ms],
        "sparse_rank_ms_all": [round(x, 2) for x in sparse_ms], "parity": bool(parity), "parity_queries": int(len(sample)),
        "parity_vs_sparse_all_queries": sparse_parity, "oracle_s": round(oracle_s, 1), **gpu_info(),
    }
    print(json.dumps(line))


if __name__ == "__main__":
    main()
