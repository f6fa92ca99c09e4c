"""Times the pipelined host sketch path on a ragged batch: pg_mash_sketch_batch with pinned and with pageable
buffers, and mash.sketch_into (PG_SKETCH_TAIL_KEEP into a caller-zeroed pageable [n, s] array).  Prints one
JSON line: per mode the median, min and max call time over --reps calls after one warm-up, and the SHA-256 of
the outputs, so that two builds of the library can be compared for speed and for identical results.

    python tools/bench_sketch_host.py [--reads 10000000] [--into-reads 2000000] [--reps 5]
"""
import argparse
import hashlib
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from poly_b200 import _lib, mash  # noqa: E402


def sha(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(memoryview(np.ascontiguousarray(a)).cast("B"))
    return h.hexdigest()[:16]


def timed(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()  # synchronous: returns when every row is in host memory
        ts.append(time.perf_counter() - t0)
    return {"median_ms": 1e3 * float(np.median(ts)), "min_ms": 1e3 * min(ts), "max_ms": 1e3 * max(ts)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=10_000_000)
    ap.add_argument("--into-reads", type=int, default=2_000_000)
    ap.add_argument("--min-len", type=int, default=100)
    ap.add_argument("--max-len", type=int, default=200)
    ap.add_argument("--k", type=int, default=21)
    ap.add_argument("--s", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--seed", type=int, default=1)
    a = ap.parse_args()
    L = _lib.lib()
    _lib.check(L.pg_init(0))
    rng = np.random.default_rng(a.seed)
    lens = rng.integers(a.min_len, a.max_len + 1, a.reads)
    off = np.zeros(a.reads + 1, np.uint64)
    off[1:] = np.cumsum(lens)
    bases = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, int(off[-1]), dtype=np.uint8)]
    n, k, s = a.reads, a.k, a.s
    stride = min(int(lens.max()) - k, s)
    count = np.zeros(n, np.uint32)
    status = np.zeros(n, np.int32)
    res = {"reads": n, "bases": int(off[-1]), "k": k, "s": s, "row_stride": stride}

    def batch(src, out):
        _lib.check(L.pg_mash_sketch_batch(src.ctypes.data, off.ctypes.data, n, k, s, 0, out.ctypes.data, stride,
                                          count.ctypes.data, status.ctypes.data))

    p_in = torch.empty(len(bases), dtype=torch.uint8, pin_memory=True).numpy()
    p_in[:] = bases
    p_out = torch.empty(n * stride, dtype=torch.int32, pin_memory=True).numpy().view(np.uint32)
    res["batch_pinned"] = timed(lambda: batch(p_in, p_out), a.reps)
    res["batch_pinned"]["sha256"] = sha(p_out, count, status)
    del p_in, p_out
    out = np.empty(n * stride, np.uint32)
    res["batch_pageable"] = timed(lambda: batch(bases, out), a.reps)
    res["batch_pageable"]["sha256"] = sha(out, count, status)
    del out

    m = min(n, a.into_reads)
    sub_off = off[: m + 1]
    sketches = np.zeros((m, s), np.uint32)  # zeroed outside the timed calls, as Go's make hands it out
    res["sketch_into_reads"] = m
    res["sketch_into_tail_keep_pageable"] = timed(lambda: mash.sketch_into(bases, sub_off, k, s, sketches), a.reps)
    res["sketch_into_tail_keep_pageable"]["sha256"] = sha(sketches)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
