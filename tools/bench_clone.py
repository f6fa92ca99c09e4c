#!/usr/bin/env python
"""Clone throughput: a digest screen and one combinatorial Golden Gate library; prints one JSON line
(profiles/h100_clone_n1.json).

  digest  --parts x --len bp parts (pg_synth_reads_dev, seeded; every other part circular) cut with the three
          base enzymes (directional), through pg_clone_digest_batch in batches of --batch parts.  Reported:
          input GB/s of the whole host call (upload, kernels, copy-back) and of the digest kernels alone
          (torch.profiler, separate untimed pass) against the 3.35 TB/s HBM3 data-sheet bound.  CPU arm: the C
          restatement (tests/clone_oracle.c) on every schedulable core over a prefix of the parts.
  golden  a backbone + --positions x --variants parts (tests/clone_util.combinatorial_library): variants **
          positions clones.  Timed: digest (pg_clone_digest_batch on the same parts); digest + enumeration that
          only counts (a call with zero caps stops there: it stores no recipes); and the full call.  The rest of
          the full call is recipe storage, ligation, seqhash, dedup and copy-back; of it, the ligation
          (clone_pieces_kernel) and seqhash kernel times come from torch.profiler, the remainder is host work.
Parity: a sample of digest items against the C restatement, and a sample of clones against the constructs
the library design predicts, with their digests against the C seqhash.  The card's name and power limit are
read in the same run."""
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
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))  # oracle and generators: parity and the CPU arm only
from poly_b200 import _lib, clone, synth  # noqa: E402
import clone_oracle  # noqa: E402
import clone_util  # noqa: E402
import seqhash_oracle  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_seqhash import gpu_info  # noqa: E402

HBM_TBPS = 3.35


def kernel_ms(fn, names):
    """Summed device time (ms) of kernels whose name contains any of names, over one call of fn."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    tot = {n: 0.0 for n in names}
    for ev in prof.key_averages():
        for n in names:
            if n in ev.key:
                tot[n] += ev.device_time_total / 1e3 if hasattr(ev, "device_time_total") else ev.cuda_time_total / 1e3
    return tot


def digest_call(seqs, off, circ, enz, ne, directional, caps):
    L = _lib.lib()
    n = len(off) - 1
    cnt, st = np.zeros(n * ne, np.uint32), np.zeros(n * ne, np.int32)
    nf, ns, no = C.c_uint64(), C.c_uint64(), C.c_uint64()
    fcap, scap, ocap = caps
    sb, so = np.empty(max(scap, 1), np.uint8), np.empty(fcap + 1, np.uint64)
    ob, oo = np.empty(max(ocap, 1), np.uint8), np.empty(2 * fcap + 1, np.uint64)
    rc = L.pg_clone_digest_batch(_lib.ptr(seqs), _lib.ptr(off), _lib.ptr(circ), n, C.cast(enz, C.c_void_p), ne, int(directional), _lib.ptr(cnt),
                                 _lib.ptr(st), _lib.ptr(sb), scap, _lib.ptr(so), _lib.ptr(ob), ocap, _lib.ptr(oo), fcap, C.byref(nf), C.byref(ns),
                                 C.byref(no))
    return rc, (nf.value, ns.value, no.value), cnt, st, sb, so, ob, oo


def bench_digest(args, dev):
    enzymes = clone.GetBaseRestrictionEnzymes()
    enz, keep = clone._enzymes(enzymes)
    ne, L, B = len(enzymes), args.len, args.batch
    st_ = torch.cuda.current_stream().cuda_stream
    batches = []
    for b in range(0, args.parts, B):
        n = min(B, args.parts - b)
        d = torch.empty(n * L, dtype=torch.uint8, device=dev)
        _lib.check(_lib.lib().pg_synth_reads_dev(d.data_ptr(), b, n, L, synth.SEED_READS, 0, 0, st_))
        torch.cuda.synchronize()
        seqs = d.cpu().numpy()
        off = np.arange(n + 1, dtype=np.uint64) * L
        circ = (np.arange(b, b + n) % 2).astype(np.uint8)
        batches.append((seqs, off, circ))
    caps = []
    for seqs, off, circ in batches:  # sizes of the outputs (untimed)
        rc, need, *_ = digest_call(seqs, off, circ, enz, ne, True, (0, 0, 0))
        caps.append(need)
    times = []
    for _ in range(args.runs):
        t0 = time.perf_counter()
        for (seqs, off, circ), cap in zip(batches, caps):
            rc, need, cnt, st, *_ = digest_call(seqs, off, circ, enz, ne, True, cap)
            assert rc in (_lib.PG_OK, _lib.PG_ERR_PANIC), rc
        times.append(time.perf_counter() - t0)
    total_bytes = args.parts * L
    ks = kernel_ms(lambda: [digest_call(s, o, c, enz, ne, True, cap) for (s, o, c), cap in zip(batches, caps)],
                   ["clone_sites_kernel", "clone_fragments_kernel", "clone_offsets_kernel", "clone_copy_kernel", "DeviceScan"])
    kernel_total = sum(ks.values())
    # parity: a sample of items of the first batch
    seqs, off, circ = batches[0]
    rc, need, cnt, st, sb, so, ob, oo = digest_call(seqs, off, circ, enz, ne, True, caps[0])
    first = np.zeros(len(cnt) + 1, np.int64)
    np.cumsum(cnt, out=first[1:])
    rng = np.random.default_rng(1)
    sample = rng.choice(len(cnt), size=min(600, len(cnt)), replace=False)
    frags_seen = 0
    for i in sample:
        p, e = divmod(int(i), ne)
        part = seqs[int(off[p]): int(off[p + 1])].tobytes()
        wrc, want = clone_oracle.cut(part, bool(circ[p]), True, enzymes[e].Name)
        got = [(sb[so[f]: so[f + 1]].tobytes(), ob[oo[2 * f]: oo[2 * f + 1]].tobytes(), ob[oo[2 * f + 1]: oo[2 * f + 2]].tobytes())
               for f in range(first[i], first[i + 1])]
        assert wrc == st[i] and got == want, ("digest parity", p, e)
        frags_seen += len(want)
    # CPU arm
    cores = len(os.sched_getaffinity(0))
    n_cpu = min(args.cpu_parts, len(off) - 1)
    t0 = time.perf_counter()
    clone_oracle.cut_counts(seqs[: n_cpu * L], off[: n_cpu + 1], circ[:n_cpu], [e.Name for e in enzymes], True, cores)
    cpu_s = time.perf_counter() - t0
    med = statistics.median(times)
    del keep
    return {
        "parts": args.parts, "part_len": L, "enzymes": [e.Name for e in enzymes], "directional": True, "batch_parts": B,
        "call_s_median": med, "call_s_runs": times, "input_gbps_call": total_bytes / med / 1e9,
        "kernel_ms": ks, "input_gbps_kernels": total_bytes / (kernel_total / 1e3) / 1e9,
        "kernel_fraction_of_hbm_bound": (total_bytes / (kernel_total / 1e3)) / (HBM_TBPS * 1e12),
        "fragments_per_batch": caps[0][0], "parity_items": len(sample), "parity_fragments": frags_seen,
        "cpu_arm": {"impl": "C restatement (tests/clone_oracle.c), not Go", "threads": cores, "parts": n_cpu,
                    "input_gbps": n_cpu * L / cpu_s / 1e9},
    }


def bench_golden(args):
    parts, want = clone_util.combinatorial_library(args.positions, args.variants, args.insert, args.backbone, seed=3)
    seqs = [p for p, _ in parts]
    off = np.zeros(len(parts) + 1, np.uint64)
    off[1:] = np.cumsum([len(s) for s in seqs])
    data = np.frombuffer(b"".join(seqs), np.uint8)
    circ = np.array([c for _, c in parts], np.uint8)
    roff = np.array([0, len(parts)], np.uint64)
    enz, keep = clone._enzymes([clone.GetBaseRestrictionEnzymes()[0]])
    L = _lib.lib()
    nb, nc = C.c_uint64(), C.c_uint64()
    bufs = {}

    def gg(bcap, ccap):
        if (bcap, ccap) not in bufs:
            bufs.clear()
            bufs[(bcap, ccap)] = (np.zeros(max(bcap, 1), np.uint8), np.zeros(ccap + 1, np.uint64), np.zeros(max(ccap, 1), np.uint8),
                                  np.zeros((max(ccap, 1), 32), np.uint8))
        out, coff, kinds, dig = bufs[(bcap, ccap)]
        counts, st = np.zeros(2, np.uint64), np.zeros(1, np.int32)
        rc = L.pg_clone_golden_gate_batch(_lib.ptr(data), _lib.ptr(off), _lib.ptr(circ), len(parts), _lib.ptr(roff), 1, C.cast(enz, C.c_void_p), bcap,
                                          ccap, _lib.ptr(out), _lib.ptr(coff), _lib.ptr(kinds), _lib.ptr(dig), _lib.ptr(counts), _lib.ptr(st),
                                          C.byref(nb), C.byref(nc))
        return rc, out, coff, kinds, dig, counts

    rc, *_ = gg(0, 0)
    need_b, need_c = nb.value, nc.value
    assert rc == _lib.PG_ERR_ARG
    gg(need_b, need_c)  # warm-up, buffers touched
    t_digest, t_enum, t_full = [], [], []
    for _ in range(args.runs):
        t0 = time.perf_counter()
        digest_call(data, off, circ, enz, 1, True, (0, 0, 0))
        t_digest.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        gg(0, 0)
        t_enum.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        rc, out, coff, kinds, dig, counts = gg(need_b, need_c)
        t_full.append(time.perf_counter() - t0)
        assert rc == _lib.PG_OK
    ks = kernel_ms(lambda: gg(need_b, need_c), ["clone_pieces_kernel", "seqhash", "blake3", "clone_sites", "clone_fragments", "clone_copy"])
    n_clones = int(counts[0])
    assert n_clones == want, (n_clones, want)
    # parity: the backbone seed closes every clone first, in the order of the variant choices
    frags = []
    for s, c in parts:
        frags += clone_oracle.cut(s, c, True, "BsaI")[1]
    n_bb = len(clone_oracle.cut(parts[0][0], parts[0][1], True, "BsaI")[1])  # a circular part may give its fragment twice
    bb, var = frags[0], frags[n_bb:]
    rng = np.random.default_rng(2)
    sample = sorted(set(rng.choice(n_clones, size=min(200, n_clones), replace=False).tolist()) | {0, n_clones - 1})
    for k in sample:
        digits, x = [], k
        for _ in range(args.positions):
            digits.append(x % args.variants)
            x //= args.variants
        digits.reverse()
        want_seq = bb[1] + bb[0]
        for i, d in enumerate(digits):
            f = var[i * args.variants + d]
            want_seq += f[1] + f[0]
        got = out[coff[k]: coff[k + 1]].tobytes()
        assert kinds[k] == 0 and got == want_seq, ("clone parity", k)
        assert seqhash_oracle.seqhash(got, "DNA", True, True)[1] == dig[k].tobytes()
    md, me, mf = statistics.median(t_digest), statistics.median(t_enum), statistics.median(t_full)
    lig_ms = ks["clone_pieces_kernel"]
    hash_ms = ks["seqhash"] + ks["blake3"]
    del keep
    return {
        "positions": args.positions, "variants": args.variants, "clones": n_clones, "loops": int(counts[1]),
        "clone_len_mean": float(np.mean(np.diff(coff[: n_clones + 1].astype(np.int64)))),
        "emitted_constructs": need_c, "emitted_bytes": need_b,
        "s_median": {"digest": md, "digest_plus_counting_enumeration": me, "full": mf},
        "split_s": {"digest": md, "enumeration_counting_only": me - md, "recipes_ligation_seqhash_dedup_copyback": mf - me},
        "kernel_ms": ks, "ligation_kernel_ms": lig_ms, "seqhash_kernel_ms": hash_ms,
        "host_share_of_rest_s": (mf - me) - (lig_ms + hash_ms) / 1e3,
        "emitted_gbps": need_b / (mf - me) / 1e9,
        "parity_clones": len(sample),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parts", type=int, default=1_000_000)
    ap.add_argument("--len", type=int, default=5000)
    ap.add_argument("--batch", type=int, default=100_000)
    ap.add_argument("--cpu-parts", type=int, default=20_000)
    ap.add_argument("--positions", type=int, default=5)
    ap.add_argument("--variants", type=int, default=10)
    ap.add_argument("--insert", type=int, default=700)
    ap.add_argument("--backbone", type=int, default=1400)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    _lib.check(_lib.lib().pg_init(0))
    rec = {"bench": "clone", **gpu_info(), "hbm_tbps_datasheet": HBM_TBPS}
    rec["digest"] = bench_digest(args, dev)
    rec["golden_gate"] = bench_golden(args)
    line = json.dumps(rec)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
