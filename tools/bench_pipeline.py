#!/usr/bin/env python
"""Multi-GPU pipeline timing (run under torchrun, one rank per GPU):
  A. cfg3 shape sharded over the ranks: K2 sketch of N_total/P long reads per rank -> NCCL
     all-gather of the sketches -> K3 row block (inverted-index join) per rank.
  B. cfg4 shape: K1 sketch of --short-reads reads per rank -> all-gather of the compact
     sketches -> K3 on a capped row block (reference semantics: every pair early-outs).
Times are CUDA events, max over ranks.  One JSON line per stage on rank 0."""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from poly_b200 import _lib, synth  # noqa: E402
from poly_b200.dist import GatheredBuffer, ShardPlan, all_gather_rows, cuda_distance_block, cuda_sketch_uniform, fused_sketch_gather  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--long-reads", type=int, default=100_000)
ap.add_argument("--short-reads", type=int, default=10_000_000, help="per rank")
ap.add_argument("--cap-rows", type=int, default=4096)
ap.add_argument("--cap-cols-per-rank", type=int, default=16384)
args = ap.parse_args()

rank, world, local = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
torch.cuda.set_device(local)
dev = torch.device("cuda", local)
os.environ.setdefault("MASTER_ADDR", "127.0.0.1"); os.environ.setdefault("MASTER_PORT", "29531")
dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
L = _lib.lib(); _lib.check(L.pg_init(local))
st = torch.cuda.current_stream().cuda_stream


def timed(fn):
    dist.barrier(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); out = fn(); e1.record(); torch.cuda.synchronize()
    t = torch.tensor([e0.elapsed_time(e1)], dtype=torch.float64, device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return out, float(t.item())


def report(**kw):
    if rank == 0:
        print(json.dumps(kw), flush=True)


# ---- A: cfg3 sharded -------------------------------------------------------------------
n, RL, k, s = args.long_reads, 10_000, 31, 2000
plan = ShardPlan(n, rank, world)
nl = plan.hi - plan.lo
reads = torch.empty(nl * RL, dtype=torch.uint8, device=dev)
_lib.check(L.pg_synth_reads_dev(reads.data_ptr(), plan.lo, nl, RL, synth.SEED_READS, 1, 100, st))
cuda_sketch_uniform(reads, nl, RL, k, s)  # warm-up
local_sk, t_sk = timed(lambda: cuda_sketch_uniform(reads, nl, RL, k, s))
gathered, t_ag = timed(lambda: all_gather_rows(local_sk, plan))
gathered, t_ag = timed(lambda: all_gather_rows(local_sk, plan))
same, _ = timed(lambda: cuda_distance_block(gathered, plan.lo, plan.hi))  # warm-up: first touch of the output, pool growth
del same
same, t_d = timed(lambda: cuda_distance_block(gathered, plan.lo, plan.hi))
diag = same[torch.arange(nl, device=dev), torch.arange(plan.lo, plan.hi, device=dev)]
ok = bool((diag == s).all().item())
report(stage="A cfg3 sharded", n_gpus=world, reads_total=n, reads_per_rank=nl, sketch_ms=t_sk, allgather_ms=t_ag,
       allgather_GB_recv_per_rank=(n - nl) * s * 4 / 1e9, distance_rowblock_ms=t_d, pairs_total=n * n, diag_ok=ok,
       family_mean_row0=float(same[0, plan.lo + 1: plan.lo + 100].float().mean().item()))
del same, gathered, local_sk, reads
torch.cuda.empty_cache()

# ---- B: cfg4 shape -----------------------------------------------------------------------
m, SL, k, s = args.short_reads, 150, 21, 1000
reads = torch.empty(m * SL, dtype=torch.uint8, device=dev)
_lib.check(L.pg_synth_reads_dev(reads.data_ptr(), rank * m, m, SL, synth.SEED_READS, 0, 0, st))
cuda_sketch_uniform(reads, m, SL, k, s)
local_sk, t_sk = timed(lambda: cuda_sketch_uniform(reads, m, SL, k, s))
plan = ShardPlan(m * world, rank, world)
gathered, t_ag = timed(lambda: all_gather_rows(local_sk, plan))
nk = local_sk.shape[1]
# capped subset: first cap-cols-per-rank sketches of every rank, padded to full Go arrays (zero tail)
cols = min(args.cap_cols_per_rank, m)
sub = torch.zeros((cols * world, s), dtype=torch.int32, device=dev)
for r in range(world):
    sub[r * cols:(r + 1) * cols, :nk] = gathered[r * m: r * m + cols]
rows = min(args.cap_rows, cols)
same, t_d = timed(lambda: cuda_distance_block(sub, rank * cols, rank * cols + rows))
report(stage="B cfg4 shape", n_gpus=world, reads_per_rank=m, sketch_ms=t_sk, sketch_gbases_per_s_total=world * m * SL / t_sk / 1e6,
       allgather_ms=t_ag, allgather_GB_recv_per_rank=(world - 1) * m * nk * 4 / 1e9,
       allgather_GBps_per_rank=(world - 1) * m * nk * 4 / t_ag / 1e6, capped_rows=rows, capped_cols=cols * world, distance_ms=t_d,
       max_same=int(same.max().item()), note="reference semantics: n=129 < s=1000 -> zero-padded unsorted sketches -> every pair early-outs (distance 1.0)")
# rows of the NCCL result the fused buffer is checked against; a full gathered copy is world x m x 129 x 4 B
# (41.3 GB at 8 ranks of 10 M reads), so it is freed before the fused buffer is allocated: one copy at a time
ref_rows = {r: gathered[r * m: r * m + 4096].clone() for r in (0, world - 1)}
del same, sub, gathered
# ---- C: the same exchange fused into the sketch kernel (TMA bulk stores to peer memory) -------
torch.cuda.empty_cache()
buf = GatheredBuffer(plan, nk)


def fused():
    fused_sketch_gather(reads, SL, k, s, buf, sync=False)


fused(); torch.cuda.synchronize(); dist.barrier()
_, t_f = timed(fused)
_, t_f2 = timed(fused)
# verify against the NCCL all-gather result (rows of the LAST rank and of rank 0)
got = buf.as_tensor()
ok = all(bool(torch.equal(got[r * m: r * m + 4096], ref_rows[r])) for r in ref_rows)
report(stage="C cfg4 fused sketch+gather (peer stores)", n_gpus=world, reads_per_rank=m, fused_ms=min(t_f, t_f2), separate_ms=t_sk + t_ag,
       bytes_out_per_rank_GB=(world - 1) * m * nk * 4 / 1e9, nvlink_GBps_out_per_rank=(world - 1) * m * nk * 4 / min(t_f, t_f2) / 1e6,
       matches_allgather=ok)
del got
buf.close()
dist.destroy_process_group()
