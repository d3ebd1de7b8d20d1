"""Fit rate of the batch-sharded NMFD fit against the unsharded fit of the same shard, and the cost of its one all-reduce per
W update.  Run it under torchrun, one process per GPU:

    torchrun --nproc_per_node N tools/nmfd_sharded_rate.py [--iters 100] [--warmup 10] [--rounds 2] [--reps 50]

Every rank holds B_local = 4 clips of 1025 x 2048 (bench.py cfg3's channels, R = 16, T = 128) and fits them at beta 1
precision "auto" and at beta 0.5 precision "f32".  Per workload and rank, one JSON line with:
  * sharded_it_s / unsharded_it_s: a timed `fit` of --iters iterations (tol -inf) after a --warmup fit, host clock around a
    device synchronise, with and without `group`; the two alternate, --rounds times each;
  * allreduce_ms: CUDA events around --reps sum-all-reduces, over the same group, of a buffer as long as the W terms
    (nmfb200_raw_terms_numel(which = 0)), i.e. the device time of the W update's exchange;
  * allreduce_bytes_per_iter: the bytes each rank contributes per iteration (the W terms, plus the 8-byte loss every 10th
    iteration).
Rank 0 first prints the card's name, power limit and maximum SM clock.  With --nproc_per_node 1 the group has one rank:
the figures are the protocol's overhead, not scaling.  Writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "pytorch-nmf_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from torchnmf_b200 import NMFD  # noqa: E402
from torchnmf_b200.engine import CudaNmfdEngine, release_workspaces  # noqa: E402

B_LOCAL, C, L, R, T = 4, 1025, 2048, 16, 128
WORKLOADS = [(1.0, "auto"), (0.5, "f32")]          # (beta, precision)


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (x.strip() for x in out.split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def inputs(rank):
    g = torch.Generator(device="cuda").manual_seed(1000 + rank)
    V = torch.rand(B_LOCAL, C, L, generator=g, device="cuda").bfloat16().float()
    W = torch.rand(C, R, T, generator=torch.Generator(device="cuda").manual_seed(7), device="cuda") + 0.1   # one replica
    H = torch.rand(B_LOCAL, R, L - T + 1, generator=g, device="cuda") + 0.1
    return V, W, H


def timed_fit(V, W0, H0, beta, prec, iters, warmup, group):
    release_workspaces()
    NMFD(W=W0, H=H0).cuda().fit(V, beta, float("-inf"), warmup, precision=prec, group=group)
    m = NMFD(W=W0, H=H0).cuda()
    if group is not None:
        dist.barrier(group)
    torch.cuda.synchronize()
    t = time.perf_counter()
    m.fit(V, beta, float("-inf"), iters, precision=prec, group=group)
    torch.cuda.synchronize()
    return iters / (time.perf_counter() - t), m


def allreduce_ms(n, reps, group):
    buf = torch.zeros(n, dtype=torch.float32, device="cuda")
    dist.all_reduce(buf, group=group)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        dist.all_reduce(buf, group=group)
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--backend", default="nccl")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "nmfd_sharded_rate.py measures on CUDA devices"
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    kw = {"device_id": torch.device("cuda", local)} if a.backend == "nccl" else {}
    dist.init_process_group(a.backend, **kw)
    rank, world, group = dist.get_rank(), dist.get_world_size(), dist.group.WORLD
    if rank == 0:
        print(json.dumps({"card": card(), "world": world, "backend": a.backend}), flush=True)
    V, W0, H0 = inputs(rank)
    for beta, prec in WORKLOADS:
        rec = {"rank": rank, "world": world, "beta": beta, "precision": prec, "V_local": [B_LOCAL, C, L], "R": R, "T": T}
        for _ in range(a.rounds):
            for sharded in (True, False):
                rate, m = timed_fit(V, W0, H0, beta, prec, a.iters, a.warmup, group if sharded else None)
                rec.setdefault("sharded_it_s" if sharded else "unsharded_it_s", []).append(round(rate, 2))
                rec["ran" if sharded else "ran_unsharded"] = m.last_fit_precision
        eng = CudaNmfdEngine(V, W0.clone(), H0.clone(), prec)
        n = int(eng._lib.nmfb200_raw_terms_numel(eng._ctx, 0, beta))
        eng.close()
        dist.barrier(group)
        rec["allreduce_ms"] = round(allreduce_ms(n, a.reps, group), 4)
        rec["allreduce_bytes_per_iter"] = 4 * n + 0.8
        print(json.dumps(rec), flush=True)
        release_workspaces()
    dist.barrier(group)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
