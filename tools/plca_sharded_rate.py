"""Iteration rate of the sharded PLCA / SIPLCA fits (`fit(..., group=...)`) against the unsharded fit of the same shard, and
the cost of the one all-reduce of [dW | dZ] per EM step.  Run it under torchrun, one process per GPU:

    torchrun --nproc_per_node N tools/plca_sharded_rate.py [--rounds 3] [--reps 50]

Per rank (seeded targets generated on the device, each rank its own shard; W and Z one replica):
  plca_dense   PLCA, 8192 x 4096 dense, R = 64, precision "f32"
  siplca       SIPLCA, 4 clips of 513 x 4096, R = 16, T = 16, precision "f32"
  plsa_sparse  PLCA on a sparse COO target, 262144 documents x 65536 terms, 200 stored entries per document (52 M;
               Poisson-like counts 1-5, duplicates summed), R = 100
One JSON line per workload and rank with:
  * sharded_it_s / unsharded_it_s: 30 / (t60 - t30), t_k the device-synchronised time of a k-iteration fit (tol = -inf)
    from the same initial factors, so the one-time set-up cancels; the median over --rounds rounds, sharded and unsharded
    alternating within each round (every round's rates are listed too);
  * allreduce_ms: CUDA events around --reps sum-all-reduces, over the same group, of one fp32 buffer of C R prod(K) + R
    floats, the length of the EM step's exchange, per all-reduce.
Rank 0 first prints the card's name, power limit and maximum SM clock.  With --nproc_per_node 1 the group has one rank:
the figures are the protocol's overhead, not scaling.  Writes nothing.
"""
import argparse
import gc
import json
import math
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "pytorch-nmf_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from torchnmf_b200 import PLCA, SIPLCA  # noqa: E402
from torchnmf_b200.engine import release_workspaces  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (x.strip() for x in out.split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def plsa(N, C, per_doc, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    rows = torch.arange(N, device="cuda").repeat_interleave(per_doc)
    cols = torch.randint(0, C, (rows.numel(),), device="cuda", generator=g)
    vals = torch.randint(1, 6, (rows.numel(),), device="cuda", generator=g).float()
    return torch.sparse_coo_tensor(torch.stack([rows, cols]), vals, (N, C)).coalesce()


def workloads(rank):
    """(name, model class, V, W shape, H shape, precision) of this rank's shard."""
    g = torch.Generator(device="cuda").manual_seed(1000 + rank)
    yield "plca_dense", PLCA, torch.rand(8192, 4096, device="cuda", generator=g), (4096, 64), (8192, 64), "f32"
    yield "siplca", SIPLCA, torch.rand(4, 513, 4096, device="cuda", generator=g), (513, 16, 16), (4, 16, 4096 - 16 + 1), "f32"
    yield "plsa_sparse", PLCA, plsa(262144, 65536, 200, 2000 + rank), (65536, 100), (262144, 100), "f32"


def factors(ws, hs, rank):
    W = torch.rand(ws, device="cuda", generator=torch.Generator(device="cuda").manual_seed(7)) + 0.1     # one replica
    H = torch.rand(hs, device="cuda", generator=torch.Generator(device="cuda").manual_seed(3000 + rank)) + 0.1
    return W, H


def timed_fit(cls, V, W0, H0, prec, iters, group):
    R = W0.shape[1]
    m = cls(W=W0, H=H0, Z=torch.full((R,), 1.0 / R)).cuda()
    gc.collect()                  # the previous fit's engine frees its context here, not inside the timed fit
    if group is not None:
        dist.barrier(group)
    torch.cuda.synchronize()
    t = time.perf_counter()
    m.fit(V, float("-inf"), iters, precision=prec, group=group)
    torch.cuda.synchronize()
    return time.perf_counter() - t


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
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--backend", default="nccl")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "plca_sharded_rate.py measures on CUDA devices"
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    kw = {"device_id": torch.device("cuda", local)} if a.backend == "nccl" else {}
    dist.init_process_group(a.backend, **kw)
    rank, world, group = dist.get_rank(), dist.get_world_size(), dist.group.WORLD
    if rank == 0:
        print(json.dumps({"card": card(), "world": world, "backend": a.backend}), flush=True)
    for name, cls, V, ws, hs, prec in workloads(rank):
        W0, H0 = factors(ws, hs, rank)
        for sharded in (True, False):                    # warm every shape and kernel
            timed_fit(cls, V, W0, H0, prec, 10, group if sharded else None)
        rates = {"sharded": [], "unsharded": []}
        for _ in range(a.rounds):
            for sharded in (True, False):
                g = group if sharded else None
                t30 = timed_fit(cls, V, W0, H0, prec, 30, g)
                t60 = timed_fit(cls, V, W0, H0, prec, 60, g)
                rates["sharded" if sharded else "unsharded"].append(30.0 / (t60 - t30))
        n = math.prod(ws) + ws[1]                        # [dW | dZ]: C R prod(K) + R floats
        dist.barrier(group)
        rec = {"workload": name, "rank": rank, "world": world, "V_local": list(V.shape), "W": list(ws), "precision": prec,
               "sharded_it_s": round(statistics.median(rates["sharded"]), 2),
               "unsharded_it_s": round(statistics.median(rates["unsharded"]), 2),
               "rounds": {k: [round(x, 2) for x in v] for k, v in rates.items()},
               "allreduce_floats": n, "allreduce_ms": round(allreduce_ms(n, a.reps, group), 4)}
        if V.is_sparse:
            rec["nnz_local"] = int(V._nnz())
        print(json.dumps(rec), flush=True)
        del V, W0, H0
        release_workspaces()
    dist.barrier(group)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
