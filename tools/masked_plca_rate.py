"""Iteration rate and peak memory of a masked PLCA fit (`fit(V, ..., mask=M)`) against the unmasked fp32 fit and a
plain-PyTorch fp32 implementation of the same EM on the GPU; one JSON line per workload.

    python tools/masked_plca_rate.py [--rounds 3]

Workloads (seeded inputs generated on the device):
  plca     PLCA 8192 x 4096 R=64, 20 % of the cells missing at random
  siplca   SIPLCA (1, 513, 4096) R=16 T=16, a gap of 10 % of the frames (every channel of frames 1800-2209 missing)
For each workload three fits run alternately, `--rounds` times each, from the same initial factors:
  masked   fit(V, mask=M)                 the masked fp32 kernels: two contraction passes over V and M per iteration
  f32      fit(V, precision="f32")        the unmasked fp32 fit, every cell
  torch    the EM written in PyTorch (fp32, on the GPU): q, the completed target and the ratio P materialised every iteration,
           the gradients by autograd through the reconstruction -- what a user would write without the masked fit
A fit's rate is 30 / (t60 - t30), t_k the device-synchronised time of a k-iteration fit (tol = -inf), so the one-time set-up
cancels; the median over the rounds is reported, with peak torch.cuda.max_memory_allocated of one 30-iteration fit (the
library's own workspace is cudaMalloc'ed outside torch's allocator and not counted there; it is the unmasked fit's plus
one partial slab).  The card's name and power limit are read in the same run.  Writes nothing.
"""
import argparse
import json
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
import torch.nn.functional as F  # noqa: E402

from torchnmf_b200 import PLCA, SIPLCA  # noqa: E402
from torchnmf_b200.constants import eps  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (x.strip() for x in out.split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def workloads():
    g = torch.Generator(device="cuda").manual_seed(0)
    V = torch.rand(8192, 4096, generator=g, device="cuda")
    M = torch.rand(8192, 4096, generator=g, device="cuda") >= 0.2
    yield "plca", (PLCA, dict(rank=64), (8192, 4096)), V, M
    V = torch.rand(1, 513, 4096, generator=g, device="cuda")
    M = torch.ones_like(V, dtype=torch.bool)
    M[..., 1800:2210] = False
    yield "siplca", (SIPLCA, dict(rank=16, T=16), (1, 513, 4096)), V, M


def torch_em(m, V, M, iters):
    """The masked EM in plain PyTorch, fp32: materialise q, the completed target and P; gradients by autograd."""
    W, H, Z = (p.detach().clone().requires_grad_(True) for p in (m.W, m.H, m.Z))
    Vo = torch.where(M, V, torch.zeros((), device=V.device))
    Vn = Vo / Vo.sum()
    for _ in range(iters):
        q = m.reconstruct(H, W, Z)
        with torch.no_grad():
            qo = torch.where(M, q, torch.zeros((), device=q.device)).sum()
            P = torch.where(M, qo * Vn, q) / (q + eps)
        gW, gH, gZ = torch.autograd.grad(q, (W, H, Z), P)
        with torch.no_grad():                                # the reference's updates at alpha = 1 (plca.py:256-288)
            Z.mul_(gZ.relu())
            Z_prior = Z.clone()
            Z.div_(Z.sum())
            over = (slice(None),) + (None,) * (W.dim() - 2)
            W.mul_(gW.relu()).div_(Z_prior[over])
            H.mul_(gH.relu()).div_(Z_prior[(slice(None),) + (None,) * (H.dim() - 2)])
    return W, H, Z


def one(kind, spec, V, M, iters):
    cls, kw, shape = spec
    torch.manual_seed(1)
    m = cls(shape, **kw).cuda()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    if kind == "masked":
        m.fit(V, float("-inf"), iters, mask=M)
    elif kind == "f32":
        m.fit(V, float("-inf"), iters, precision="f32")
    else:
        torch_em(m, V, M, iters)
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    info = card()
    for name, spec, V, M in workloads():
        kinds = ("masked", "f32", "torch")
        for k in kinds:                                      # warm every shape and kernel
            one(k, spec, V, M, 10)
        rates = {k: [] for k in kinds}
        for _ in range(args.rounds):
            for k in kinds:
                t30 = one(k, spec, V, M, 30)
                t60 = one(k, spec, V, M, 60)
                rates[k].append(30.0 / (t60 - t30))
        peak = {}
        for k in kinds:
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            one(k, spec, V, M, 30)
            peak[k] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
        med = {k: statistics.median(v) for k, v in rates.items()}
        print(json.dumps({"workload": name, "card": info, "iters_per_s": {k: round(v, 2) for k, v in med.items()},
                          "rounds": {k: [round(x, 2) for x in v] for k, v in rates.items()},
                          "masked_vs_f32": round(med["masked"] / med["f32"], 3),
                          "masked_vs_torch": round(med["masked"] / med["torch"], 2),
                          "peak_mib_above_inputs": {k: round(v, 1) for k, v in peak.items()}}), flush=True)


if __name__ == "__main__":
    main()
