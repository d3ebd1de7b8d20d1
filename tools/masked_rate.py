"""Fit rate of a masked fit (`fit(V, ..., mask=M)`) against the unmasked fits and the BetaMu workaround; one JSON line per
workload.

    python tools/masked_rate.py [--iters 50] [--warmup 3] [--rounds 3]

Workloads (30 % of the cells missing at random, seeded inputs generated on the device):
  nmf_b1     NMF 16384 x 4096 R=64 at beta 1
  nmf_b0.5   the same at beta 0.5
  nmfd_b1    NMFD 4 x 1025 x 2048 R=16 T=128 at beta 1
For each workload four fits run alternately, `--rounds` times each, from the same initial factors, every one timed over
`--iters` iterations after a `--warmup` fit of the same shapes (device-synchronised, so a fit's one-time target
registration is included):
  masked      fit(V, beta, mask=M)                      the masked fp32 kernels
  f32         fit(V, beta, precision="f32")             the unmasked fp32 kernels, all cells
  auto        fit(V, beta)                              the unmasked default (tensor cores where they apply)
  betamu      trainer.BetaMu([W, H], beta) with the closure (V[M], model()[M]): the generic autograd route a masked fit
              took before, two backward passes through the materialised reconstruction per factor update
Reported per fit: iterations per second of every round and their median.  The card's name and power limit are read in the
same run.  Writes nothing.
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

from torchnmf_b200 import NMF, NMFD  # noqa: E402
from torchnmf_b200.engine import release_workspaces  # noqa: E402
from torchnmf_b200.trainer import BetaMu  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (x.strip() for x in out.split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def inputs(vshape, wshape, hshape, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    V = torch.rand(*vshape, generator=g, device="cuda")
    W = torch.rand(*wshape, generator=g, device="cuda") + 0.1
    H = torch.rand(*hshape, generator=g, device="cuda") + 0.1
    M = torch.rand(*vshape, generator=g, device="cuda") >= 0.3
    return V, W, H, M


def run(mode, cls, V, M, W0, H0, beta, iters):
    m = cls(W=W0, H=H0).cuda()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    if mode == "betamu":
        opt = BetaMu([m.W, m.H], beta)
        Vo = V[M]

        def closure():
            opt.zero_grad()
            return Vo, m()[M]

        for _ in range(iters):
            opt.step(closure)
    else:
        kw = {"masked": {"mask": M}, "f32": {"precision": "f32"}, "auto": {}}[mode]
        assert m.fit(V, beta, float("-inf"), iters, **kw) == iters
    torch.cuda.synchronize()
    return iters / (time.perf_counter() - t0)


def workload(name, cls, V, W0, H0, M, beta, a):
    modes = ("masked", "f32", "auto", "betamu")
    for mode in modes:                                  # warm-up: module loads, cached workspaces of these shapes
        run(mode, cls, V, M, W0, H0, beta, a.warmup)
    rates = {mode: [] for mode in modes}
    for _ in range(a.rounds):
        for mode in modes:
            rates[mode].append(run(mode, cls, V, M, W0, H0, beta, a.iters))
    med = {mode: statistics.median(r) for mode, r in rates.items()}
    out = {"workload": name, "shape": list(V.shape), "R": W0.shape[1], "beta": beta,
           "missing": round(1 - float(M.float().mean()), 4), "iters": a.iters, "card": a.card,
           "it_per_s": rates, "median_it_per_s": med,
           "masked_over_f32": med["masked"] / med["f32"], "masked_over_betamu": med["masked"] / med["betamu"]}
    release_workspaces()
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("masked_rate.py needs a CUDA device")
    a.card = card()
    N, C, R = 16384, 4096, 64
    V, W, H, M = inputs((N, C), (C, R), (N, R), 0)
    for beta in (1.0, 0.5):
        workload(f"nmf_b{beta:g}", NMF, V, W, H, M, beta, a)
    del V, W, H, M
    B, C, L, R, T = 4, 1025, 2048, 16, 128
    V, W, H, M = inputs((B, C, L), (C, R, T), (B, R, L - T + 1), 1)
    workload("nmfd_b1", NMFD, V, W, H, M, 1.0, a)


if __name__ == "__main__":
    main()
