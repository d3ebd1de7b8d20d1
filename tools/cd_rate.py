"""Coordinate descent (`solver="cd"`) against the multiplicative updates (`solver="mu"`) at beta 2, both on the fp32 kernels;
prints one JSON line.

    python tools/cd_rate.py [--reps 3] [--mu-iters 200]

Workloads (targets and factors generated on the device from fixed seeds; V = rand, factors rand + 0.1):
  dense_big     65536 x 4096, R = 64 (bench.py's beta-2 shape)
  dense_small   256 x 512, R = 16
  sparse        65536 x 8192 with 0.5 % of the cells stored, R = 64 (a sparse COO target on the sparse kernels)
For each solver, median of --reps:
  it_per_s      iterations per second, counting the iterations alone: 30 / (time of a 60-iteration fit - time of a
                30-iteration fit), tol = -inf;
  time_to_mu_s  wall time of the shortest fit that reaches the loss MU reaches after --mu-iters iterations: MU's own
                --mu-iters fit, and the "cd" fit of the fewest iterations (a multiple of 10) whose loss is at or below it.
The card's name, power limit and maximum SM clock are read in the same run.  Writes nothing.
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

from torchnmf_b200 import NMF  # noqa: E402
from torchnmf_b200.engine import CudaNmfEngine, CudaSparseNmfEngine  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (x.strip() for x in out.split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def target(N, C, density, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    if density is None:
        return torch.rand(N, C, generator=g, device="cuda")
    idx = torch.randint(0, N * C, (int(N * C * density),), generator=g, device="cuda").unique()
    vals = torch.rand(idx.numel(), generator=g, device="cuda")
    return torch.sparse_coo_tensor(torch.stack([idx // C, idx % C]), vals, (N, C)).coalesce()


def factors(N, C, R, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.rand(C, R, generator=g, device="cuda") + 0.1, torch.rand(N, R, generator=g, device="cuda") + 0.1


def fit(V, W0, H0, solver, iters):
    """(seconds, module) of one fit of `iters` iterations from (W0, H0), ended by a device synchronise."""
    m = NMF(W=W0.clone(), H=H0.clone()).cuda()
    torch.cuda.synchronize()
    t = time.perf_counter()
    m.fit(V, 2, float("-inf"), iters, precision="f32", solver=solver)
    torch.cuda.synchronize()
    return time.perf_counter() - t, m


def loss(V, m):
    """1/2 |V - H W^T|^2 of a module's factors, from the library's loss launch."""
    W, H = m.W.data, m.H.data
    eng = CudaSparseNmfEngine(V, W, H) if V.is_sparse else CudaNmfEngine(V, W, H, "f32")
    try:
        return eng.loss(2)
    finally:
        eng.close()


def workload(V, W0, H0, reps, mu_iters):
    out = {}
    for solver in ("cd", "mu"):
        fit(V, W0, H0, solver, 10)                                          # warm-up: modules, workspaces
        rates = []
        for _ in range(reps):
            t30, _ = fit(V, W0, H0, solver, 30)
            t60, _ = fit(V, W0, H0, solver, 60)
            rates.append(30.0 / (t60 - t30))
        out[solver] = {"it_per_s": statistics.median(rates)}
    times = [fit(V, W0, H0, "mu", mu_iters)[0] for _ in range(reps)]
    goal = loss(V, fit(V, W0, H0, "mu", mu_iters)[1])
    out["mu"].update(time_to_mu_s=statistics.median(times), iters_to_mu=mu_iters, loss=goal)
    k = 10
    while k <= mu_iters:
        cur = loss(V, fit(V, W0, H0, "cd", k)[1])
        if cur <= goal:
            break
        k += 10
    if k <= mu_iters:
        times = [fit(V, W0, H0, "cd", k)[0] for _ in range(reps)]
        out["cd"].update(time_to_mu_s=statistics.median(times), iters_to_mu=k, loss=cur)
    else:
        out["cd"].update(time_to_mu_s=None, iters_to_mu=None, loss=cur)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--mu-iters", type=int, default=200)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("cd_rate.py needs a CUDA device")
    res = {"card": card()}
    for name, (N, C, R, density) in {"dense_big": (65536, 4096, 64, None), "dense_small": (256, 512, 16, None),
                                     "sparse": (65536, 8192, 64, 0.005)}.items():
        V = target(N, C, density, seed=1)
        W0, H0 = factors(N, C, R, seed=2)
        res[name] = {"shape": [N, C, R], "density": density, **workload(V, W0, H0, a.reps, a.mu_iters)}
        del V
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
