"""Coordinate descent (`solver="cd"`) against the multiplicative updates (`solver="mu"`) at beta 2 on the observed cells of a
sparse mask (`NMF.fit(V, 2, ..., mask=M)`); prints one JSON line.

    python tools/observed_cd_rate.py [--reps 3] [--mu-iters 200]

Workloads (generated on the device from fixed seeds; V's stored entries are exactly the observed cells, the mask stores True
there; factors rand + 0.1):
  uniform_64    65536 x 8192, 0.5 % of the cells observed uniformly at random, R = 64 (two 32-component groups: the
                residual workspace is in play)
  uniform_32    262144 x 131072, 0.01 % observed uniformly, R = 32 (one group)
  zipf_32       ratings-like: 200000 users x 50000 items, 5 M draws of (user, item) with item popularity Zipf (exponent 1)
                and users uniform, repeats collapsed, ratings in 1 .. 5, R = 32.  The most popular item takes about 9 %
                of the draws, so its column holds ~10^5 cells while the mean column holds ~100 (the output reports both)
For each solver, median of --reps:
  it_per_s      iterations per second, counting the iterations alone: 30 / (time of a 60-iteration fit - time of a
                30-iteration fit), tol = -inf;
  time_to_mu_s  wall time of the shortest fit that reaches the observed loss MU reaches after --mu-iters iterations: MU's own
                --mu-iters fit, and the "cd" fit of the fewest iterations (a multiple of 10) whose loss is at or below it.
Every fit's wall time includes building the observed set from the mask (the same work for both solvers).  The card's
name, power limit and maximum SM clock are read in the same run.  Writes nothing.
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
from torchnmf_b200.engine import CudaObservedNmfEngine  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (x.strip() for x in out.split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def uniform(N, C, density, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    lin = torch.randint(0, N * C, (int(N * C * density),), generator=g, device="cuda").unique()
    vals = torch.rand(lin.numel(), generator=g, device="cuda") + 1e-3
    return torch.sparse_coo_tensor(torch.stack([lin // C, lin % C]), vals, (N, C)).coalesce()


def zipf(N, C, nnz, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    p = 1.0 / torch.arange(1, C + 1, device="cuda", dtype=torch.float64)
    cols = torch.multinomial((p / p.sum()).float(), nnz, replacement=True, generator=g)
    rows = torch.randint(0, N, (nnz,), generator=g, device="cuda")
    lin = (rows * C + cols).unique()
    vals = torch.randint(1, 6, (lin.numel(),), generator=g, device="cuda").float()
    return torch.sparse_coo_tensor(torch.stack([lin // C, lin % C]), vals, (N, C)).coalesce()


def factors(N, C, R, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.rand(C, R, generator=g, device="cuda") + 0.1, torch.rand(N, R, generator=g, device="cuda") + 0.1


def fit(V, M, W0, H0, solver, iters):
    """(seconds, module) of one fit of `iters` iterations from (W0, H0), ended by a device synchronise."""
    m = NMF(W=W0.clone(), H=H0.clone()).cuda()
    torch.cuda.synchronize()
    t = time.perf_counter()
    m.fit(V, 2, float("-inf"), iters, solver=solver, mask=M)
    torch.cuda.synchronize()
    return time.perf_counter() - t, m


def loss(V, m):
    """1/2 sum_obs (v - h_n . w_c)^2 of a module's factors, from the library's observed-cell loss launch."""
    eng = CudaObservedNmfEngine(V, m.W.data, m.H.data)
    try:
        return eng.loss(2)
    finally:
        eng.close()


def workload(V, W0, H0, reps, mu_iters):
    M = torch.sparse_coo_tensor(V.indices(), torch.ones(V._nnz(), dtype=torch.bool, device="cuda"), V.shape)
    cols = torch.bincount(V.indices()[1], minlength=V.shape[1])
    out = {"observed": V._nnz(), "longest_column": int(cols.max()), "mean_column": float(cols.float().mean())}
    for solver in ("cd", "mu"):
        fit(V, M, W0, H0, solver, 10)                                        # warm-up: modules, workspaces
        rates = []
        for _ in range(reps):
            t30, _ = fit(V, M, W0, H0, solver, 30)
            t60, _ = fit(V, M, W0, H0, solver, 60)
            rates.append(30.0 / (t60 - t30))
        out[solver] = {"it_per_s": statistics.median(rates)}
    times = [fit(V, M, W0, H0, "mu", mu_iters)[0] for _ in range(reps)]
    goal = loss(V, fit(V, M, W0, H0, "mu", mu_iters)[1])
    out["mu"].update(time_to_mu_s=statistics.median(times), iters_to_mu=mu_iters, loss=goal)
    k = 10
    while k <= mu_iters:
        cur = loss(V, fit(V, M, W0, H0, "cd", k)[1])
        if cur <= goal:
            break
        k += 10
    if k <= mu_iters:
        times = [fit(V, M, W0, H0, "cd", k)[0] for _ in range(reps)]
        out["cd"].update(time_to_mu_s=statistics.median(times), iters_to_mu=k, loss=cur)
    else:
        out["cd"].update(time_to_mu_s=None, iters_to_mu=None, loss=cur)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--mu-iters", type=int, default=200)
    ap.add_argument("--only", default=None, help="comma-separated workload names")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("observed_cd_rate.py needs a CUDA device")
    res = {"card": card()}
    work = {"uniform_64": (lambda: uniform(65536, 8192, 0.005, 1), 65536, 8192, 64),
            "uniform_32": (lambda: uniform(262144, 131072, 1e-4, 1), 262144, 131072, 32),
            "zipf_32": (lambda: zipf(200000, 50000, 5_000_000, 1), 200000, 50000, 32)}
    for name, (make, N, C, R) in work.items():
        if a.only and name not in a.only.split(","):
            continue
        V = make()
        W0, H0 = factors(N, C, R, seed=2)
        res[name] = {"shape": [N, C, R], **workload(V, W0, H0, a.reps, a.mu_iters)}
        del V
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
