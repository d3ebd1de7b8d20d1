"""Iteration rate of `BatchedNMF.fit(..., solver="cd")` against a Python loop of `NMF.fit(..., solver="cd")` and against
batched multiplicative updates, at beta 2 on the fp32 kernels; prints one JSON line.

    python tools/batched_cd_rate.py [--reps 3] [--loop-sample 64] [--mu-iters 200]

Workloads (seeded inputs generated on the device; V = rand, factors rand + 0.1):
  many       1024 problems of 256 x 512, R = 16, each with its own V
  restarts   32 restarts of one shared 4096 x 2048 V, R = 32
  single     one problem of 16384 x 4096, R = 64 (B = 1)
Fits:
  batched_cd   BatchedNMF(W=W0, H=H0).fit(V, 2, ..., solver="cd") over every problem
  loop_cd      for b: NMF(W=W0[b], H=H0[b]).fit(V[b], 2, ..., solver="cd"), over the first --loop-sample problems
  batched_mu   BatchedNMF(...).fit(V, 2, ..., precision="f32") (many only)
Rates are problem-iterations per second for the iterations alone: problems x 30 / (time of a 60-iteration fit - time of a
30-iteration fit), tol = -inf, each fit device-synchronised, median of --reps, after one warm-up fit per shape.
many also reports time_to_mu_s: the wall time of batched MU's --mu-iters fit, and of the batched cd fit of the fewest
iterations (a multiple of 10) after which every problem's loss is at or below the loss batched MU reaches for it.
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

from torchnmf_b200 import NMF, BatchedNMF  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (x.strip() for x in out.split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def inputs(B, N, C, R, shared, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    V = torch.rand(N, C, generator=g, device="cuda") if shared else torch.rand(B, N, C, generator=g, device="cuda")
    return V, torch.rand(B, C, R, generator=g, device="cuda") + 0.1, torch.rand(B, N, R, generator=g, device="cuda") + 0.1


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t, out


def fit_batched(V, W0, H0, iters, solver):
    m = BatchedNMF(W=W0.clone(), H=H0.clone()).cuda()
    m.fit(V, 2, float("-inf"), iters, precision="f32", solver=solver)
    return m


def fit_loop(V, W0, H0, iters, n):
    for b in range(n):
        NMF(W=W0[b].clone(), H=H0[b].clone()).cuda().fit(V if V.dim() == 2 else V[b], 2, float("-inf"), iters, solver="cd")


def rate(fn, problems, reps):
    fn(10)                                                      # warm-up: modules, contexts, workspaces
    rates = []
    for _ in range(reps):
        t30, _ = timed(lambda: fn(30))
        t60, _ = timed(lambda: fn(60))
        rates.append(problems * 30.0 / (t60 - t30))
    return statistics.median(rates)


def losses(V, m):
    """1/2 |V_b - H_b W_b^T|^2 of every problem, float64 sums of the fp32 residual."""
    E = V - torch.bmm(m.H.data, m.W.data.transpose(1, 2))
    return 0.5 * (E.double() ** 2).sum((1, 2))


def time_to_mu(V, W0, H0, mu_iters, reps):
    t_mu = statistics.median(timed(lambda: fit_batched(V, W0, H0, mu_iters, "mu"))[0] for _ in range(reps))
    goal = losses(V, fit_batched(V, W0, H0, mu_iters, "mu"))
    k = 10
    while k <= mu_iters and not bool((losses(V, fit_batched(V, W0, H0, k, "cd")) <= goal).all()):
        k += 10
    out = {"mu": {"iters": mu_iters, "time_s": t_mu}, "cd": {"iters": None, "time_s": None}}
    if k <= mu_iters:
        t_cd = statistics.median(timed(lambda: fit_batched(V, W0, H0, k, "cd"))[0] for _ in range(reps))
        out["cd"] = {"iters": k, "time_s": t_cd}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--loop-sample", type=int, default=64)
    ap.add_argument("--mu-iters", type=int, default=200)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("batched_cd_rate.py needs a CUDA device")
    res = {"card": card(), "unit": "problem-iterations per second"}
    for name, (B, N, C, R, shared) in {"many": (1024, 256, 512, 16, False), "restarts": (32, 4096, 2048, 32, True),
                                       "single": (1, 16384, 4096, 64, False)}.items():
        V, W0, H0 = inputs(B, N, C, R, shared, seed=1)
        n = min(B, a.loop_sample)
        w = {"B": B, "N": N, "C": C, "R": R, "shared_V": shared,
             "batched_cd": rate(lambda k: fit_batched(V, W0, H0, k, "cd"), B, a.reps),
             "loop_cd": rate(lambda k: fit_loop(V, W0, H0, k, n), n, a.reps)}
        if name == "many":
            w["batched_mu"] = rate(lambda k: fit_batched(V, W0, H0, k, "mu"), B, a.reps)
            w["time_to_mu_s"] = time_to_mu(V, W0, H0, a.mu_iters, a.reps)
        res[name] = w
        del V, W0, H0
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
