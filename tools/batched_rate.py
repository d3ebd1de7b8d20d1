"""Iteration rate of `BatchedNMF.fit` against a Python loop of `NMF.fit`; one JSON line per workload and fit.

    python tools/batched_rate.py [--rounds 3] [--loop-sample 64]

Workloads (seeded inputs generated on the device):
  many_b2, many_b1   1024 problems of 256 x 512, R = 16, each with its own V, at beta 2 and 1
  restarts_b1        32 restarts of one shared 4096 x 2048 V, R = 32, beta 1
  single_b1          one problem of 16384 x 4096, R = 64, beta 1 (B = 1)
Fits:
  batched      BatchedNMF(W=W0, H=H0).fit(V, ...) over every problem of the workload
  loop_f32     for b: NMF(W=W0[b], H=H0[b]).fit(V[b], ..., precision="f32")
  loop_auto    the same loop at precision="auto" (the tensor cores where the shape allows them)
The loops run over the first `--loop-sample` problems only (all of them when there are fewer); every rate is per problem
iteration, so a loop's rate does not depend on how many problems it covers.  Each fit is timed (device-synchronised) at 60
and at 30 iterations with tol = -inf, after one warm-up fit of the same shape; the rate is problems x 30 over the
difference, i.e. the iterations alone, without each fit's setup.  The median of `--rounds` rounds is reported, the fits of a
workload alternating within a round.  The card's name and power limit are read in the same run.  Writes nothing.
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
from torchnmf_b200.engine import release_workspaces  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (x.strip() for x in out.split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def inputs(B, N, C, R, shared, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    V = torch.rand(*((N, C) if shared else (B, N, C)), generator=g, device="cuda")
    W0 = torch.rand(B, C, R, generator=g, device="cuda") + 0.1
    H0 = torch.rand(B, N, R, generator=g, device="cuda") + 0.1
    return V, W0, H0


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t


def fit_batched(V, W0, H0, beta, iters):
    m = BatchedNMF(W=W0, H=H0).cuda()
    return lambda: m.fit(V, beta, float("-inf"), iters)


def fit_loop(V, W0, H0, beta, iters, precision, n):
    mods = [NMF(W=W0[b], H=H0[b]).cuda() for b in range(n)]
    Vs = [V if V.dim() == 2 else V[b] for b in range(n)]
    return lambda: [m.fit(v, beta, float("-inf"), iters, precision=precision) for m, v in zip(mods, Vs)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--loop-sample", type=int, default=64)
    args = ap.parse_args()
    dev = card()
    workloads = [("many_b2", 1024, 256, 512, 16, False, 2, True), ("many_b1", 1024, 256, 512, 16, False, 1, True),
                 ("restarts_b1", 32, 4096, 2048, 32, True, 1, True), ("single_b1", 1, 16384, 4096, 64, False, 1, False)]
    for name, B, N, C, R, shared, beta, with_auto in workloads:
        V, W0, H0 = inputs(B, N, C, R, shared, seed=B + N)
        n_loop = min(B, args.loop_sample)
        fits = {"batched": (B, lambda it: fit_batched(V, W0, H0, beta, it)),
                "loop_f32": (n_loop, lambda it: fit_loop(V, W0, H0, beta, it, "f32", n_loop))}
        if with_auto:
            fits["loop_auto"] = (n_loop, lambda it: fit_loop(V, W0, H0, beta, it, "auto", n_loop))
        for _, make in fits.values():                  # warm-up: every shape the timed fits use
            timed(make(10))
        rates = {k: [] for k in fits}
        for _ in range(args.rounds):
            for k, (probs, make) in fits.items():
                t60 = timed(make(60))
                t30 = timed(make(30))
                rates[k].append(probs * 30 / (t60 - t30))
        for k, r in rates.items():
            print(json.dumps({"workload": name, "fit": k, "B": B, "N": N, "C": C, "R": R, "shared_V": shared, "beta": beta,
                              "problems_timed": fits[k][0], "problem_it_per_s": statistics.median(r),
                              "rounds": r, "card": dev}), flush=True)
        del V, W0, H0
        release_workspaces()
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
