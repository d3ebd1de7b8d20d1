"""Iteration rate of `BatchedNMFD.fit` against a Python loop of `NMFD.fit`; one JSON line per workload and fit.

    python tools/batched_nmfd_rate.py [--rounds 3] [--loop-sample 64]

Workloads (seeded inputs generated on the device; V[p] is (1, C, L), one spectrogram-like clip):
  many_b1, many_b0.5   256 problems of (1, 513, 512), R = 8, T = 16, each with its own V, at beta 1 and 0.5
  restarts_b1          32 restarts of one shared (1, 1025, 2048) V, R = 16, T = 32, beta 1
  single_b1            one problem of (1, 1025, 8192), R = 16, T = 128, beta 1 (P = 1)
Fits:
  batched      BatchedNMFD(W=W0, H=H0).fit(V, ...) over every problem of the workload
  loop_f32     for p: NMFD(W=W0[p], H=H0[p]).fit(V[p], ..., precision="f32")
  loop_auto    the same loop at precision="auto" (NMFD's tensor cores at beta 1)
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

from torchnmf_b200 import NMFD, BatchedNMFD  # noqa: E402
from torchnmf_b200.engine import release_workspaces  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (x.strip() for x in out.split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def inputs(P, C, L, R, T, shared, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    V = torch.rand(*((1, C, L) if shared else (P, 1, C, L)), generator=g, device="cuda")
    W0 = torch.rand(P, C, R, T, generator=g, device="cuda") + 0.1
    H0 = torch.rand(P, 1, R, L - T + 1, generator=g, device="cuda") + 0.1
    return V, W0, H0


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t


def fit_batched(V, W0, H0, beta, iters):
    m = BatchedNMFD(W=W0, H=H0).cuda()
    return lambda: m.fit(V, beta, float("-inf"), iters)


def fit_loop(V, W0, H0, beta, iters, precision, n):
    mods = [NMFD(W=W0[p], H=H0[p]).cuda() for p in range(n)]
    Vs = [V if V.dim() == 3 else V[p] for p in range(n)]
    return lambda: [m.fit(v, beta, float("-inf"), iters, precision=precision) for m, v in zip(mods, Vs)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--loop-sample", type=int, default=64)
    args = ap.parse_args()
    dev = card()
    workloads = [("many_b1", 256, 513, 512, 8, 16, False, 1, True), ("many_b0.5", 256, 513, 512, 8, 16, False, 0.5, True),
                 ("restarts_b1", 32, 1025, 2048, 16, 32, True, 1, True),
                 ("single_b1", 1, 1025, 8192, 16, 128, False, 1, False)]
    for name, P, C, L, R, T, shared, beta, with_auto in workloads:
        V, W0, H0 = inputs(P, C, L, R, T, shared, seed=P + C)
        n_loop = min(P, args.loop_sample)
        fits = {"batched": (P, lambda it: fit_batched(V, W0, H0, beta, it)),
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
            print(json.dumps({"workload": name, "fit": k, "P": P, "C": C, "L": L, "R": R, "T": T, "shared_V": shared, "beta": beta,
                              "problems_timed": fits[k][0], "problem_it_per_s": statistics.median(r),
                              "rounds": r, "card": dev}), flush=True)
        del V, W0, H0
        release_workspaces()
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
