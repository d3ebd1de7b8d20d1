"""Iteration rate of `BatchedNMFD.fit(V, ..., lengths=L)` (a ragged batch of clips) against a Python loop of `NMFD.fit` on
each clip's real frames; one JSON line per workload and fit.

    python tools/batched_nmfd_ragged_rate.py [--rounds 3] [--loop-sample 64]

Workloads (seeded inputs generated on the device): 256 clips of (1, 513, L_p), L_p drawn uniformly from [128, 1024],
R = 8, T = 16, each with its own V, stored padded to 1024 frames; at beta 1 and 0.5.
Fits:
  ragged       BatchedNMFD(W=W0, H=H0).fit(V, ..., lengths=L) over every clip
  loop_f32     for p: NMFD(W=W0[p], H=H0[p, ..., :L_p - T + 1]).fit(V[p, ..., :L_p], ..., precision="f32")
  loop_auto    the same loop at precision="auto" (NMFD's tensor cores at beta 1)
  padded       for scale only: the uniform batch on V zero-padded to 1024 frames, which fits another model
The loops run over the first `--loop-sample` clips only; every rate is per problem iteration, so a loop's rate does not
depend on how many clips it covers (the sample's mean length is printed beside it).  Protocol of
tools/batched_nmfd_rate.py: each fit is timed (device-synchronised) at 60 and at 30 iterations with tol = -inf, after one
warm-up fit of the same shape; the rate is problems x 30 over the difference.  The median of `--rounds` rounds is reported,
the fits alternating within a round.  The card's name and power limit are read in the same run.  Writes nothing.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "pytorch-nmf_b200"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

from batched_nmfd_rate import card, timed  # noqa: E402
from torchnmf_b200 import NMFD, BatchedNMFD  # noqa: E402
from torchnmf_b200.engine import release_workspaces  # noqa: E402

P, C, X, R, T = 256, 513, 1024, 8, 16


def inputs(seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    lengths = torch.randint(128, X + 1, (P,), generator=g, device="cuda").tolist()
    V = torch.rand(P, 1, C, X, generator=g, device="cuda")
    W0 = torch.rand(P, C, R, T, generator=g, device="cuda") + 0.1
    H0 = torch.rand(P, 1, R, X - T + 1, generator=g, device="cuda") + 0.1
    for p, L in enumerate(lengths):
        V[p, ..., L:] = 0.0
    return V, W0, H0, lengths


def fit_batched(V, W0, H0, beta, iters, lengths=None):
    m = BatchedNMFD(W=W0, H=H0).cuda()
    kw = {} if lengths is None else {"lengths": lengths}
    return lambda: m.fit(V, beta, float("-inf"), iters, **kw)


def fit_loop(V, W0, H0, lengths, beta, iters, precision, n):
    mods = [NMFD(W=W0[p], H=H0[p, ..., :lengths[p] - T + 1].contiguous()).cuda() for p in range(n)]
    Vs = [V[p, ..., :lengths[p]].contiguous() for p in range(n)]
    return lambda: [m.fit(v, beta, float("-inf"), iters, precision=precision) for m, v in zip(mods, Vs)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--loop-sample", type=int, default=64)
    args = ap.parse_args()
    dev = card()
    for beta in (1, 0.5):
        V, W0, H0, lengths = inputs(seed=17)
        n_loop = min(P, args.loop_sample)
        fits = {"ragged": (P, lambda it: fit_batched(V, W0, H0, beta, it, lengths)),
                "loop_f32": (n_loop, lambda it: fit_loop(V, W0, H0, lengths, beta, it, "f32", n_loop)),
                "loop_auto": (n_loop, lambda it: fit_loop(V, W0, H0, lengths, beta, it, "auto", n_loop)),
                "padded": (P, lambda it: fit_batched(V, W0, H0, beta, it))}
        for _, make in fits.values():                  # warm-up: every shape the timed fits use
            timed(make(10))
        rates = {k: [] for k in fits}
        for _ in range(args.rounds):
            for k, (probs, make) in fits.items():
                t60 = timed(make(60))
                t30 = timed(make(30))
                rates[k].append(probs * 30 / (t60 - t30))
        for k, r in rates.items():
            n = fits[k][0]
            print(json.dumps({"workload": f"ragged_b{beta}", "fit": k, "P": P, "C": C, "X": X, "R": R, "T": T, "beta": beta,
                              "problems_timed": n, "mean_length": sum(lengths[:n]) / n,
                              "problem_it_per_s": statistics.median(r), "rounds": r, "card": dev}), flush=True)
        del V, W0, H0
        release_workspaces()
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
