"""Iteration rate of a ragged `BatchedPLCA.fit(V, ..., lengths=L)` against a Python loop of `PLCA.fit` on each problem's rows
and against the uniform batch on the same data zero-padded; one JSON line per fit.

    python tools/batched_plca_ragged_rate.py [--rounds 3] [--loop-sample 64]

Workload (seeded inputs generated on the device): 1024 PLCA problems over C = 512 columns, R = 16, problem p with L_p rows
drawn uniformly from [64, 512] (seed 0), stored padded to N = 512 rows.
Fits:
  ragged       BatchedPLCA(W=W0, H=H0).fit(V, ..., lengths=L): problem p is the EM fit of V[p, :L_p]
  loop_f32     for p: PLCA(W=W0[p], H=H0[p, :L_p]).fit(V[p, :L_p], ..., precision="f32")
  padded       BatchedPLCA(W=W0, H=H0).fit(V with rows L_p: zeroed): a different model -- the zero rows count as observed
               zeros in each problem's normalised target and receive H mass -- timed only as the speed of the uniform
               batch on the padded size
The loop runs over the first `--loop-sample` problems only; every rate is per problem iteration (the loop's and the ragged
fit's counting each problem once whatever its length).  Each fit is timed (device-synchronised) at 60 and at 30 iterations
with tol = -inf, after one warm-up fit; the rate is problems x 30 over the difference, i.e. the iterations alone.  The
median of `--rounds` rounds is reported, the fits alternating within a round.  The card's name and power limit are read
in the same run.  Writes nothing.
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

from batched_plca_rate import card, timed  # noqa: E402
from torchnmf_b200 import PLCA, BatchedPLCA  # noqa: E402
from torchnmf_b200.engine import release_workspaces  # noqa: E402

P, N, C, R = 1024, 512, 512, 16


def inputs(seed=0):
    g = torch.Generator().manual_seed(seed)
    lengths = torch.randint(64, N + 1, (P,), generator=g).tolist()
    gd = torch.Generator(device="cuda").manual_seed(seed)
    V = torch.rand(P, N, C, generator=gd, device="cuda")
    W0 = torch.rand(P, C, R, generator=gd, device="cuda") + 0.1
    H0 = torch.rand(P, N, R, generator=gd, device="cuda") + 0.1
    rows = torch.arange(N, device="cuda") < torch.tensor(lengths, device="cuda").unsqueeze(1)
    V *= rows.unsqueeze(2)                       # the padding is zero: the padded fit's target
    H0 *= rows.unsqueeze(2)                      # and H's padding rows hold no mass at the start of the ragged fit
    return V, W0, H0, lengths


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--loop-sample", type=int, default=64)
    args = ap.parse_args()
    dev = card()
    V, W0, H0, lengths = inputs()
    n_loop = min(P, args.loop_sample)

    def ragged(it):
        m = BatchedPLCA(W=W0, H=H0).cuda()
        return lambda: m.fit(V, float("-inf"), it, lengths=lengths)

    def padded(it):
        m = BatchedPLCA(W=W0, H=H0).cuda()
        return lambda: m.fit(V, float("-inf"), it)

    def loop(it):
        mods = [PLCA(W=W0[p], H=H0[p, :lengths[p]], Z=torch.ones(R) / R).cuda() for p in range(n_loop)]
        return lambda: [m.fit(V[p, :lengths[p]], float("-inf"), it, precision="f32") for p, m in enumerate(mods)]
    fits = {"ragged": (P, ragged), "loop_f32": (n_loop, loop), "padded": (P, padded)}
    for _, make in fits.values():
        timed(make(10))
    rates = {k: [] for k in fits}
    for _ in range(args.rounds):
        for k, (probs, make) in fits.items():
            t60 = timed(make(60))
            t30 = timed(make(30))
            rates[k].append(probs * 30 / (t60 - t30))
    for k, r in rates.items():
        print(json.dumps({"fit": k, "P": P, "N_max": N, "C": C, "R": R,
                          "lengths": [min(lengths), max(lengths), sum(lengths) / P], "problems_timed": fits[k][0],
                          "problem_it_per_s": statistics.median(r), "rounds": r, "card": dev}), flush=True)
    release_workspaces()


if __name__ == "__main__":
    main()
