"""Iteration rate of fits with fixed components of W (`fit(V, ..., fixed_W=F)`) against the plain fit of the same rank and
the `trainer.BetaMu` closure workaround; one JSON line per workload.

    python tools/fixed_w_rate.py [--rounds 3]

Workloads (seeded inputs generated on the device):
  nmf_auto   NMF 1025 x 16384, R = 80 with the first 64 components fixed, beta 1, precision "auto"
  nmf_f32    the same at precision "f32"
  siplca     SIPLCA (1, 513, 8192), R = 32 with the first 24 components fixed, T = 16
Each fit is timed twice from the same initial factors, over 30 and over 60 iterations (tol -inf, device-synchronised), and
its iteration rate is 30 / (t60 - t30): the iterations alone, without the one-time target registration and the loss
evaluations both runs share.  Modes, run alternately, `--rounds` times each after one warm-up round:
  fixed    fit(V, ..., fixed_W=F)
  plain    fit(V, ...) of the same R, every component free
  betamu   (NMF only) trainer.BetaMu([W_free, H], beta) with a closure that concatenates the fixed columns (a buffer) with the
           free ones (a Parameter): the route a fixed subset of W took before, two autograd backward passes per update.
           SIPLCA's fit is EM, which BetaMu does not run.
Reported: every round's rate and the median.  The card's name and power limit are read in the same run.  Writes nothing.
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

from torchnmf_b200 import NMF, SIPLCA  # noqa: E402
from torchnmf_b200.engine import release_workspaces  # noqa: E402
from torchnmf_b200.trainer import BetaMu  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (x.strip() for x in out.split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def timed(fn, iters):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn(iters)
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def rate(fn):
    return 30 / (timed(fn, 60) - timed(fn, 30))


def nmf_runner(mode, V, W0, H0, F, precision):
    def fit(iters):
        if mode == "betamu":
            Wfix = W0[:, F].clone()
            Wfree = torch.nn.Parameter(W0[:, ~F].clone())
            H = torch.nn.Parameter(H0.clone())
            opt = BetaMu([Wfree, H], 1)

            def closure():
                opt.zero_grad()
                return V, H @ torch.cat([Wfix, Wfree], 1).t()

            for _ in range(iters):
                opt.step(closure)
            return
        m = NMF(W=W0, H=H0).cuda()
        kw = {"fixed_W": F} if mode == "fixed" else {}
        assert m.fit(V, 1, float("-inf"), iters, precision=precision, **kw) == iters
    return fit


def siplca_runner(mode, V, W0, H0, Z0, F):
    def fit(iters):
        m = SIPLCA(W=W0, H=H0, Z=Z0).cuda()
        kw = {"fixed_W": F} if mode == "fixed" else {}
        m.fit(V, float("-inf"), iters, **kw)
    return fit


def workload(name, make, modes, meta, a):
    for mode in modes:                                   # warm-up: module loads, cached workspaces of these shapes
        make(mode)(3)
    rates = {mode: [] for mode in modes}
    for _ in range(a.rounds):
        for mode in modes:
            rates[mode].append(rate(make(mode)))
    med = {mode: statistics.median(r) for mode, r in rates.items()}
    out = {"workload": name, **meta, "card": a.card, "it_per_s": rates, "median_it_per_s": med,
           "fixed_over_plain": med["fixed"] / med["plain"]}
    if "betamu" in med:
        out["fixed_over_betamu"] = med["fixed"] / med["betamu"]
    release_workspaces()
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fixed_w_rate.py needs a CUDA device")
    a.card = card()
    g = torch.Generator(device="cuda").manual_seed(0)
    N, C, R, K = 1025, 16384, 80, 64
    V = torch.rand(N, C, generator=g, device="cuda")
    W0, H0 = torch.rand(C, R, generator=g, device="cuda") + 0.1, torch.rand(N, R, generator=g, device="cuda") + 0.1
    F = torch.arange(R, device="cuda") < K
    for prec in ("auto", "f32"):
        workload(f"nmf_{prec}", lambda mode: nmf_runner(mode, V, W0, H0, F, prec), ("fixed", "plain", "betamu"),
                 {"shape": [N, C], "R": R, "fixed": K, "beta": 1, "precision": prec}, a)
    del V, W0, H0
    B, C, L, R, K, T = 1, 513, 8192, 32, 24, 16
    V = torch.rand(B, C, L, generator=g, device="cuda")
    W0 = torch.rand(C, R, T, generator=g, device="cuda")
    H0 = torch.rand(B, R, L - T + 1, generator=g, device="cuda")
    Z0 = torch.rand(R, generator=g, device="cuda")
    F = torch.arange(R, device="cuda") < K
    workload("siplca", lambda mode: siplca_runner(mode, V, W0, H0, Z0, F), ("fixed", "plain"),
             {"shape": [B, C, L], "R": R, "fixed": K, "T": T}, a)


if __name__ == "__main__":
    main()
