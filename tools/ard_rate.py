"""Iteration rate of ARD fits (`fit(V, ..., ard=ARD())`) against the plain fit of the same shape; one JSON line per workload.

    python tools/ard_rate.py [--rounds 3]

Workloads (seeded inputs generated on the device):
  nmf_auto   NMF 65536 x 4096, R = 64, beta 1, precision "auto" (bench.py's configs[1])
  nmf_f32    NMF 16384 x 4096, R = 64, beta 0.5, precision "f32"
  nmfd       NMFD (1, 1025, 8192), R = 16, T = 128, beta 1
Each fit is timed twice from the same initial factors, over 30 and over 60 iterations (tol -inf, device-synchronised), and
its iteration rate is 30 / (t60 - t30): the iterations alone, without the one-time registrations both runs share.  Modes,
run alternately, `--rounds` times each after one warm-up round: `ard` (the ARD fit: each iteration's W and H updates take
the per-component penalties, then the lambda update runs) and `plain` (the fit without it).  Reported: every round's rate,
the median and the ratio of the medians.  The card's name and power limit are read in the same run.  Writes nothing.
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
from torchnmf_b200.nmf import ARD  # noqa: E402


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


def runner(cls, mode, V, W0, H0, beta, precision):
    def fit(iters):
        m = cls(W=W0, H=H0).cuda()
        kw = {"ard": ARD()} if mode == "ard" else {}
        assert m.fit(V, beta, float("-inf"), iters, precision=precision, **kw) == iters
    return fit


def workload(name, make, meta, a):
    modes = ("ard", "plain")
    for mode in modes:                                   # warm-up: module loads, cached workspaces of these shapes
        make(mode)(3)
    rates = {mode: [] for mode in modes}
    for _ in range(a.rounds):
        for mode in modes:
            rates[mode].append(rate(make(mode)))
    med = {mode: statistics.median(r) for mode, r in rates.items()}
    print(json.dumps({"workload": name, **meta, "card": a.card, "it_per_s": rates, "median_it_per_s": med,
                      "ard_over_plain": med["ard"] / med["plain"]}), flush=True)
    release_workspaces()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ard_rate.py needs a CUDA device")
    a.card = card()
    g = torch.Generator(device="cuda").manual_seed(0)
    for name, (N, C, beta, prec) in (("nmf_auto", (65536, 4096, 1, "auto")), ("nmf_f32", (16384, 4096, 0.5, "f32"))):
        R = 64
        V = torch.rand(N, C, generator=g, device="cuda")
        W0, H0 = torch.rand(C, R, generator=g, device="cuda") + 0.1, torch.rand(N, R, generator=g, device="cuda") + 0.1
        workload(name, lambda mode: runner(NMF, mode, V, W0, H0, beta, prec),
                 {"shape": [N, C], "R": R, "beta": beta, "precision": prec}, a)
        del V, W0, H0
    B, C, L, R, T = 1, 1025, 8192, 16, 128
    V = torch.rand(B, C, L, generator=g, device="cuda")
    W0 = torch.rand(C, R, T, generator=g, device="cuda") + 0.1
    H0 = torch.rand(B, R, L - T + 1, generator=g, device="cuda") + 0.1
    workload("nmfd", lambda mode: runner(NMFD, mode, V, W0, H0, 1, "auto"),
             {"shape": [B, C, L], "R": R, "T": T, "beta": 1, "precision": "auto"}, a)


if __name__ == "__main__":
    main()
