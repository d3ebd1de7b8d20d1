"""Fit rate of a fit on the cells of a sparse mask (`fit(V, ..., mask=M)` with a sparse COO `M`) against the dense-mask fit
and the BetaMu workaround; one JSON line per workload.

    python tools/observed_rate.py [--iters 50] [--warmup 3] [--rounds 3]

Workloads (observed cells drawn at random, seeded inputs generated on the device):
  rec     262144 x 131072, 0.01 % observed, R=32, beta 1 and 0.5: the observed fit alone (V sparse at the observed cells).
          The dense mask (V 128 GiB in fp32, M 32 GiB) and BetaMu (the dense reconstruction) cannot hold this shape.
  mid     65536 x 8192, 0.5 % observed, R=64, beta 1 and 0.5
  dense   16384 x 4096, 70 % observed, R=64, beta 1: where the dense masked path wins
For each workload the fits run alternately, `--rounds` times each, from the same initial factors, every one timed over
`--iters` iterations after a `--warmup` fit of the same shapes (device-synchronised, so a fit's one-time work -- building the
observed set, registering the target -- is included):
  observed    fit(V, beta, mask=M_sparse)                  the observed-cell gathers, O(observed x R) per update
  dense_mask  fit(V, beta, mask=M_sparse.to_dense())       the dense masked fp32 kernels, O(N C R) per update
  betamu      trainer.BetaMu([W, H], beta) with the closure (V_obs, model()[rows, cols]): two backward passes through the
              materialised reconstruction per factor update
Reported per fit: iterations per second of every round and their median, and the peak of torch.cuda.max_memory_allocated
over its rounds (the inputs included).  The card's name and power limit are read in the same run.  Writes nothing.
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
from torchnmf_b200.engine import release_workspaces  # noqa: E402
from torchnmf_b200.trainer import BetaMu  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (x.strip() for x in out.split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def inputs(N, C, R, frac, seed, dense):
    """W, H, the sparse mask and V: dense (N, C) when `dense`, else sparse with values at the observed cells only."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    W = torch.rand(C, R, generator=g, device="cuda") + 0.1
    H = torch.rand(N, R, generator=g, device="cuda") + 0.1
    if dense:
        V = torch.rand(N, C, generator=g, device="cuda")
        Ms = (torch.rand(N, C, generator=g, device="cuda") < frac).to_sparse()
    else:
        lin = torch.unique(torch.randint(0, N * C, (int(frac * N * C),), generator=g, device="cuda"))
        idx = torch.stack([lin // C, lin % C])
        V = torch.sparse_coo_tensor(idx, torch.rand(lin.numel(), generator=g, device="cuda"), (N, C)).coalesce()
        Ms = torch.sparse_coo_tensor(idx, torch.ones(lin.numel(), dtype=torch.bool, device="cuda"), (N, C)).coalesce()
    return V, W, H, Ms


def run(mode, V, Ms, Md, W0, H0, beta, iters):
    m = NMF(W=W0, H=H0).cuda()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    if mode == "betamu":
        opt = BetaMu([m.W, m.H], beta)
        rows, cols = Ms.indices()
        Vo = V[rows, cols]

        def closure():
            opt.zero_grad()
            return Vo, m()[rows, cols]

        for _ in range(iters):
            opt.step(closure)
    else:
        assert m.fit(V, beta, float("-inf"), iters, mask=Ms if mode == "observed" else Md) == iters
    torch.cuda.synchronize()
    return iters / (time.perf_counter() - t0)


def workload(name, V, W0, H0, Ms, beta, modes, a):
    Md = Ms.to_dense() if "dense_mask" in modes else None
    for mode in modes:                                  # warm-up: module loads, cached workspaces of these shapes
        run(mode, V, Ms, Md, W0, H0, beta, a.warmup)
    rates = {mode: [] for mode in modes}
    peak = {mode: 0 for mode in modes}
    for _ in range(a.rounds):
        for mode in modes:
            torch.cuda.reset_peak_memory_stats()
            rates[mode].append(run(mode, V, Ms, Md, W0, H0, beta, a.iters))
            peak[mode] = max(peak[mode], torch.cuda.max_memory_allocated())
    med = {mode: statistics.median(r) for mode, r in rates.items()}
    N, C = V.shape
    out = {"workload": name, "shape": [N, C], "R": W0.shape[1], "beta": beta, "observed": Ms._nnz(),
           "observed_frac": Ms._nnz() / (N * C), "iters": a.iters, "card": a.card, "it_per_s": rates,
           "median_it_per_s": med, "max_memory_allocated": peak}
    for mode in modes[1:]:
        out[f"observed_over_{mode}"] = med["observed"] / med[mode]
    release_workspaces()
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("observed_rate.py needs a CUDA device")
    a.card = card()
    V, W, H, Ms = inputs(262144, 131072, 32, 1e-4, 0, dense=False)
    for beta in (1.0, 0.5):
        workload(f"rec_b{beta:g}", V, W, H, Ms, beta, ("observed",), a)
    del V, W, H, Ms
    V, W, H, Ms = inputs(65536, 8192, 64, 5e-3, 1, dense=True)
    for beta in (1.0, 0.5):
        workload(f"mid_b{beta:g}", V, W, H, Ms, beta, ("observed", "dense_mask", "betamu"), a)
    del V, W, H, Ms
    V, W, H, Ms = inputs(16384, 4096, 64, 0.7, 2, dense=True)
    workload("dense_b1", V, W, H, Ms, 1.0, ("observed", "dense_mask", "betamu"), a)


if __name__ == "__main__":
    main()
