"""Fit rate of a weighted fit (`fit(V, ..., weight=Wt)`) against the masked fit of the same cells and a plain-PyTorch
weighted MU loop; one JSON line per workload.

    python tools/weighted_rate.py [--iters 30] [--warmup 3] [--rounds 3]

Workloads (seeded inputs generated on the device; weights uniform in [0.25, 4) on the kept cells):
  nmf_b1, nmf_b0.5   NMF 16384 x 4096 R=64, 30 % of the cells of weight 0, dense weight
  nmfd_b1            NMFD 4 x 1025 x 2048 R=16 T=128 at beta 1, 30 % of weight 0, dense weight
  sp_mid_b1          NMF 65536 x 8192 R=64, a sparse weight storing 0.5 % of the cells, dense V
  sp_rec_b1          NMF 262144 x 131072 R=32, a sparse weight storing 0.01 % of the cells, sparse V
Fits, run alternately `--rounds` times each from the same initial factors after a `--warmup` fit of the same shapes,
each timed (device-synchronised) over `--iters` and over 2 x `--iters` iterations: `fit_it_per_s` is `--iters` over the
first time, one fit's setup (validation, target registration, the sparse workloads' observed-set construction) included;
`it_per_s` is `--iters` over the difference of the two, the iterations alone:
  weighted   fit(V, beta, weight=Wt)
  masked     fit(V, beta, mask=Wt > 0)            the same cells without weights
  torch      the weighted MU update written in plain PyTorch: the reconstruction WH materialised, num / den of each
             factor from two backward passes of w V (WH + eps)^(beta-2) and w (WH + eps)^(beta-1) (dense workloads only:
             the only route real-valued weights had before)
Reported per fit: both rates of every round and their medians; for the dense NMF workloads also `contract_ms`, the device
time (CUDA events, median of 3 x 20 launches) of one W and one H contraction of the weighted and of the masked kernels on
one context.  The card's name and power limit are read in the same run.  Writes nothing.
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
from torchnmf_b200.engine import CudaNmfEngine, release_workspaces  # noqa: E402

EPS = float(torch.finfo(torch.float32).eps)


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (x.strip() for x in out.split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def dense_inputs(vshape, wshape, hshape, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    V = torch.rand(*vshape, generator=g, device="cuda")
    W = torch.rand(*wshape, generator=g, device="cuda") + 0.1
    H = torch.rand(*hshape, generator=g, device="cuda") + 0.1
    Wt = 0.25 + 3.75 * torch.rand(*vshape, generator=g, device="cuda")
    Wt.masked_fill_(torch.rand(*vshape, generator=g, device="cuda") < 0.3, 0.0)
    return V, W, H, Wt


def torch_step(m, V, Wt, beta):
    """One weighted MU iteration in plain PyTorch (nmf.py:78-92 on the two backward passes of the weighted loss)."""
    for p in (m.W, m.H):
        with torch.enable_grad():
            WH = m.reconstruct(m.H, m.W) if p is m.W else m.reconstruct(m.H, m.W.detach())
            x = WH.detach() + EPS
            Pn = Wt * V * x.pow(beta - 2) if beta != 2 else Wt * V
            Pp = Wt * x.pow(beta - 1) if beta != 2 else Wt * WH.detach()
            num, = torch.autograd.grad(WH, p, Pn, retain_graph=True)
            den, = torch.autograd.grad(WH, p, Pp)
        gamma = 1.0 / (2.0 - beta) if beta < 1 else 1.0
        with torch.no_grad():
            p.mul_(((num.clamp_min(0) + EPS) / (den.clamp_min(0) + EPS)).pow(gamma))


def run(mode, cls, V, sel, W0, H0, beta, iters):
    m = cls(W=W0, H=H0).cuda()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    if mode == "torch":
        Vd = torch.nan_to_num(V)
        for _ in range(iters):
            torch_step(m, Vd, sel, beta)
    else:
        assert m.fit(V, beta, float("-inf"), iters, **sel) == iters
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def contract_ms(V, W0, H0, sels, beta):
    """Device time of one W and one H contraction (nmfb200_nmf_contract_only) per selector, on one fp32 context."""
    eng = CudaNmfEngine(V, W0.clone(), H0.clone(), "f32")
    out = {}
    try:
        for mode in ("weighted", "masked"):
            if mode == "weighted":
                eng.set_weight(sels[mode]["weight"])
            else:
                eng.set_mask(sels[mode]["mask"])
            times = []
            for rep in range(4):                        # the first repetition warms up
                t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0.record()
                for _ in range(20):
                    eng.contract_only(0, beta)
                    eng.contract_only(1, beta)
                t1.record()
                t1.synchronize()
                if rep:
                    times.append(t0.elapsed_time(t1) / 20)
            out[mode] = statistics.median(times)
    finally:
        eng.close()
    return out


def workload(name, cls, V, W0, H0, sels, beta, a, extra):
    for mode, sel in sels.items():                      # warm-up: module loads, cached workspaces of these shapes
        run(mode, cls, V, sel, W0, H0, beta, a.warmup)
    fit_rates = {mode: [] for mode in sels}
    rates = {mode: [] for mode in sels}
    for _ in range(a.rounds):
        for mode, sel in sels.items():
            t1 = run(mode, cls, V, sel, W0, H0, beta, a.iters)
            t2 = run(mode, cls, V, sel, W0, H0, beta, 2 * a.iters)
            fit_rates[mode].append(a.iters / t1)
            rates[mode].append(a.iters / (t2 - t1))
    med = {mode: statistics.median(r) for mode, r in rates.items()}
    out = {"workload": name, "shape": list(V.shape), "R": W0.shape[1], "beta": beta, **extra, "iters": a.iters,
           "card": a.card, "it_per_s": rates, "median_it_per_s": med, "fit_it_per_s": fit_rates,
           "median_fit_it_per_s": {mode: statistics.median(r) for mode, r in fit_rates.items()},
           "weighted_over_masked": med["weighted"] / med["masked"]}
    if "torch" in med:
        out["weighted_over_torch"] = med["weighted"] / med["torch"]
    if cls is NMF and not V.is_sparse and not sels["weighted"]["weight"].is_sparse:
        out["contract_ms"] = contract_ms(V, W0, H0, sels, beta)
    release_workspaces()
    print(json.dumps(out), flush=True)


def sparse_cells(N, C, share, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    nnz = int(share * N * C)
    lin = torch.unique(torch.randint(0, N * C, (nnz,), generator=g, device="cuda"))
    idx = torch.stack([lin // C, lin % C])
    w = 0.25 + 3.75 * torch.rand(lin.numel(), generator=g, device="cuda")
    return idx, w, g


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("weighted_rate.py needs a CUDA device")
    a.card = card()
    N, C, R = 16384, 4096, 64
    V, W, H, Wt = dense_inputs((N, C), (C, R), (N, R), 0)
    sels = {"weighted": {"weight": Wt}, "masked": {"mask": Wt > 0}, "torch": Wt}
    for beta in (1.0, 0.5):
        workload(f"nmf_b{beta:g}", NMF, V, W, H, sels, beta, a, {"zero_weight": 0.3})
    del V, W, H, Wt, sels
    B, C, L, R, T = 4, 1025, 2048, 16, 128
    V, W, H, Wt = dense_inputs((B, C, L), (C, R, T), (B, R, L - T + 1), 1)
    sels = {"weighted": {"weight": Wt}, "masked": {"mask": Wt > 0}, "torch": Wt}
    workload("nmfd_b1", NMFD, V, W, H, sels, 1.0, a, {"zero_weight": 0.3})
    del V, W, H, Wt, sels
    for name, (N, C, R, share, sparse_v) in {"sp_mid_b1": (65536, 8192, 64, 0.005, False),
                                             "sp_rec_b1": (262144, 131072, 32, 0.0001, True)}.items():
        idx, w, g = sparse_cells(N, C, share, 2)
        if sparse_v:
            V = torch.sparse_coo_tensor(idx, torch.rand(idx.shape[1], generator=g, device="cuda"), (N, C))
        else:
            V = torch.rand(N, C, generator=g, device="cuda")
        W0 = torch.rand(C, R, generator=g, device="cuda") + 0.1
        H0 = torch.rand(N, R, generator=g, device="cuda") + 0.1
        sels = {"weighted": {"weight": torch.sparse_coo_tensor(idx, w, (N, C))},
                "masked": {"mask": torch.sparse_coo_tensor(idx, torch.ones_like(w, dtype=torch.bool), (N, C))}}
        workload(name, NMF, V, W0, H0, sels, 1.0, a, {"stored": int(idx.shape[1])})
        del V, W0, H0, sels


if __name__ == "__main__":
    main()
