"""Rate of the rank-blocked fp32 NMF kernels at ranks 256, 512 and 1024 on one GPU; prints one JSON line.

    python tools/high_rank_rate.py [--iters 20] [--warmup 3] [--launches 10]

For a 32768 x 4096 target at R in {256, 512, 1024} and beta in {1, 2}: the device-resident fp32 `NMF.fit` rate (iterations
per second after a warm-up fit), the `nmfb200_nmf_contract_only` kernel time of the W and H updates (CUDA events over
`--launches` launches), the algorithmic FLOPs of each over that time against the 67 TFLOP/s FP32 data-sheet figure of the
H100 SXM, and the recompute factor of the plan (S is recomputed once per block of 256 output components).  Then the ratio of
the R = 512 and R = 256 iteration times per beta, and the unmodified reference's `.cuda()` rate at the same shapes when it is
installed under oracle/_ref.  The card's name and power limit are read in the same run.  Writes nothing.
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "pytorch-nmf_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

from torchnmf_b200 import NMF  # noqa: E402
from torchnmf_b200.engine import CudaNmfEngine  # noqa: E402

N, C = 32768, 4096
RANKS = (256, 512, 1024)
BETAS = (1.0, 2.0)
FP32_PEAK = 67e12


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (x.strip() for x in out.split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def rank_blocks(R):
    return -(-R // 256)


def min_flops(R, beta):
    """One factor update: S = F G^T (2 N C R) and the numerator (2 N C R), plus the denominator (2 N C R) for beta != 1."""
    return (4 if beta == 1 else 6) * N * C * R


def recompute(R, beta):
    nb = rank_blocks(R)
    return (nb + 1) / 2 if beta == 1 else (nb + 2) / 3


def inputs(R, dev):
    g = torch.Generator(device=dev).manual_seed(0)
    V = torch.rand(N, C, generator=g, device=dev).bfloat16().float()
    W = torch.rand(C, R, generator=g, device=dev) + 0.1
    H = torch.rand(N, R, generator=g, device=dev) + 0.1
    return V, W, H


def fit_rate(V, W0, H0, beta, iters, warmup):
    m = NMF(W=W0.clone(), H=H0.clone())
    m.fit(V, beta, float("-inf"), warmup, precision="f32")
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    m.fit(V, beta, float("-inf"), iters, precision="f32")
    torch.cuda.synchronize()
    assert m.last_fit_precision == "f32"
    return iters / (time.perf_counter() - t0)


def contract_ms(V, W0, H0, beta, launches):
    eng = CudaNmfEngine(V, W0.clone(), H0.clone(), "f32")
    out = []
    for which in (0, 1):
        eng.contract_only(which, beta)
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(launches):
            eng.contract_only(which, beta)
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b) / launches)
    eng.check_health()
    eng.close()
    return out


def reference_rate(V, W0, H0, beta, iters):
    ref_dir = os.path.join(ROOT, "oracle", "_ref")
    if not os.path.isdir(os.path.join(ref_dir, "torchnmf")):
        return None
    if ref_dir not in sys.path:
        sys.path.insert(0, ref_dir)
    import torchnmf.nmf as ref_nmf
    m = ref_nmf.NMF(W=W0.clone(), H=H0.clone()).cuda()
    m.fit(V, beta, float("-inf"), 1)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    m.fit(V, beta, float("-inf"), iters)
    torch.cuda.synchronize()
    return iters / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--launches", type=int, default=10)
    ap.add_argument("--ref-iters", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("high_rank_rate.py needs a CUDA device")
    dev = torch.device("cuda")
    res = {"card": card(), "shape": [N, C], "fp32_datasheet_tflops": FP32_PEAK / 1e12, "runs": []}
    per_iter = {}
    for R in RANKS:
        V, W0, H0 = inputs(R, dev)
        for beta in BETAS:
            rate = fit_rate(V, W0, H0, beta, a.iters, a.warmup)
            ms_w, ms_h = contract_ms(V, W0, H0, beta, a.launches)
            f = min_flops(R, beta)
            run = {"R": R, "beta": beta, "rank_blocks": rank_blocks(R), "recompute_factor": recompute(R, beta),
                   "fit_it_per_s": rate, "contract_ms": {"W": ms_w, "H": ms_h},
                   "algorithmic_tflops": {"W": f / ms_w / 1e9, "H": f / ms_h / 1e9},
                   "executed_tflops": {"W": f * recompute(R, beta) / ms_w / 1e9,
                                       "H": f * recompute(R, beta) / ms_h / 1e9}}
            run["algorithmic_share_of_fp32_datasheet"] = {k: v * 1e12 / FP32_PEAK for k, v in run["algorithmic_tflops"].items()}
            ref = reference_rate(V, W0, H0, beta, a.ref_iters)
            run["reference_cuda_it_per_s"] = ref if ref is not None else "not installed"
            per_iter[(R, beta)] = 1.0 / rate
            res["runs"].append(run)
            print(json.dumps(run), file=sys.stderr, flush=True)
        del V, W0, H0
        torch.cuda.empty_cache()
    res["r512_over_r256_iteration_time"] = {str(b): per_iter[(512, b)] / per_iter[(256, b)] for b in BETAS}
    # what the FLOP model predicts for that ratio: twice the rank, times the recompute factor of two blocks
    res["flop_model_r512_over_r256"] = {str(b): 2 * recompute(512, b) / recompute(256, b) for b in BETAS}
    assert all(math.isfinite(x) for x in per_iter.values())
    print(json.dumps(res))


if __name__ == "__main__":
    main()
