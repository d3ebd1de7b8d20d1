"""Fit rate and device memory of sparse targets at beta 0.5 and 1.5 on the any-beta sparse engine against the densified
path; prints one JSON line.

    python tools/sparse_beta_rate.py [--iters 50] [--warmup 2] [--big-iters 3] [--calls 20]

Workloads (targets generated on the device from fixed seeds, factors rand + 0.5):
  mid   65536 x 8192, 0.5 % stored, R = 64: `NMF.fit` iterations per second and torch's peak allocation above what was
        allocated before the fit, on the sparse engine (no dense copy of V) and on the densified path
        (`_sparse_kernels = False`: V.to_dense() on the device, the fused fp32 kernels).  Then the device time per call of the
        V-free denominator contraction (simt_contract_kernel in its V-free mode) and of the dense kGeneric contraction, both
        factors, from torch.profiler over `--calls` raw-terms calls of each engine (a run of its own after the timed fits),
        and the CUDA-event time of those whole raw-terms calls.
  big   262144 x 131072, about 0.01 % stored, R = 32: the sparse engine's rate and peak allocation (its dense form would take
        128 GiB).
The card's name, power limit and maximum SM clock are read in the same run.  Writes nothing.
"""
import argparse
import json
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
from torchnmf_b200.engine import CudaNmfEngine, CudaSparseAnyBetaEngine, release_workspaces  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (x.strip() for x in out.split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def sparse_target(N, C, density, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    nnz = int(N * C * density)
    idx = torch.randint(0, N * C, (nnz,), generator=g, device="cuda").unique()
    vals = torch.rand(idx.numel(), generator=g, device="cuda") + 0.5
    return torch.sparse_coo_tensor(torch.stack([idx // C, idx % C]), vals, (N, C)).coalesce()


def factors(N, C, R, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.rand(C, R, generator=g, device="cuda") + 0.5, torch.rand(N, R, generator=g, device="cuda") + 0.5


def timed_fit(V, W0, H0, beta, iters, warmup, densify):
    """(iterations per second, torch's peak allocation growth in bytes) of one fit after a warm-up fit."""
    m = NMF(W=W0.clone(), H=H0.clone()).cuda()
    m._sparse_kernels = not densify
    m.fit(V, beta, float("-inf"), warmup)
    release_workspaces()
    m.W.data.copy_(W0)
    m.H.data.copy_(H0)
    torch.cuda.synchronize()
    alloc0 = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    n = m.fit(V, beta, float("-inf"), iters)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    assert n == iters
    peak = torch.cuda.max_memory_allocated() - alloc0
    release_workspaces()
    return {"it_per_s": iters / dt, "torch_peak_growth_bytes": peak,
            "factors_finite": bool(torch.isfinite(m.W).all() and torch.isfinite(m.H).all())}


def contraction_times(V, W0, H0, beta, calls):
    """Device time per call of the contraction kernels (torch.profiler) and CUDA-event time per raw-terms call."""
    engines = {"vfree_sparse": CudaSparseAnyBetaEngine(V, W0.clone(), H0.clone()),
               "dense_kgeneric": CudaNmfEngine(V.to_dense(), W0.clone(), H0.clone(), "f32")}
    out = {}
    for tag, eng in engines.items():
        for which in (0, 1):
            eng.raw_terms(which, beta)                    # warm-up
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(calls):
            for which in (0, 1):
                eng.raw_terms(which, beta)
        b.record()
        torch.cuda.synchronize()
        acts = [torch.profiler.ProfilerActivity.CUDA]
        with torch.profiler.profile(activities=acts) as prof:
            for _ in range(calls):
                for which in (0, 1):
                    eng.raw_terms(which, beta)
            torch.cuda.synchronize()
        kern = [e for e in prof.key_averages() if "simt_contract_kernel" in e.key]
        dev_us = sum(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) for e in kern)
        out[tag] = {"contraction_us_per_update": dev_us / (2 * calls),
                    "contraction_kernels": sorted({e.key[:120] for e in kern}),
                    "raw_terms_ms_per_update_events": a.elapsed_time(b) / (2 * calls)}
        eng.close()
    release_workspaces()
    out["vfree_over_dense"] = (out["vfree_sparse"]["contraction_us_per_update"]
                               / out["dense_kgeneric"]["contraction_us_per_update"])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--big-iters", type=int, default=3)
    ap.add_argument("--calls", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sparse_beta_rate.py needs a CUDA device")
    res = {"card": card(), "iters": a.iters, "workloads": []}
    N, C, R = 65536, 8192, 64
    V = sparse_target(N, C, 0.005, 0)
    W0, H0 = factors(N, C, R, 1)
    for beta in (0.5, 1.5):
        w = {"workload": "mid", "shape": [N, C], "nnz": int(V._nnz()), "R": R, "beta": beta,
             "sparse": timed_fit(V, W0, H0, beta, a.iters, a.warmup, False),
             "densified": timed_fit(V, W0, H0, beta, a.iters, a.warmup, True),
             "contraction": contraction_times(V, W0, H0, beta, a.calls)}
        w["speedup_sparse_over_densified"] = w["sparse"]["it_per_s"] / w["densified"]["it_per_s"]
        print(json.dumps(w), file=sys.stderr, flush=True)
        res["workloads"].append(w)
    del V, W0, H0
    torch.cuda.empty_cache()
    N, C, R = 262144, 131072, 32
    V = sparse_target(N, C, 1e-4, 2)
    W0, H0 = factors(N, C, R, 3)
    for beta in (0.5, 1.5):
        w = {"workload": "big", "shape": [N, C], "nnz": int(V._nnz()), "R": R, "beta": beta,
             "dense_fp32_bytes_would_be": 4 * N * C,
             "sparse": timed_fit(V, W0, H0, beta, a.big_iters, 1, False)}
        print(json.dumps(w), file=sys.stderr, flush=True)
        res["workloads"].append(w)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
