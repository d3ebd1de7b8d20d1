"""Iteration rate of PLCA fits on sparse targets (`PLCA.fit(V)` with V sparse COO), against the dense fp32 and fp16 fits of
V.to_dense() where the dense form fits on the card, and the device time of one EM step's two sparse gathers against the two
sparse-NMF numerator calls the step would take without them; one JSON line per workload.

    python tools/sparse_plca_rate.py [--rounds 3]

Workloads (seeded targets generated on the device; stored values Poisson-like counts 1-5, duplicates summed):
  plsa_r100 / plsa_r512  262144 documents x 65536 terms, ~200 stored entries per document (52 M), rank 100 / 512: its dense
                         fp32 form is 64 GiB, so only the sparse fit runs
  dense_1pct / dense_0.1pct  32768 x 16384 at 1 % / 0.1 % stored, rank 64: the sparse fit, and the dense fit of V.to_dense()
                         at precision "f32" and "f16"
A fit's rate is 30 / (t60 - t30), t_k the device-synchronised time of a k-iteration fit (tol = -inf) from the same initial
factors, so the one-time set-up (coalescing, both compressed forms, the context) cancels; the median over `--rounds` rounds
is reported, the fits of a round alternating.  "gathers_ms": CUDA-event time of one nmfb200_plca_sparse_terms call (the
row gather with its dot products and ratios, and the column gather of the ratios) against two nmfb200_raw_terms calls at
beta 1 on a sparse NMF context with the same factor pair (each a gather with its own dot products, plus a column sum), the
median of 20 calls each, at ranks <= 256.  The card's name and power limit are read in the same run.  Writes nothing.
"""
import argparse
import gc
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

from torchnmf_b200 import PLCA  # noqa: E402
from torchnmf_b200.engine import CudaSparseNmfEngine, CudaSparsePlcaEngine  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (x.strip() for x in out.split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def target(N, C, nnz, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    if nnz >= N:      # documents: the same number of terms each
        rows = torch.arange(N, device="cuda").repeat_interleave(nnz // N)
    else:
        rows = torch.randint(0, N, (nnz,), device="cuda", generator=g)
    cols = torch.randint(0, C, (rows.numel(),), device="cuda", generator=g)
    vals = torch.randint(1, 6, (rows.numel(),), device="cuda", generator=g).float()
    return torch.sparse_coo_tensor(torch.stack([rows, cols]), vals, (N, C)).coalesce()


def workloads():
    yield "plsa_r100", target(262144, 65536, 262144 * 200, 0), 100, ("sparse",)
    yield "plsa_r512", target(262144, 65536, 262144 * 200, 0), 512, ("sparse",)
    yield "dense_1pct", target(32768, 16384, 32768 * 16384 // 100, 1), 64, ("sparse", "f32", "f16")
    yield "dense_0.1pct", target(32768, 16384, 32768 * 16384 // 1000, 2), 64, ("sparse", "f32", "f16")


def one(kind, V, Vd, R, iters):
    torch.manual_seed(1)
    m = PLCA(tuple(V.shape), rank=R).cuda()
    gc.collect()                  # the previous fit's engine frees its context here, not inside the timed fit
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    if kind == "sparse":
        m.fit(V, float("-inf"), iters)
    else:
        m.fit(Vd, float("-inf"), iters, precision=kind)
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def event_ms(fn, reps=20):
    for _ in range(3):
        fn()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return statistics.median(times)


def gathers(V, R):
    """ms of one sparse PLCA terms call and of two sparse NMF raw-terms calls at beta 1, on the same (W, Hz)."""
    N, C = V.shape
    g = torch.Generator(device="cuda").manual_seed(3)
    W = torch.rand(C, R, device="cuda", generator=g)
    Hz = torch.rand(N, R, device="cuda", generator=g)
    W /= W.sum(0)
    Hz /= Hz.sum()
    vals = V.values()
    Vn = torch.sparse_coo_tensor(V.indices(), vals / vals.sum(), V.shape, is_coalesced=True)
    eng = CudaSparsePlcaEngine(Vn, W, Hz)
    try:
        plca = event_ms(lambda: eng.plca_terms(Hz))
    finally:
        eng.close()
    nmf = CudaSparseNmfEngine(Vn, W, Hz, "f32")
    try:
        two = event_ms(lambda: (nmf.raw_terms(0, 1.0), nmf.raw_terms(1, 1.0)))
    finally:
        nmf.close()
    return {"plca_sparse_terms": round(plca, 3), "two_raw_terms": round(two, 3), "speedup": round(two / plca, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    info = card()
    for name, V, R, kinds in workloads():
        Vd = V.to_dense() if len(kinds) > 1 else None
        for k in kinds:                                      # warm every shape and kernel
            one(k, V, Vd, R, 10)
        rates = {k: [] for k in kinds}
        for _ in range(args.rounds):
            for k in kinds:
                t30 = one(k, V, Vd, R, 30)
                t60 = one(k, V, Vd, R, 60)
                rates[k].append(30.0 / (t60 - t30))
        med = {k: statistics.median(v) for k, v in rates.items()}
        rec = {"workload": name, "shape": list(V.shape), "nnz": int(V._nnz()), "rank": R, "card": info,
               "iters_per_s": {k: round(v, 2) for k, v in med.items()},
               "rounds": {k: [round(x, 2) for x in v] for k, v in rates.items()}}
        if len(kinds) > 1:
            rec["sparse_vs_dense"] = {k: round(med["sparse"] / med[k], 3) for k in kinds if k != "sparse"}
        if R <= 256:
            rec["gathers_ms"] = gathers(V, R)
        print(json.dumps(rec), flush=True)
        del Vd


if __name__ == "__main__":
    main()
