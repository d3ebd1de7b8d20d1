"""Fit rate and per-update device time of NMF2D / NMF3D / SIPLCA2 at precision "f32" (the CUDA-core sliding kernels) and
"f16" (the tensor-core sliding GEMMs, beta 1), and how far their outputs are apart; prints one JSON line per workload and
the card's name and power limit, all read in the same run.

    python tools/nd_tc_rate.py [--iters 50] [--warmup 3] [--rounds 2] [--reps 20]

Per workload, the two precisions run alternately, `--rounds` times each, from the same seeded inputs:
  * it/s: a timed `fit` of --iters iterations (tol -inf) after a --warmup fit, host clock around a device synchronise;
  * update_w_ms / update_h_ms / loss_ms: CUDA events around --reps calls of one engine's W update, H update and loss at
    beta 1, on the fit's shapes (each update is the reconstruction, the contraction and the ratio stage);
  * out_diff: max over W and H of |f16 - f32| / (1e-3 |f32| + 1e-5 max |f32|) after the timed fits (1 = the north-star
    tolerance).
Writes nothing.
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

from torchnmf_b200 import NMF2D, NMF3D, SIPLCA2  # noqa: E402
from torchnmf_b200.engine import CudaNmfdEngine, release_workspaces  # noqa: E402

# (name, class, V shape, rank, kernel size)
WORKLOADS = [
    ("nmf2d-1ch", NMF2D, (1, 1, 256, 1024), 16, (8, 32)),          # one-channel spectrogram-like target
    ("nmf2d-c128", NMF2D, (2, 128, 24, 512), 32, (4, 16)),         # 128 channels
    ("nmf3d-c16", NMF3D, (1, 16, 16, 24, 256), 16, (3, 4, 16)),
    ("siplca2-c64", SIPLCA2, (1, 64, 48, 512), 16, (4, 16)),
]


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (x.strip() for x in out.split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def inputs(shape, R, K, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    B, C, *X = shape
    J = [x - k + 1 for x, k in zip(X, K)]
    V = torch.rand(*shape, generator=g, device="cuda")
    W = torch.rand(C, R, *K, generator=g, device="cuda") + 0.1
    H = torch.rand(B, R, *J, generator=g, device="cuda") + 0.1
    return V, W, H


def fit(cls, V, W0, H0, prec, iters):
    if cls is SIPLCA2:                                      # normalises W, H, Z and V itself
        R = W0.shape[1]
        m = cls(W=W0.clone(), H=H0.clone(), Z=torch.full((R,), 1.0 / R, device=W0.device)).cuda()
        m.fit(V, float("-inf"), iters, precision=prec)
        return m
    m = cls(W=W0.clone(), H=H0.clone()).cuda()
    m.fit(V, 1, float("-inf"), iters, precision=prec)
    return m


def timed_fit(cls, V, W0, H0, prec, iters, warmup):
    release_workspaces()
    fit(cls, V, W0, H0, prec, warmup)
    torch.cuda.synchronize()
    t = time.perf_counter()
    m = fit(cls, V, W0, H0, prec, iters)
    torch.cuda.synchronize()
    return iters / (time.perf_counter() - t), m


def event_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def update_times(V, W0, H0, prec, reps):
    release_workspaces()
    eng = CudaNmfdEngine(V, W0.clone(), H0.clone(), prec)
    assert eng.precision_for(1) == prec, (eng.precision_for(1), prec)
    out = {"update_w_ms": event_ms(lambda: eng.update_w(1.0, 1.0, 0.0, 0.0), reps),
           "update_h_ms": event_ms(lambda: eng.update_h(1.0, 1.0, 0.0, 0.0), reps),
           "loss_ms": event_ms(lambda: eng.loss_tensor(1.0), reps)}
    eng.close()
    return out


def diff(a, b):
    atol = 1e-5 * float(b.abs().max())
    return float(((a - b).abs() / (1e-3 * b.abs() + atol)).max())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "nd_tc_rate.py measures on a CUDA device"
    print(json.dumps({"card": card()}))
    for name, cls, shape, R, K in WORKLOADS:
        V, W0, H0 = inputs(shape, R, K, seed=len(name))
        Vin = V / V.sum() if cls is SIPLCA2 else V
        rec = {"workload": name, "V": list(shape), "R": R, "K": list(K)}
        models = {}
        for _ in range(a.rounds):
            for prec in ("f32", "f16"):
                rate, m = timed_fit(cls, V, W0, H0, prec, a.iters, a.warmup)
                assert m.last_fit_precision == prec
                rec.setdefault(prec + "_it_s", []).append(round(rate, 2))
                models[prec] = m
        for prec in ("f32", "f16"):
            rec[prec + "_times"] = {k: round(v, 4) for k, v in update_times(Vin, W0, H0, prec, a.reps).items()}
        rec["out_diff"] = max(diff(models["f16"].W.data, models["f32"].W.data),
                              diff(models["f16"].H.data, models["f32"].H.data))
        print(json.dumps(rec))
        release_workspaces()


if __name__ == "__main__":
    main()
