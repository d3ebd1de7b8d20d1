"""Iteration rate of the batched PLCA fits against a Python loop of the single fits, and how a batched iteration's device time
splits between the raw-terms passes and the EM step; one JSON line per workload and fit.

    python tools/batched_plca_rate.py [--rounds 3] [--loop-sample 64]

Workloads (seeded inputs generated on the device):
  many_plca       1024 PLCA problems of 256 x 512, R = 16, each with its own V
  clips_siplca    256 SIPLCA problems of one clip (1, 513, 512), R = 8, T = 16, each with its own V
  restarts_plca   32 restarts of one shared 4096 x 2048 V, R = 32
  single_plca     one PLCA problem of 8192 x 4096, R = 64 (P = 1)
Fits:
  batched     BatchedPLCA / BatchedSIPLCA(W=W0, H=H0).fit(V, ...) over every problem of the workload
  loop_f32    for p: PLCA / SIPLCA(W=W0[p], H=H0[p]).fit(V[p], ..., precision="f32")
The loops run over the first `--loop-sample` problems only (all of them when there are fewer); every rate is per problem
iteration.  Each fit is timed (device-synchronised) at 60 and at 30 iterations with tol = -inf, after one warm-up fit of the
same shape; the rate is problems x 30 over the difference, i.e. the iterations alone.  The median of `--rounds` rounds is
reported, the fits alternating within a round.  The split line times, with CUDA events on the batched engine, 20 calls of
nmfb200_plca_iterate(1) against 20 pairs of nmfb200_raw_terms (which also take the column sums the EM iteration skips, so
the raw-terms share is an upper bound).  The card's name and power limit are read in the same run.  Writes nothing.
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

from torchnmf_b200 import PLCA, SIPLCA, BatchedPLCA, BatchedSIPLCA  # noqa: E402
from torchnmf_b200 import engine as _engine  # noqa: E402
from torchnmf_b200.engine import release_workspaces  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (x.strip() for x in out.split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def inputs(P, vshape, wshape, hshape, shared, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    V = torch.rand(*(vshape if shared else (P,) + vshape), generator=g, device="cuda")
    W0 = torch.rand(P, *wshape, generator=g, device="cuda") + 0.1
    H0 = torch.rand(P, *hshape, generator=g, device="cuda") + 0.1
    return V, W0, H0


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t


def fit_batched(cls, V, W0, H0, iters):
    m = cls(W=W0, H=H0).cuda()
    return lambda: m.fit(V, float("-inf"), iters)


def fit_loop(cls, V, W0, H0, iters, n, shared):
    R = W0.shape[2]
    mods = [cls(W=W0[p], H=H0[p], Z=torch.ones(R) / R).cuda() for p in range(n)]
    Vs = [V if shared else V[p] for p in range(n)]
    return lambda: [m.fit(v, float("-inf"), iters, precision="f32") for m, v in zip(mods, Vs)]


def split(batched_cls, engine_cls, V, W0, H0, shared, reps=20):
    """Device milliseconds per iteration: (plca_iterate(1), the two raw-terms passes)."""
    m = batched_cls(W=W0, H=H0).cuda()
    W, H, Z = m.W.data, m.H.data, m.Z.data
    P = W.shape[0]
    Vn = V / V.sum() if shared else V / V.sum(list(range(1, V.dim())), keepdim=True)
    Hz = (H * Z.reshape(P, 1, -1, *([1] * (H.dim() - 3)))).contiguous()
    eng = engine_cls(Vn.contiguous(), W, Hz)
    try:
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        eng.plca_iterate(2, H, Z, True, True, True)
        eng.raw_terms(0, 1.0); eng.raw_terms(1, 1.0)
        ev[0].record()
        for _ in range(reps):
            eng.plca_iterate(1, H, Z, True, True, True)
        ev[1].record()
        for _ in range(reps):
            eng.raw_terms(0, 1.0); eng.raw_terms(1, 1.0)
        ev[2].record()
        torch.cuda.synchronize()
        return ev[0].elapsed_time(ev[1]) / reps, ev[1].elapsed_time(ev[2]) / reps
    finally:
        eng.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--loop-sample", type=int, default=64)
    args = ap.parse_args()
    dev = card()
    # name, batched class, single class, engine, P, V's single shape, W's and H's per-problem shapes, shared V
    workloads = [
        ("many_plca", BatchedPLCA, PLCA, _engine.CudaBatchedNmfEngine, 1024, (256, 512), (512, 16), (256, 16), False),
        ("clips_siplca", BatchedSIPLCA, SIPLCA, _engine.CudaBatchedNmfdEngine, 256, (1, 513, 512), (513, 8, 16),
         (1, 8, 497), False),
        ("restarts_plca", BatchedPLCA, PLCA, _engine.CudaBatchedNmfEngine, 32, (4096, 2048), (2048, 32), (4096, 32), True),
        ("single_plca", BatchedPLCA, PLCA, _engine.CudaBatchedNmfEngine, 1, (8192, 4096), (4096, 64), (8192, 64), False),
    ]
    for name, bcls, scls, ecls, P, vshape, wshape, hshape, shared in workloads:
        V, W0, H0 = inputs(P, vshape, wshape, hshape, shared, seed=P + vshape[0])
        n_loop = min(P, args.loop_sample)
        fits = {"batched": (P, lambda it: fit_batched(bcls, V, W0, H0, it)),
                "loop_f32": (n_loop, lambda it: fit_loop(scls, V, W0, H0, it, n_loop, shared))}
        for _, make in fits.values():                  # warm-up: every shape the timed fits use
            timed(make(10))
        rates = {k: [] for k in fits}
        for _ in range(args.rounds):
            for k, (probs, make) in fits.items():
                t60 = timed(make(60))
                t30 = timed(make(30))
                rates[k].append(probs * 30 / (t60 - t30))
        base = {"workload": name, "P": P, "V": list(vshape), "W": list(wshape), "H": list(hshape), "shared_V": shared}
        for k, r in rates.items():
            print(json.dumps({**base, "fit": k, "problems_timed": fits[k][0], "problem_it_per_s": statistics.median(r),
                              "rounds": r, "card": dev}), flush=True)
        it_ms, terms_ms = split(bcls, ecls, V, W0, H0, shared)
        print(json.dumps({**base, "split_ms_per_iteration": {"plca_iterate": it_ms, "raw_terms_pair": terms_ms,
                                                             "em_step_at_least": it_ms - terms_ms}, "card": dev}),
              flush=True)
        del V, W0, H0
        release_workspaces()
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
