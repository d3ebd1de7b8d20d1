"""Fit rate, device memory and bit-identity of an fp32 target against the same values held as bfloat16; prints one JSON line.

    python tools/half_target_rate.py [--iters 100] [--warmup 3] [--rounds 2] [--big-iters 3]

For each workload the fp32 target (V.float()) and the bf16 target V are fitted alternately, `--rounds` times each, from the
same initial factors:
  cfg2      NMF 65536 x 4096 R=64 beta 1 (BASELINE.json configs[1]) at precision f32 and auto
  r300      the same target at R=300, fp32 (rank-blocked kernels)
  cfg3      NMFD 1025 x 8192 R=16 T=128 (BASELINE.json configs[2]) at beta 1 (tensor cores) and beta 2 (fp32)
Per run: `NMF.fit` iterations per second (a timed fit of --iters iterations after a --warmup fit, device-synchronised, so
it includes the fit's one-time target registration), the target's own bytes, torch's peak allocation during the fit above
what was allocated before it, and the bytes the library holds for the fit (the drop of cudaMemGetInfo's free memory while
the fit's context is parked in the workspace cache, less torch's reserve growth) and their sum with the target's bytes:
the device memory the fit holds.  Per workload: whether the fp32-target and
bf16-target fits give byte-equal W and H.  If cudaMemGetInfo reports at least 60 GB free, a few iterations of the one-GPU
bf16 8192 x 2^20 R=128 fit (BASELINE.json configs[3] on one card, fed as 2^20 x 8192), which an fp32 copy of the target
would not leave room for; otherwise the line says it was skipped.  The card's name and power limit are read in the same run.
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

from torchnmf_b200 import NMF, NMFD  # noqa: E402
from torchnmf_b200.engine import release_workspaces  # noqa: E402

GB = 1e9


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (x.strip() for x in out.split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def nmf_target(N, C, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.rand(N, C, generator=g, device="cuda").bfloat16()


def nmf_factors(N, C, R, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.rand(C, R, generator=g, device="cuda") + 0.1, torch.rand(N, R, generator=g, device="cuda") + 0.1


def nmfd_inputs(B, C, L, R, T, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    V = torch.rand(B, C, L, generator=g, device="cuda").bfloat16()
    W = torch.rand(C, R, T, generator=g, device="cuda") + 0.1
    H = torch.rand(B, R, L - T + 1, generator=g, device="cuda") + 0.1
    return V, W, H


def one_fit(cls, V, W0, H0, beta, precision, iters, warmup):
    """(rate, memory record, model) of one timed fit on a fresh workspace."""
    m = cls(W=W0.clone(), H=H0.clone())
    release_workspaces()
    torch.cuda.synchronize()
    m.fit(V, beta, float("-inf"), warmup, precision=precision)          # warm-up: module loads, the same shapes
    release_workspaces()
    m.W.data.copy_(W0)
    m.H.data.copy_(H0)
    torch.cuda.synchronize()
    free0, reserved0, alloc0 = torch.cuda.mem_get_info()[0], torch.cuda.memory_reserved(), torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    n = m.fit(V, beta, float("-inf"), iters, precision=precision)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    assert n == iters
    free1, reserved1 = torch.cuda.mem_get_info()[0], torch.cuda.memory_reserved()
    mem = {"target_bytes": V.numel() * V.element_size(),
           "torch_peak_growth_bytes": torch.cuda.max_memory_allocated() - alloc0,
           "library_bytes": (free0 - free1) - (reserved1 - reserved0)}
    mem["device_bytes_held"] = sum(mem.values())
    release_workspaces()
    return iters / dt, mem, m


def workload(name, cls, V16, W0, H0, beta, precision, a):
    runs = {"fp32": [], "bf16": []}
    models = {}
    Vf = V16.float()
    for _ in range(a.rounds):
        for tag, V in (("fp32", Vf), ("bf16", V16)):
            rate, mem, m = one_fit(cls, V, W0, H0, beta, precision, a.iters, a.warmup)
            runs[tag].append({"it_per_s": rate, **mem, "fit_precision": m.last_fit_precision})
            models[tag] = m
    equal = all(torch.equal(getattr(models["fp32"], k).data, getattr(models["bf16"], k).data) for k in ("W", "H"))
    out = {"workload": name, "beta": beta, "precision": precision, "runs": runs, "outputs_byte_equal": equal}
    del Vf
    torch.cuda.empty_cache()
    print(json.dumps(out), file=sys.stderr, flush=True)
    return out


def big_fit(iters):
    free = torch.cuda.mem_get_info()[0]
    if free < 60 * GB:
        return {"skipped": f"only {free / GB:.1f} GB free (needs 60)"}
    N, C, R = 1 << 20, 8192, 128
    g = torch.Generator(device="cuda").manual_seed(1)
    V = torch.empty(N, C, dtype=torch.bfloat16, device="cuda")
    for i in range(0, N, 1 << 16):                   # generated in slabs: no fp32 temporary of the whole target
        V[i:i + (1 << 16)] = torch.rand(min(1 << 16, N - i), C, generator=g, device="cuda")
    W0 = torch.rand(C, R, generator=g, device="cuda") + 0.1
    H0 = torch.rand(N, R, generator=g, device="cuda") + 0.1
    m = NMF(W=W0, H=H0)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    n = m.fit(V, 1, float("-inf"), iters)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    out = {"shape": [N, C], "R": R, "iters": n, "seconds": dt, "it_per_s_including_setup": n / dt,
           "fit_precision": m.last_fit_precision, "target_bytes": V.numel() * 2,
           "free_bytes_before": free, "factors_finite": bool(torch.isfinite(m.W).all() and torch.isfinite(m.H).all())}
    release_workspaces()
    del V, W0, H0, m
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--big-iters", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("half_target_rate.py needs a CUDA device")
    res = {"card": card(), "iters": a.iters, "rounds": a.rounds, "workloads": []}
    V = nmf_target(65536, 4096, 0)
    W, H = nmf_factors(65536, 4096, 64, 1)
    for prec in ("f32", "auto"):
        res["workloads"].append(workload("cfg2", NMF, V, W, H, 1.0, prec, a))
    W, H = nmf_factors(65536, 4096, 300, 2)
    res["workloads"].append(workload("r300", NMF, V, W, H, 1.0, "f32", a))
    del V, W, H
    V, W, H = nmfd_inputs(1, 1025, 8192, 16, 128, 3)
    for beta, prec in ((1.0, "auto"), (2.0, "f32")):
        res["workloads"].append(workload("cfg3", NMFD, V, W, H, beta, prec, a))
    del V, W, H
    torch.cuda.empty_cache()
    res["one_gpu_8192x2^20_r128_bf16"] = big_fit(a.big_iters)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
