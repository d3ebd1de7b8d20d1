"""Generate tests/golden/reference_batched_nd.npz: batches of independent NMFD / NMF2D / NMF3D problems, each fitted on its own
by the UNMODIFIED reference (torchnmf 0.3.5, importable from oracle/_ref: oracle/build_ref.py) on the CPU.

    python tools/make_golden_batched_nd.py

Each case is P = 4 problems of one shape at one beta: NMFD at 0.5, 1 and 2, NMF2D at 1 and NMF3D at 2.  Problem p has its
own target V[p] (a low-rank convolutive product plus uniform noise whose level grows with p, rounded to bf16-representable
values) and its own initial factors W0[p] / H0[p] (|randn|), and is fitted by `torchnmf.nmf.NMFD(W=W0[p], H=H0[p])
.fit(V[p], beta, tol, max_iter)` (NMF2D / NMF3D alike).  The tolerance of each case is chosen so that the problems stop at
different iteration counts; the counts are stored with the factors.
"""
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.make_golden import GOLD  # noqa: E402  (imports the reference)
from torchnmf.nmf import NMFD, NMF2D, NMF3D  # noqa: E402

P = 4
NOISE = torch.tensor([0.02, 0.2, 0.6, 1.5])
MODELS = {"nmfd": (NMFD, F.conv1d), "nmf2d": (NMF2D, F.conv2d), "nmf3d": (NMF3D, F.conv3d)}


def cases():
    """name -> (model, B, C, X, R, K, beta, tol, max_iter, seed)"""
    return {
        "nmfd_b0.5": ("nmfd", 2, 12, (40,), 4, (5,), 0.5, 2e-3, 200, 20),
        "nmfd_b1": ("nmfd", 2, 12, (40,), 4, (5,), 1, 1e-3, 200, 21),
        "nmfd_b2": ("nmfd", 2, 12, (40,), 4, (5,), 2, 5e-4, 200, 22),
        "nmf2d_b1": ("nmf2d", 2, 5, (9, 14), 3, (2, 4), 1, 1e-3, 200, 26),
        "nmf3d_b2": ("nmf3d", 1, 4, (5, 6, 9), 3, (2, 2, 3), 2, 5e-4, 200, 24),
    }


def inputs(model, B, C, X, R, K, seed):
    conv = MODELS[model][1]
    g = torch.Generator().manual_seed(seed)
    J = tuple(x - k + 1 for x, k in zip(X, K))
    Vs = []
    for p in range(P):
        Ht = torch.rand(B, 2, *J, generator=g)
        Wt = torch.rand(C, 2, *K, generator=g)
        clean = conv(Ht, Wt.flip(tuple(range(2, Wt.dim()))), padding=tuple(k - 1 for k in K))
        Vs.append(clean + torch.rand(B, C, *X, generator=g) * NOISE[p])
    V = (torch.stack(Vs) + 0.01).bfloat16().float()
    W0 = torch.randn(P, C, R, *K, generator=g).abs()
    H0 = torch.randn(P, B, R, *J, generator=g).abs()
    return V, W0, H0


def main():
    torch.set_num_threads(1)                # deterministic reduction order
    flat = {}
    for name, (model, B, C, X, R, K, beta, tol, max_iter, seed) in cases().items():
        V, W0, H0 = inputs(model, B, C, X, R, K, seed)
        Ws, Hs, its = [], [], []
        for p in range(P):
            m = MODELS[model][0](W=W0[p], H=H0[p])
            its.append(m.fit(V[p], beta=beta, tol=tol, max_iter=max_iter))
            Ws.append(m.W.detach().clone())
            Hs.append(m.H.detach().clone())
        rec = dict(V=V, W0=W0, H0=H0, W=torch.stack(Ws), H=torch.stack(Hs))
        for k, v in rec.items():
            flat[f"{name}/{k}"] = v.numpy()
        flat[f"{name}/n_iter"] = np.array(its, dtype=np.int64)
        for k, v in dict(beta=beta, tol=tol, max_iter=max_iter).items():
            flat[f"{name}/{k}"] = np.array(v, dtype=np.float64)
        print(name, "n_iter", its)
    path = os.path.join(GOLD, "reference_batched_nd.npz")
    np.savez_compressed(path, **flat)
    print(f"wrote {path} ({os.path.getsize(path) / 1e6:.2f} MB)")


if __name__ == "__main__":
    main()
