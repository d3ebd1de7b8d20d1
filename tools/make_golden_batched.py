"""Generate tests/golden/reference_batched.npz: batches of independent NMF problems, each fitted on its own by the UNMODIFIED
reference (torchnmf 0.3.5, importable from oracle/_ref: oracle/build_ref.py) on the CPU.

    python tools/make_golden_batched.py

Each case is B = 4 problems of one shape at one beta (0.5, 1 or 2).  Problem b has its own target V[b] (a rank-3 product
plus uniform noise whose level grows with b, rounded to bf16-representable values) and its own initial factors W0[b] / H0[b]
(|randn|), and is fitted by `torchnmf.nmf.NMF(W=W0[b], H=H0[b]).fit(V[b], beta, tol, max_iter)`.  The tolerance of each
case is chosen so that the problems stop at different iteration counts; the counts are stored with the factors.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.make_golden import GOLD  # noqa: E402  (imports the reference)
from torchnmf.nmf import NMF  # noqa: E402

B, N, C, R = 4, 48, 36, 6


def inputs(seed):
    g = torch.Generator().manual_seed(seed)
    Ht = torch.rand(B, N, 3, generator=g)
    Wt = torch.rand(B, C, 3, generator=g)
    noise = torch.rand(B, N, C, generator=g) * torch.tensor([0.02, 0.2, 0.6, 1.5]).view(B, 1, 1)
    V = (Ht @ Wt.transpose(1, 2) + noise + 0.01).bfloat16().float()
    W0 = torch.randn(B, C, R, generator=g).abs()
    H0 = torch.randn(B, N, R, generator=g).abs()
    return V, W0, H0


def cases():
    """name -> (beta, tol, max_iter, seed)"""
    return {"b0.5": (0.5, 2e-3, 200, 10), "b1": (1, 1e-3, 200, 11), "b2": (2, 5e-4, 200, 12)}


def main():
    torch.set_num_threads(1)                # deterministic reduction order
    flat = {}
    for name, (beta, tol, max_iter, seed) in cases().items():
        V, W0, H0 = inputs(seed)
        Ws, Hs, its = [], [], []
        for b in range(B):
            m = NMF(W=W0[b], H=H0[b])
            its.append(m.fit(V[b], beta=beta, tol=tol, max_iter=max_iter))
            Ws.append(m.W.detach().clone())
            Hs.append(m.H.detach().clone())
        rec = dict(V=V, W0=W0, H0=H0, W=torch.stack(Ws), H=torch.stack(Hs))
        for k, v in rec.items():
            flat[f"{name}/{k}"] = v.numpy()
        flat[f"{name}/n_iter"] = np.array(its, dtype=np.int64)
        for k, v in dict(beta=beta, tol=tol, max_iter=max_iter).items():
            flat[f"{name}/{k}"] = np.array(v, dtype=np.float64)
        print(name, "n_iter", its)
    path = os.path.join(GOLD, "reference_batched.npz")
    np.savez_compressed(path, **flat)
    print(f"wrote {path} ({os.path.getsize(path) / 1e6:.2f} MB)")


if __name__ == "__main__":
    main()
