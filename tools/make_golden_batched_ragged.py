"""Generate tests/golden/reference_batched_ragged.npz: ragged batches of independent NMF problems -- one shared column count,
a different row count per problem -- each fitted on its own by the UNMODIFIED reference (torchnmf 0.3.5, importable from
oracle/_ref: oracle/build_ref.py) on the CPU.

    python tools/make_golden_batched_ragged.py

Each case is B = 5 problems at one beta (0.5, 1 or 2), stored padded to N rows: V (B, N, C) and H0 / H (B, N, R), with
`lengths[b]` real rows in problem b.  Problem b's real target V[b, :L] is a rank-3 product plus uniform noise whose level
grows with b, rounded to bf16-representable values, and it is fitted by
`torchnmf.nmf.NMF(W=W0[b], H=H0[b, :L]).fit(V[b, :L], beta, tol, max_iter)`.  The padding rows of V are NaN and those of
H0 and H a sentinel (7.0): a fit of the padded batch must neither read the former nor write the latter.  The tolerance of
each case is chosen so that the problems stop at different iteration counts; the counts are stored with the factors.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.make_golden import GOLD  # noqa: E402  (imports the reference)
from torchnmf.nmf import NMF  # noqa: E402

B, N, C, R = 5, 48, 36, 6
LENGTHS = [48, 17, 31, 5, 40]
SENTINEL = 7.0


def inputs(seed):
    g = torch.Generator().manual_seed(seed)
    Ht = torch.rand(B, N, 3, generator=g)
    Wt = torch.rand(B, C, 3, generator=g)
    noise = torch.rand(B, N, C, generator=g) * torch.tensor([0.02, 0.2, 0.6, 1.0, 1.5]).view(B, 1, 1)
    V = (Ht @ Wt.transpose(1, 2) + noise + 0.01).bfloat16().float()
    W0 = torch.randn(B, C, R, generator=g).abs()
    H0 = torch.randn(B, N, R, generator=g).abs()
    for b, L in enumerate(LENGTHS):
        V[b, L:] = float("nan")
        H0[b, L:] = SENTINEL
    return V, W0, H0


def cases():
    """name -> (beta, tol, max_iter, seed)"""
    return {"b0.5": (0.5, 2e-3, 200, 20), "b1": (1, 1e-3, 200, 21), "b2": (2, 5e-4, 200, 22)}


def main():
    torch.set_num_threads(1)                # deterministic reduction order
    flat = {}
    for name, (beta, tol, max_iter, seed) in cases().items():
        V, W0, H0 = inputs(seed)
        Ws, its = [], []
        H = H0.clone()
        for b, L in enumerate(LENGTHS):
            m = NMF(W=W0[b], H=H0[b, :L])
            its.append(m.fit(V[b, :L], beta=beta, tol=tol, max_iter=max_iter))
            Ws.append(m.W.detach().clone())
            H[b, :L] = m.H.detach()
        rec = dict(V=V, W0=W0, H0=H0, W=torch.stack(Ws), H=H)
        for k, v in rec.items():
            flat[f"{name}/{k}"] = v.numpy()
        flat[f"{name}/n_iter"] = np.array(its, dtype=np.int64)
        flat[f"{name}/lengths"] = np.array(LENGTHS, dtype=np.int64)
        for k, v in dict(beta=beta, tol=tol, max_iter=max_iter).items():
            flat[f"{name}/{k}"] = np.array(v, dtype=np.float64)
        print(name, "n_iter", its)
    path = os.path.join(GOLD, "reference_batched_ragged.npz")
    np.savez_compressed(path, **flat)
    print(f"wrote {path} ({os.path.getsize(path) / 1e6:.2f} MB)")


if __name__ == "__main__":
    main()
