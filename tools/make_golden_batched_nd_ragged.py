"""Generate tests/golden/reference_batched_nd_ragged.npz: ragged batches of independent NMFD / NMF2D / NMF3D problems -- one
shape but for the length of the last convolved axis, which differs per problem -- each fitted on its own real positions by
the UNMODIFIED reference (torchnmf 0.3.5, importable from oracle/_ref: oracle/build_ref.py) on the CPU.

    python tools/make_golden_batched_nd_ragged.py

Each case is P = 4 problems at one beta: NMFD at 0.5, 1 and 2, NMF2D at 1 and NMF3D at 2.  They are stored padded to the
longest length X_last: V (P, B, C, *X) and H0 / H (P, B, R, *(X - K + 1)), with `lengths[p]` real positions of V[p] along
the last axis and lengths[p] - K_last + 1 of H[p].  Problem p's real target is a low-rank convolutive product plus uniform
noise whose level grows with p, rounded to bf16-representable values, and it is fitted by
`torchnmf.nmf.NMFD(W=W0[p], H=H0[p, ..., :L - K_last + 1]).fit(V[p, ..., :L], beta, tol, max_iter)` (NMF2D / NMF3D alike).
The padding of V is NaN and that of H0 and H a sentinel (7.0): a fit of the padded batch must neither read the former nor
write the latter.  The tolerance of each case is chosen so that the problems stop at different iteration counts; the counts
are stored with the factors.
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
SENTINEL = 7.0
MODELS = {"nmfd": (NMFD, F.conv1d), "nmf2d": (NMF2D, F.conv2d), "nmf3d": (NMF3D, F.conv3d)}


def cases():
    """name -> (model, B, C, X (padded), R, K, lengths, beta, tol, max_iter, seed)"""
    return {
        "nmfd_b0.5": ("nmfd", 2, 12, (40,), 4, (5,), [40, 17, 5, 29], 0.5, 2e-3, 200, 30),
        "nmfd_b1": ("nmfd", 2, 12, (40,), 4, (5,), [40, 17, 5, 29], 1, 1e-3, 200, 31),
        "nmfd_b2": ("nmfd", 2, 12, (40,), 4, (5,), [40, 17, 5, 29], 2, 5e-4, 200, 32),
        "nmf2d_b1": ("nmf2d", 2, 5, (9, 14), 3, (2, 4), [14, 6, 4, 11], 1, 1e-3, 200, 36),
        "nmf3d_b2": ("nmf3d", 1, 4, (5, 6, 9), 3, (2, 2, 3), [9, 3, 7, 5], 2, 5e-4, 200, 34),
    }


def inputs(model, B, C, X, R, K, lengths, seed):
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
    for p, L in enumerate(lengths):
        V[p, ..., L:] = float("nan")
        H0[p, ..., L - K[-1] + 1:] = SENTINEL
    return V, W0, H0


def main():
    torch.set_num_threads(1)                # deterministic reduction order
    flat = {}
    for name, (model, B, C, X, R, K, lengths, beta, tol, max_iter, seed) in cases().items():
        V, W0, H0 = inputs(model, B, C, X, R, K, lengths, seed)
        Ws, its = [], []
        H = H0.clone()
        for p, L in enumerate(lengths):
            lin = L - K[-1] + 1
            m = MODELS[model][0](W=W0[p], H=H0[p, ..., :lin].contiguous())
            its.append(m.fit(V[p, ..., :L].contiguous(), beta=beta, tol=tol, max_iter=max_iter))
            Ws.append(m.W.detach().clone())
            H[p, ..., :lin] = m.H.detach()
        rec = dict(V=V, W0=W0, H0=H0, W=torch.stack(Ws), H=H)
        for k, v in rec.items():
            flat[f"{name}/{k}"] = v.numpy()
        flat[f"{name}/n_iter"] = np.array(its, dtype=np.int64)
        flat[f"{name}/lengths"] = np.array(lengths, dtype=np.int64)
        for k, v in dict(beta=beta, tol=tol, max_iter=max_iter).items():
            flat[f"{name}/{k}"] = np.array(v, dtype=np.float64)
        print(name, "n_iter", its)
    path = os.path.join(GOLD, "reference_batched_nd_ragged.npz")
    np.savez_compressed(path, **flat)
    print(f"wrote {path} ({os.path.getsize(path) / 1e6:.2f} MB)")


if __name__ == "__main__":
    main()
