"""Generate tests/golden/reference_observed.npz: fits on the observed cells of a SPARSE target, with the observed cells given
as a sparse mask, through the UNMODIFIED reference (torchnmf 0.3.5, importable from oracle/_ref: oracle/build_ref.py), on
the CPU.

    python tools/make_golden_observed.py

The reference fits the observed cells with `trainer.BetaMu` and a closure that selects them; on a sparse target that closure
reads the densified target, so an observed cell V does not store counts as an observed zero:

    opt = torchnmf.trainer.BetaMu([model.W, model.H], beta, l1_reg, l2_reg)
    def closure():
        opt.zero_grad()
        return V.to_dense()[M], model()[M]
    opt.step(closure)                                           # W then H, every iteration

with fit()'s loop around it (tools/make_golden_masked.py: run_masked_reference).  The targets are V of
oracle/make_golden.py (seed 0, bf16-representable) kept at a random 35 % of the cells (seed 3), so many observed cells are
unstored zeros and many stored entries lie outside the mask (seed 2, 45 % observed).  Row 4 and column 9 of the mask are
empty, and V stores nothing in row 17 and column 30, where the mask observes cells.  Fields: V (dense, the values of the
sparse target), S (where the sparse target stores an entry), M (the dense mask), W0 / H0, W / H, losses and the metadata.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from make_golden_masked import random_mask, run_masked_reference  # noqa: E402  (imports the reference)
from oracle.make_golden import GOLD, make_inputs, ref_nmf  # noqa: E402

SHAPE = (71, 53, 6)                         # N, C, R: off every warp and block edge


def cases():
    """name -> (beta, max_iter, alpha, l1_ratio, trainable_W)"""
    out = {f"obs_b{beta}": (beta, 20, 0.0, 0.0, True) for beta in (1, 0.5, 2)}
    out["obs_b1_alpha"] = (1, 20, 0.1, 0.5, True)
    out["obs_b0.5_frozenW"] = (0.5, 20, 0.0, 0.0, False)
    return out


def inputs():
    N, C, R = SHAPE
    V, W0, H0 = make_inputs((N, C), (C, R), (N, R))
    g = torch.Generator().manual_seed(3)
    S = torch.rand(N, C, generator=g) < 0.35
    S[17] = False
    S[:, 30] = False
    V = V * S
    M = random_mask((N, C), 0.55)
    M[4] = False
    M[:, 9] = False
    return V, S, M, W0, H0


def main():
    torch.set_num_threads(1)                # deterministic reduction order
    V, S, M, W0, H0 = inputs()
    Vs = torch.sparse_coo_tensor(S.nonzero().t(), V[S], V.shape).coalesce()
    flat = {}
    for name, (beta, iters, alpha, l1r, tw) in cases().items():
        Vd = Vs.to_dense()                  # the closure's V.to_dense()[M]
        W, H, n_iter, losses = run_masked_reference(ref_nmf.NMF, Vd, M, W0, H0, beta, float("-inf"), iters, alpha, l1r,
                                                    trainable_W=tw)
        for k, v in dict(V=V, S=S, M=M, W0=W0, H0=H0, W=W, H=H).items():
            flat[f"{name}/{k}"] = v.numpy()
        flat[f"{name}/losses"] = np.array(losses, dtype=np.float64)
        meta = dict(n_iter=n_iter, beta=beta, tol=float("-inf"), max_iter=iters, alpha=alpha, l1_ratio=l1r, trainable_W=int(tw))
        for k, v in meta.items():
            flat[f"{name}/{k}"] = np.array(v, dtype=np.float64)
        print(name, "n_iter", n_iter, "loss", losses[-1])
    path = os.path.join(GOLD, "reference_observed.npz")
    np.savez_compressed(path, **flat)
    print(f"wrote {path} ({os.path.getsize(path) / 1e6:.2f} MB)")


if __name__ == "__main__":
    main()
