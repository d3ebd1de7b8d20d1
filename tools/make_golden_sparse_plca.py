"""Generate tests/golden/reference_sparse_plca.npz: PLCA fits of sparse count matrices through the UNMODIFIED reference
(torchnmf 0.3.5, importable from oracle/_ref: oracle/build_ref.py), on the CPU in float64.

    python tools/make_golden_sparse_plca.py

The reference's PLCA takes dense targets only, so each case stores its target as COO triplets (rows, cols, vals, explicit
zeros included) and runs `PLCA(W=W0, H=H0, Z=Z0, ...).fit(V.to_dense(), tol, iters, False, W_alpha, H_alpha, Z_alpha)` in
float64 (the default dtype is set so that the module's parameters are).  Inputs: the stored cells and their Poisson counts
from seed 0, W0 / H0 = |randn| and Z0 = rand + 0.1 from seed 1 (as the PLCA cases of oracle/make_golden.py).  The cases
are small enough to keep the file small: one 400 x 300 case at 2 %, the others 200 x 150 at 4 %, and the rank-300 case
24 x 20 (its dot products still span two blocks of 256 components).  Indices are stored as int32.  Tensor alphas are
0-d: the reference takes no other tensor alpha (`alpha != 1` must be one bool).
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.make_golden import GOLD  # noqa: E402  (imports the reference)
import torchnmf.plca as ref_plca  # noqa: E402


def cases():
    """name -> (N, C, R, density, target recipe, iterations, tol, ctor kw, alphas (W, H, Z), tensor alphas)"""
    inf = float("-inf")
    one = (1.0, 1.0, 1.0)
    return {
        "poisson": (400, 300, 8, 0.02, "counts", 50, inf, {}, one, False),
        "empty": (200, 150, 8, 0.04, "empty", 40, inf, {}, one, False),
        "frozenW": (200, 150, 8, 0.04, "counts", 30, inf, dict(trainable_W=False), one, False),
        "alpha": (200, 150, 8, 0.04, "counts", 30, inf, {}, (1.05, 1.02, 1.1), False),
        "alpha_tensor": (200, 150, 8, 0.04, "counts", 30, inf, {}, (0.999, 1.01, 0.95), True),
        "tol": (200, 150, 8, 0.04, "counts", 300, 1e-3, {}, one, False),
        "r300": (24, 20, 300, 0.3, "counts", 20, inf, {}, one, False),
    }


def target(N, C, density, recipe):
    """(rows, cols, vals) of a coalesced COO target: Poisson counts, all positive for "counts"; for "empty", rows 0-19 and
    columns 0-14 store nothing and the counts include explicit zeros."""
    g = torch.Generator().manual_seed(0)
    stored = torch.rand(N, C, generator=g, dtype=torch.float64) < density
    if recipe == "counts":
        vals = 1.0 + torch.poisson(torch.full((N, C), 2.0, dtype=torch.float64), generator=g)
    else:
        stored[:20] = False
        stored[:, :15] = False
        vals = torch.poisson(torch.full((N, C), 1.0, dtype=torch.float64), generator=g)
    rows, cols = stored.nonzero(as_tuple=True)
    return rows, cols, vals[rows, cols]


def inputs(N, C, R):
    torch.manual_seed(1)
    W0, H0 = torch.randn(C, R, dtype=torch.float32).abs(), torch.randn(N, R, dtype=torch.float32).abs()
    Z0 = torch.rand(R, dtype=torch.float32) + 0.1
    return W0, H0, Z0


def main():
    torch.set_num_threads(1)                # deterministic reduction order
    torch.set_default_dtype(torch.float64)  # the reference's modules run in float64
    flat = {}
    for name, (N, C, R, density, recipe, iters, tol, kw, alphas, tensor_alpha) in cases().items():
        rows, cols, vals = target(N, C, density, recipe)
        V = torch.zeros(N, C, dtype=torch.float64)
        V[rows, cols] = vals
        W0, H0, Z0 = inputs(N, C, R)
        m = ref_plca.PLCA(W=W0.double(), H=H0.double(), Z=Z0.double(), **kw)
        assert m.W.dtype == torch.float64
        fit_alphas = tuple(torch.tensor(a, dtype=torch.float64) for a in alphas) if tensor_alpha else alphas
        n_iter, norm = m.fit(V, tol, iters, False, *fit_alphas)
        arrays = dict(rows=rows.int(), cols=cols.int(), vals=vals.float(), W0=W0, H0=H0, Z0=Z0, W=m.W.detach(),
                      H=m.H.detach(), Z=m.Z.detach())
        for k, v in arrays.items():
            flat[f"{name}/{k}"] = v.numpy()
        meta = dict(N=N, C=C, n_iter=n_iter, norm=float(norm), iters=iters, tol=tol, W_alpha=alphas[0], H_alpha=alphas[1],
                    Z_alpha=alphas[2], tensor_alpha=int(tensor_alpha),
                    **{k: int(kw.get(k, True)) for k in ("trainable_W", "trainable_H", "trainable_Z")})
        for k, v in meta.items():
            flat[f"{name}/{k}"] = np.array(v, dtype=np.float64)
        print(name, "nnz", len(vals), "zeros", int((vals == 0).sum()), "n_iter", n_iter, "norm", float(norm))
    path = os.path.join(GOLD, "reference_sparse_plca.npz")
    np.savez_compressed(path, **flat)
    print(f"wrote {path} ({os.path.getsize(path) / 1e6:.2f} MB)")


if __name__ == "__main__":
    main()
