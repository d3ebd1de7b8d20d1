"""Generate tests/golden/reference_masked.npz: fits on the observed cells of the target only, through the UNMODIFIED
reference (torchnmf 0.3.5, importable from oracle/_ref: oracle/build_ref.py), on the CPU.

    python tools/make_golden_masked.py

The reference has no masked `fit`; its own way to fit the observed cells is `trainer.BetaMu` with a closure that selects
them.  Each case runs

    opt = torchnmf.trainer.BetaMu([model.W, model.H], beta, l1_reg, l2_reg)
    def closure():
        opt.zero_grad()
        return V[M], model()[M]
    opt.step(closure)                                           # W then H, every iteration

from the same initial factors as oracle/make_golden.py (V = rand rounded to bf16-representable values from seed 0, W0 / H0 =
|randn| from seed 1; the mask from seed 2), with fit()'s loop around it: the loss sqrt(2 beta_div(model()[M], V[M])) before
the first and after every 10th iteration, and the stop rule of nmf.py:405.  BetaMu adds eps after l1 / l2 where fit()
adds it before: the same numbers at alpha = 0, a rounding apart otherwise.  Every field is stored whole (the cases are
small); V holds NaN at the missing cells of the `nan` cases, which a masked fit must never read.
"""
import math
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.make_golden import GOLD, make_inputs, ref_nmf  # noqa: E402  (imports the reference)
from torchnmf.metrics import beta_div  # noqa: E402
from torchnmf.trainer import BetaMu  # noqa: E402


def random_mask(shape, missing, seed=2):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(*shape, generator=g) >= missing


def run_masked_reference(cls, V, M, W0, H0, beta, tol, max_iter, alpha, l1_ratio, trainable_W=True, trainable_H=True):
    m = cls(W=W0, H=H0, trainable_W=trainable_W, trainable_H=trainable_H)
    opt = BetaMu([m.W, m.H], beta, alpha * l1_ratio, alpha * (1 - l1_ratio))
    Vo = V[M]

    def closure():
        opt.zero_grad()                     # the reference's own idiom (its tests/test_trainer.py): no gradient carried over
        return Vo, m()[M]

    def loss():
        with torch.no_grad():
            return math.sqrt(2.0 * float(beta_div(m()[M], Vo, beta)))

    loss_init = previous = loss()
    losses = [loss_init]
    n_iter = -1
    for n_iter in range(max_iter):
        opt.step(closure)
        if n_iter % 10 == 9:
            cur = loss()
            losses.append(cur)
            if (previous - cur) / loss_init < tol:
                break
            previous = cur
    return m.W.detach().clone(), m.H.detach().clone(), n_iter + 1, losses


NMF_SHAPE = (97, 83, 8)                     # N, C, R: off every tile edge
ND_SHAPES = {                               # kind: (V shape, kernel size, R)
    "nmfd": ((2, 21, 61), (5,), 4),
    "nmf2d": ((2, 5, 12, 20), (2, 3), 3),
    "nmf3d": ((1, 3, 6, 7, 16), (2, 2, 3), 3),
}
CLS = {"nmf": ref_nmf.NMF, "nmfd": ref_nmf.NMFD, "nmf2d": ref_nmf.NMF2D, "nmf3d": ref_nmf.NMF3D}


def cases():
    """name -> (kind, mask recipe, beta, tol, max_iter, alpha, l1_ratio, trainable_W, nan at the missing cells)"""
    out = {}
    for beta in (0, 0.5, 1, 1.5, 2):
        out[f"nmf_rand30_b{beta}"] = ("nmf", "rand30", beta, float("-inf"), 20, 0.0, 0.0, True, beta == 1)
    out["nmf_rowcol_b1"] = ("nmf", "rowcol", 1, float("-inf"), 20, 0.0, 0.0, True, True)
    out["nmf_rowcol_b0.5"] = ("nmf", "rowcol", 0.5, float("-inf"), 20, 0.0, 0.0, True, False)
    out["nmf_rand30_b1.5_alpha"] = ("nmf", "rand30", 1.5, float("-inf"), 20, 0.1, 0.5, True, False)
    out["nmf_rand30_b1_frozenW"] = ("nmf", "rand30", 1, float("-inf"), 20, 0.0, 0.0, False, False)
    out["nmf_rand30_b1_tol"] = ("nmf", "rand30", 1, 1e-2, 200, 0.0, 0.0, True, False)
    for beta in (1, 0.5, 2):
        out[f"nmfd_rand30_b{beta}"] = ("nmfd", "rand30", beta, float("-inf"), 20, 0.0, 0.0, True, beta == 1)
    for beta in (1, 0):
        out[f"nmf2d_rand30_b{beta}"] = ("nmf2d", "rand30", beta, float("-inf"), 20, 0.0, 0.0, True, False)
    out["nmf3d_rand30_b1.5"] = ("nmf3d", "rand30", 1.5, float("-inf"), 20, 0.0, 0.0, True, False)
    return out


def inputs(kind, recipe, beta):
    floor = 2 ** -7 if beta <= 0 else 0.0
    if kind == "nmf":
        N, C, R = NMF_SHAPE
        V, W0, H0 = make_inputs((N, C), (C, R), (N, R), floor=floor)
    else:
        vs, ks, R = ND_SHAPES[kind]
        B, C, X = vs[0], vs[1], vs[2:]
        V, W0, H0 = make_inputs(vs, (C, R, *ks), (B, R, *(x - k + 1 for x, k in zip(X, ks))), floor=floor)
    if recipe == "rand30":
        M = random_mask(V.shape, 0.3)
    else:                                   # 10 % at random, whole rows and whole columns, two of each fully missing
        M = random_mask(V.shape, 0.1)
        M[5] = False
        M[60] = False
        M[:, 7] = False
        M[:, 50] = False
    return V, M, W0, H0


def main():
    torch.set_num_threads(1)                # deterministic reduction order
    flat = {}
    for name, (kind, recipe, beta, tol, iters, alpha, l1r, tw, nan) in cases().items():
        V, M, W0, H0 = inputs(kind, recipe, beta)
        if nan:
            V = V.masked_fill(~M, float("nan"))
        W, H, n_iter, losses = run_masked_reference(CLS[kind], V, M, W0, H0, beta, tol, iters, alpha, l1r, trainable_W=tw)
        rec = dict(V=V, M=M, W0=W0, H0=H0, W=W, H=H)
        for k, v in rec.items():
            flat[f"{name}/{k}"] = v.numpy()
        flat[f"{name}/kind"] = np.array(kind)
        flat[f"{name}/losses"] = np.array(losses, dtype=np.float64)
        meta = dict(n_iter=n_iter, beta=beta, tol=tol, max_iter=iters, alpha=alpha, l1_ratio=l1r, trainable_W=int(tw))
        for k, v in meta.items():
            flat[f"{name}/{k}"] = np.array(v, dtype=np.float64)
        print(name, "n_iter", n_iter, "loss", losses[-1])
    path = os.path.join(GOLD, "reference_masked.npz")
    np.savez_compressed(path, **flat)
    print(f"wrote {path} ({os.path.getsize(path) / 1e6:.2f} MB)")


if __name__ == "__main__":
    main()
