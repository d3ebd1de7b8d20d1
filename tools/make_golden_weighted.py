"""Generate tests/golden/reference_weighted.npz: fits with integer per-cell weights, through the UNMODIFIED reference
(torchnmf 0.3.5, importable from oracle/_ref: oracle/build_ref.py), on the CPU.

    python tools/make_golden_weighted.py

The reference has no weighted `fit`; with integer weights w its own `trainer.BetaMu` expresses one by gathering each cell
w times.  Each case runs

    idx = torch.arange(V.numel()).repeat_interleave(Wt.flatten())      # cell k listed Wt[k] times
    opt = torchnmf.trainer.BetaMu([model.W, model.H], beta, l1_reg, l2_reg)
    def closure():
        opt.zero_grad()
        return V.flatten()[idx], model().flatten()[idx]
    opt.step(closure)                                                   # W then H, every iteration

so the loss is sum w d_beta(v | x) and the backward pass through the repeated gather sums each cell's terms w times.  The
inputs are those of tools/make_golden_masked.py (V rounded to bf16-representable values from seed 0, W0 / H0 = |randn| from
seed 1) with weights drawn from {0, 1, 2, 3} (seed 2), and fit()'s loop around it: the loss sqrt(2 sum w d_beta) before the
first and after every 10th iteration, and the stop rule of nmf.py:405.  V holds NaN at the zero-weight cells of the `nan`
cases, which a weighted fit must never read.
"""
import math
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from oracle.make_golden import GOLD  # noqa: E402  (imports the reference)
from make_golden_masked import CLS, inputs  # noqa: E402
from torchnmf.metrics import beta_div  # noqa: E402
from torchnmf.trainer import BetaMu  # noqa: E402


def random_weight(shape, seed=2):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 4, shape, generator=g)


def run_weighted_reference(cls, V, Wt, W0, H0, beta, tol, max_iter, alpha, l1_ratio, trainable_W=True):
    m = cls(W=W0, H=H0, trainable_W=trainable_W)
    opt = BetaMu([m.W, m.H], beta, alpha * l1_ratio, alpha * (1 - l1_ratio))
    idx = torch.arange(V.numel()).repeat_interleave(Wt.flatten())
    Vo = V.flatten()[idx]

    def closure():
        opt.zero_grad()
        return Vo, m().flatten()[idx]

    def loss():
        with torch.no_grad():
            return math.sqrt(2.0 * float(beta_div(m().flatten()[idx], Vo, beta)))

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


def cases():
    """name -> (kind, beta, tol, max_iter, alpha, l1_ratio, trainable_W, nan at the zero-weight cells)"""
    out = {}
    for beta in (0, 0.5, 1, 1.5, 2):
        out[f"nmf_w03_b{beta}"] = ("nmf", beta, float("-inf"), 20, 0.0, 0.0, True, beta in (1, 2))
    out["nmf_w03_b1.5_alpha"] = ("nmf", 1.5, float("-inf"), 20, 0.1, 0.5, True, False)
    out["nmf_w03_b1_frozenW"] = ("nmf", 1, float("-inf"), 20, 0.0, 0.0, False, False)
    out["nmf_w03_b1_tol"] = ("nmf", 1, 1e-2, 200, 0.0, 0.0, True, False)
    for beta in (1, 0.5, 2):
        out[f"nmfd_w03_b{beta}"] = ("nmfd", beta, float("-inf"), 20, 0.0, 0.0, True, beta == 1)
    for beta in (1, 0):
        out[f"nmf2d_w03_b{beta}"] = ("nmf2d", beta, float("-inf"), 20, 0.0, 0.0, True, False)
    out["nmf3d_w03_b1.5"] = ("nmf3d", 1.5, float("-inf"), 20, 0.0, 0.0, True, False)
    return out


def main():
    torch.set_num_threads(1)                # deterministic reduction order
    flat = {}
    for name, (kind, beta, tol, iters, alpha, l1r, tw, nan) in cases().items():
        V, _, W0, H0 = inputs(kind, "rand30", beta)
        Wt = random_weight(V.shape)
        if nan:
            V = V.masked_fill(Wt == 0, float("nan"))
        W, H, n_iter, losses = run_weighted_reference(CLS[kind], V, Wt, W0, H0, beta, tol, iters, alpha, l1r, trainable_W=tw)
        rec = dict(V=V, Wt=Wt.float(), W0=W0, H0=H0, W=W, H=H)
        for k, v in rec.items():
            flat[f"{name}/{k}"] = v.numpy()
        flat[f"{name}/kind"] = np.array(kind)
        flat[f"{name}/losses"] = np.array(losses, dtype=np.float64)
        meta = dict(n_iter=n_iter, beta=beta, tol=tol, max_iter=iters, alpha=alpha, l1_ratio=l1r, trainable_W=int(tw))
        for k, v in meta.items():
            flat[f"{name}/{k}"] = np.array(v, dtype=np.float64)
        print(name, "n_iter", n_iter, "loss", losses[-1])
    path = os.path.join(GOLD, "reference_weighted.npz")
    np.savez_compressed(path, **flat)
    print(f"wrote {path} ({os.path.getsize(path) / 1e6:.2f} MB)")


if __name__ == "__main__":
    main()
