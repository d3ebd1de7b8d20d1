"""Generate tests/golden/reference_masked_plca.npz: PLCA / SIPLCA / SIPLCA2 / SIPLCA3 fits on partially observed targets,
through the UNMODIFIED reference (torchnmf 0.3.5, importable from oracle/_ref: oracle/build_ref.py), on the CPU in float64.

    python tools/make_golden_masked_plca.py

The reference's PLCA `fit` takes no mask.  Each iteration of the missing-data EM is its EM step on the completed target, so
every case builds one reference module from W0 / H0 / Z0 (float64: the default dtype is set so that its parameters are) and
runs, each iteration,

    q = module()                                   # the reference's own reconstruction, summing to 1
    Vt = where(M, q_O V / sum_O V, q)              # q_O = sum_O q: the expected complete data
    module.fit(Vt, tol=-inf, max_iter=1, W_alpha=..., H_alpha=..., Z_alpha=...)

with the loss sqrt(2 sum_O [v (log(v + eps) - log(x + eps)) - v + x]), x = q sum_O V / q_O, before the first iteration and
after every 10th, and the reference's stop rule, applied here.  norm = sum_O V / q_O at the final factors.  Inputs: V = 3 x
rand rounded to bf16-representable values from seed 0, W0 / H0 = |randn| and Z0 = rand + 0.1 from seed 1 (as the PLCA cases
of oracle/make_golden.py), the mask from seed 2.  V holds NaN at the missing cells of the `nan` case, which a masked fit
must never read.  Tensor alphas are 0-d: the reference takes no other tensor alpha (`alpha != 1` must be one bool).
"""
import math
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.make_golden import GOLD  # noqa: E402  (imports the reference)
import torchnmf.plca as ref_plca  # noqa: E402
from torchnmf.constants import eps as EPS  # noqa: E402

SHAPES = {                          # model: (V shape, kernel size, R); the ND shapes are tools/make_golden_masked.py's
    "PLCA": ((97, 83), (), 8),
    "SIPLCA": ((2, 21, 61), (5,), 4),
    "SIPLCA2": ((2, 5, 12, 20), (2, 3), 3),
    "SIPLCA3": ((1, 3, 6, 7, 16), (2, 2, 3), 3),
}
CLS_ID = {"PLCA": 0, "SIPLCA": 1, "SIPLCA2": 2, "SIPLCA3": 3}


def cases():
    """name -> (model, R (None: SHAPES'), mask recipe, iterations, tol, ctor kw, alphas (W, H, Z), tensor alphas, nan)"""
    inf = float("-inf")
    one = (1.0, 1.0, 1.0)
    return {
        "plca_rand30": ("PLCA", None, "rand30", 50, inf, {}, one, False, False),
        "plca_gap": ("PLCA", None, "gap", 30, inf, {}, one, False, False),
        "plca_frozenW": ("PLCA", None, "rand30", 30, inf, dict(trainable_W=False), one, False, False),
        "plca_alpha": ("PLCA", None, "rand30", 30, inf, {}, (1.05, 1.02, 1.1), False, False),
        "plca_alpha_tensor": ("PLCA", None, "rand30", 30, inf, {}, (0.999, 1.01, 0.95), True, False),
        "plca_tol": ("PLCA", None, "rand30", 300, 1e-3, {}, one, False, False),
        "plca_all": ("PLCA", None, "all", 30, inf, {}, one, False, False),
        "plca_nan": ("PLCA", None, "rand30", 30, inf, {}, one, False, True),
        "plca_r300": ("PLCA", 300, "rand30", 20, inf, {}, one, False, False),
        "siplca_rand30": ("SIPLCA", None, "rand30", 30, inf, {}, one, False, False),
        "siplca2_rand30": ("SIPLCA2", None, "rand30", 20, inf, {}, one, False, False),
        "siplca3_rand30": ("SIPLCA3", None, "rand30", 20, inf, {}, one, False, False),
    }


def inputs(model, R):
    vs, ks, R0 = SHAPES[model]
    R = R or R0
    torch.manual_seed(0)
    V = torch.rand(*vs, dtype=torch.float32).bfloat16().float() * 3
    torch.manual_seed(1)
    if model == "PLCA":
        N, C = vs
        W0, H0 = torch.randn(C, R, dtype=torch.float32).abs(), torch.randn(N, R, dtype=torch.float32).abs()
    else:
        B, C, *X = vs
        W0 = torch.randn(C, R, *ks, dtype=torch.float32).abs()
        H0 = torch.randn(B, R, *(x - k + 1 for x, k in zip(X, ks)), dtype=torch.float32).abs()
    Z0 = torch.rand(R, dtype=torch.float32) + 0.1
    return V, W0, H0, Z0


def make_mask(shape, recipe):
    if recipe == "all":
        return torch.ones(shape, dtype=torch.bool)
    g = torch.Generator().manual_seed(2)
    if recipe == "rand30":
        return torch.rand(*shape, generator=g, dtype=torch.float32) >= 0.3
    M = torch.rand(*shape, generator=g, dtype=torch.float32) >= 0.05        # "gap": 5 % at random and 16 whole columns
    M[:, 30:46] = False
    return M


def observed_loss(V, M, q):
    v = V[M]
    qo = torch.where(M, q, torch.zeros((), dtype=q.dtype)).sum()
    x = (q * (v.sum() / qo))[M]
    d = float((v * (torch.log(v + EPS) - torch.log(x + EPS)) - v + x).sum())
    return math.sqrt(2.0 * d) if d >= 0 else float("nan")


def run(model, V, M, W0, H0, Z0, iters, tol, kw, alphas):
    m = getattr(ref_plca, model)(W=W0.double(), H=H0.double(), Z=Z0.double(), **kw)
    assert m.W.dtype == torch.float64
    Vo = torch.where(M, V.double(), torch.zeros((), dtype=torch.float64))
    Vn = Vo / Vo.sum()
    W_alpha, H_alpha, Z_alpha = alphas

    def model_q():
        with torch.no_grad():
            return m().detach()

    loss_init = previous = observed_loss(Vo, M, model_q())
    losses = [loss_init]
    n_iter = -1
    for n_iter in range(iters):
        q = model_q()
        qo = torch.where(M, q, torch.zeros((), dtype=q.dtype)).sum()
        Vt = torch.where(M, qo * Vn, q)
        m.fit(Vt, float("-inf"), 1, False, W_alpha, H_alpha, Z_alpha)
        if n_iter % 10 == 9:
            cur = observed_loss(Vo, M, model_q())
            losses.append(cur)
            if (previous - cur) / loss_init < tol:
                break
            previous = cur
    q = model_q()
    norm = float(Vo.sum() / torch.where(M, q, torch.zeros((), dtype=q.dtype)).sum())
    return m.W.detach().clone(), m.H.detach().clone(), m.Z.detach().clone(), n_iter, norm, losses


def main():
    torch.set_num_threads(1)                # deterministic reduction order
    torch.set_default_dtype(torch.float64)  # the reference's modules run in float64
    flat = {}
    for name, (model, R, recipe, iters, tol, kw, alphas, tensor_alpha, nan) in cases().items():
        V, W0, H0, Z0 = inputs(model, R)
        M = make_mask(V.shape, recipe)
        if nan:
            V = V.masked_fill(~M, float("nan"))
        fit_alphas = tuple(torch.tensor(a, dtype=torch.float64) for a in alphas) if tensor_alpha else alphas
        W, H, Z, n_iter, norm, losses = run(model, V, M, W0, H0, Z0, iters, tol, kw, fit_alphas)
        for k, v in dict(V=V, M=M, W0=W0, H0=H0, Z0=Z0, W=W, H=H, Z=Z).items():
            flat[f"{name}/{k}"] = v.numpy()
        flat[f"{name}/losses"] = np.array(losses, dtype=np.float64)
        meta = dict(cls=CLS_ID[model], n_iter=n_iter, norm=norm, iters=iters, tol=tol, W_alpha=alphas[0], H_alpha=alphas[1],
                    Z_alpha=alphas[2], tensor_alpha=int(tensor_alpha),
                    **{k: int(kw.get(k, True)) for k in ("trainable_W", "trainable_H", "trainable_Z")})
        for k, v in meta.items():
            flat[f"{name}/{k}"] = np.array(v, dtype=np.float64)
        print(name, "n_iter", n_iter, "loss", losses[-1], "norm", norm)
    path = os.path.join(GOLD, "reference_masked_plca.npz")
    np.savez_compressed(path, **flat)
    print(f"wrote {path} ({os.path.getsize(path) / 1e6:.2f} MB)")


if __name__ == "__main__":
    main()
