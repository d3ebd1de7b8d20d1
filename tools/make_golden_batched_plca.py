"""Generate tests/golden/reference_batched_plca.npz: batches of independent PLCA / SIPLCA / SIPLCA2 / SIPLCA3 problems, each
fitted on its own by the UNMODIFIED reference (torchnmf 0.3.5, importable from oracle/_ref: oracle/build_ref.py) on the CPU.

    python tools/make_golden_batched_plca.py

Each case is P = 4 problems of one shape.  Problem p has its own target V[p] (a low-rank product or convolution plus uniform
noise whose level grows with p, rounded to bf16-representable values) -- or, for the restarts case, one target shared by
every problem -- and its own initial factors W0[p] / H0[p] (|randn|) and Z0[p] (uniform), and is fitted by
`torchnmf.plca.PLCA(W=W0[p], H=H0[p], Z=Z0[p], trainable_*=...).fit(V[p], tol, max_iter, W_alpha=..., ...)` (SIPLCA*
alike).  The cases cover every model, scalar alphas != 1, a tensor W_alpha, frozen Z, frozen W and restarts.  The
reference takes a tensor alpha only if it is 0-d (plca.py:273 compares it with 1), so the tensor case gives problem p the 0-d
W_alpha[p]; the batched fit takes them as one (P, 1, 1) tensor.  The tolerance of each case is chosen so that the problems
stop at different iteration counts where the model allows it; the counts and norms are stored with the factors.
"""
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.make_golden import GOLD  # noqa: E402  (imports the reference)
from torchnmf.plca import PLCA, SIPLCA, SIPLCA2, SIPLCA3  # noqa: E402

P = 4
NOISE = torch.tensor([0.02, 0.2, 0.6, 1.5])
MODELS = {"plca": (PLCA, None), "siplca": (SIPLCA, F.conv1d), "siplca2": (SIPLCA2, F.conv2d),
          "siplca3": (SIPLCA3, F.conv3d)}


def cases():
    """name -> (model, B, C, X, R, K, tol, max_iter, seed, W_alpha, H_alpha, Z_alpha, train_W, train_Z, shared).
    PLCA: V (N, C) with N = X[0]; W_alpha "tensor": a 0-d tensor per problem, values in [1, 1.5]."""
    return {
        "plca": ("plca", 1, 20, (30,), 4, (), 1e-3, 200, 40, 1., 1., 1., True, True, False),
        "plca_alpha": ("plca", 1, 20, (30,), 4, (), 1e-4, 200, 41, 1.3, 1.1, 0.9, True, True, False),
        "plca_walpha_tensor": ("plca", 1, 20, (30,), 4, (), 1e-5, 200, 42, "tensor", 1., 1., True, True, False),
        "plca_frozen_z": ("plca", 1, 20, (30,), 4, (), 1e-3, 200, 43, 1., 1., 1., True, False, False),
        "plca_frozen_w": ("plca", 1, 20, (30,), 4, (), 1e-3, 200, 44, 1., 1., 1., False, True, False),
        "plca_restarts": ("plca", 1, 20, (30,), 4, (), 1e-3, 200, 45, 1., 1., 1., True, True, True),
        "siplca": ("siplca", 2, 12, (40,), 4, (5,), 1e-2, 200, 46, 1., 1., 1., True, True, False),
        "siplca2": ("siplca2", 1, 5, (9, 14), 3, (2, 4), 1e-4, 200, 47, 1., 1.2, 1., True, True, False),
        "siplca3": ("siplca3", 1, 4, (5, 6, 9), 3, (2, 2, 3), 1e-2, 200, 48, 1., 1., 1., True, True, False),
    }


def inputs(model, B, C, X, R, K, seed, shared):
    conv = MODELS[model][1]
    g = torch.Generator().manual_seed(seed)
    J = tuple(x - k + 1 for x, k in zip(X, K))
    Vs = []
    for p in range(P):
        if model == "plca":
            clean = torch.rand(X[0], 2, generator=g) @ torch.rand(2, C, generator=g)
            noise = torch.rand(X[0], C, generator=g)
        else:
            Ht = torch.rand(B, 2, *J, generator=g)
            Wt = torch.rand(C, 2, *K, generator=g)
            clean = conv(Ht, Wt.flip(tuple(range(2, Wt.dim()))), padding=tuple(k - 1 for k in K))
            noise = torch.rand(B, C, *X, generator=g)
        Vs.append(clean + noise * NOISE[1 if shared else p])
    V = (torch.stack([Vs[0]] * P if shared else Vs) + 0.01).bfloat16().float()
    if model == "plca":
        W0 = torch.randn(P, C, R, generator=g).abs()
        H0 = torch.randn(P, X[0], R, generator=g).abs()
    else:
        W0 = torch.randn(P, C, R, *K, generator=g).abs()
        H0 = torch.randn(P, B, R, *J, generator=g).abs()
    Z0 = torch.rand(P, R, generator=g) + 0.2
    Wa = 1. + 0.5 * torch.rand(P, generator=g)
    return V, W0, H0, Z0, Wa


def main():
    torch.set_num_threads(1)                # deterministic reduction order
    flat = {}
    for name, (model, B, C, X, R, K, tol, max_iter, seed, wa, ha, za, tw, tz, shared) in cases().items():
        V, W0, H0, Z0, Wa = inputs(model, B, C, X, R, K, seed, shared)
        Ws, Hs, Zs, its, norms = [], [], [], [], []
        for p in range(P):
            m = MODELS[model][0](W=W0[p], H=H0[p], Z=Z0[p], trainable_W=tw, trainable_Z=tz)
            W_alpha = Wa[p] if wa == "tensor" else wa
            n_iter, norm = m.fit(V[p], tol=tol, max_iter=max_iter, W_alpha=W_alpha, H_alpha=ha, Z_alpha=za)
            its.append(n_iter)
            norms.append(float(norm))
            Ws.append(m.W.detach().clone())
            Hs.append(m.H.detach().clone())
            Zs.append(m.Z.detach().clone())
        rec = dict(V=V, W0=W0, H0=H0, Z0=Z0, W=torch.stack(Ws), H=torch.stack(Hs), Z=torch.stack(Zs))
        if wa == "tensor":
            rec["W_alpha"] = Wa
        for k, v in rec.items():
            flat[f"{name}/{k}"] = v.numpy()
        flat[f"{name}/n_iter"] = np.array(its, dtype=np.int64)
        flat[f"{name}/norm"] = np.array(norms, dtype=np.float64)
        flat[f"{name}/model"] = np.array(model)
        scal = dict(tol=tol, max_iter=max_iter, H_alpha=ha, Z_alpha=za, trainable_W=tw, trainable_Z=tz, shared=shared)
        if wa != "tensor":
            scal["W_alpha"] = wa
        for k, v in scal.items():
            flat[f"{name}/{k}"] = np.array(v, dtype=np.float64)
        print(name, "n_iter", its)
    path = os.path.join(GOLD, "reference_batched_plca.npz")
    np.savez_compressed(path, **flat)
    print(f"wrote {path} ({os.path.getsize(path) / 1e6:.2f} MB)")


if __name__ == "__main__":
    main()
