"""Generate tests/golden/reference_batched_plca_ragged.npz: ragged batches of independent PLCA problems, each fitted on its own
real rows by the UNMODIFIED reference (torchnmf 0.3.5, importable from oracle/_ref: oracle/build_ref.py) on the CPU, in
float64.

    python tools/make_golden_batched_plca_ragged.py

Each case is P = 4 problems padded to N = 30 rows over C = 20 columns, rank 4.  Problem p has L[p] real rows: its target
V[p, :L[p]] (a rank-2 product plus uniform noise whose level grows with p, rounded to bf16-representable values), and its
initial factors W0[p] (|randn|), H0[p, :L[p]] (|randn|) and Z0[p] (uniform).  The padding rows of V are NaN and those of H0
zero, so the batched constructor normalises each problem's H0 over its real rows.  Problem p is fitted by
`torchnmf.plca.PLCA(W=W0[p], H=H0[p, :L[p]], Z=Z0[p], trainable_*=...).fit(V[p, :L[p]], tol, max_iter, W_alpha=..., ...)`
with every tensor in float64.  The cases cover scalar alphas != 1, a tensor W_alpha (a 0-d tensor per problem: the
reference compares alpha with 1, so the batched fit takes them as one (P, 1, 1) tensor), frozen Z, frozen W, a problem of
one row, a problem of N rows, and tolerances at which the problems stop at different counts.  The counts and norms are
stored with the factors (the padding rows of the stored H are zero).
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.make_golden import GOLD  # noqa: E402  (imports the reference)
from torchnmf.plca import PLCA  # noqa: E402

P, N, C, R = 4, 30, 20, 4
NOISE = torch.tensor([0.02, 0.2, 0.6, 1.5])


def cases():
    """name -> (lengths, tol, max_iter, seed, W_alpha, H_alpha, Z_alpha, train_W, train_Z); W_alpha "tensor": a 0-d tensor
    per problem, values in [1, 1.5].  A problem of at most R rows can be fitted exactly: its loss falls towards 0, where the
    stop rule's relative decrease is fp32 rounding, so problems of one row run to max_iter (tol = -1)."""
    return {
        "plain": ([30, 6, 17, 24], 1e-3, 200, 60, 1., 1., 1., True, True),
        "alpha": ([12, 30, 7, 25], 1e-4, 200, 61, 1.3, 1.1, 0.9, True, True),
        "walpha_tensor": ([30, 8, 21, 11], 1e-5, 200, 62, "tensor", 1., 1., True, True),
        "frozen_z": ([19, 30, 5, 27], 1e-3, 200, 63, 1., 1., 1., True, False),
        "frozen_w": ([9, 14, 30, 22], 1e-3, 200, 64, 1., 1., 1., False, True),
        "stops": ([26, 30, 9, 18], 3e-4, 200, 65, 1., 1., 1., True, True),
        "one_row": ([1, 30, 1, 13], -1.0, 40, 66, 1., 1., 1., True, True),
    }


def inputs(lengths, seed):
    g = torch.Generator().manual_seed(seed)
    V = torch.full((P, N, C), float("nan"))
    H0 = torch.zeros(P, N, R)
    for p, n in enumerate(lengths):
        clean = torch.rand(n, 2, generator=g) @ torch.rand(2, C, generator=g)
        V[p, :n] = ((clean + NOISE[p] * torch.rand(n, C, generator=g)) + 0.01).bfloat16().float()
    W0 = torch.randn(P, C, R, generator=g).abs()
    for p, n in enumerate(lengths):
        H0[p, :n] = torch.randn(n, R, generator=g).abs()
    Z0 = torch.rand(P, R, generator=g) + 0.2
    Wa = 1. + 0.5 * torch.rand(P, generator=g)
    return V, W0, H0, Z0, Wa


def main():
    torch.set_num_threads(1)                # deterministic reduction order
    flat = {}
    for name, (lengths, tol, max_iter, seed, wa, ha, za, tw, tz) in cases().items():
        V, W0, H0, Z0, Wa = inputs(lengths, seed)
        W, H, Z = torch.zeros(P, C, R), torch.zeros(P, N, R), torch.zeros(P, R)
        its, norms = [], []
        d = torch.float64
        torch.set_default_dtype(d)          # the reference's parameters and its whole fit in float64
        for p, n in enumerate(lengths):
            m = PLCA(W=W0[p].to(d), H=H0[p, :n].to(d), Z=Z0[p].to(d), trainable_W=tw, trainable_Z=tz)
            W_alpha = Wa[p].to(d) if wa == "tensor" else wa
            n_iter, norm = m.fit(V[p, :n].to(d), tol=tol, max_iter=max_iter, W_alpha=W_alpha, H_alpha=ha, Z_alpha=za)
            its.append(n_iter)
            norms.append(float(norm))
            W[p], H[p, :n], Z[p] = m.W.detach().float(), m.H.detach().float(), m.Z.detach().float()
        torch.set_default_dtype(torch.float32)
        rec = dict(V=V, W0=W0, H0=H0, Z0=Z0, W=W, H=H, Z=Z)
        if wa == "tensor":
            rec["W_alpha"] = Wa
        for k, v in rec.items():
            flat[f"{name}/{k}"] = v.numpy()
        flat[f"{name}/lengths"] = np.array(lengths, dtype=np.int64)
        flat[f"{name}/n_iter"] = np.array(its, dtype=np.int64)
        flat[f"{name}/norm"] = np.array(norms, dtype=np.float64)
        scal = dict(tol=tol, max_iter=max_iter, H_alpha=ha, Z_alpha=za, trainable_W=tw, trainable_Z=tz)
        if wa != "tensor":
            scal["W_alpha"] = wa
        for k, v in scal.items():
            flat[f"{name}/{k}"] = np.array(v, dtype=np.float64)
        print(name, "lengths", lengths, "n_iter", its)
    path = os.path.join(GOLD, "reference_batched_plca_ragged.npz")
    np.savez_compressed(path, **flat)
    print(f"wrote {path} ({os.path.getsize(path) / 1e3:.0f} KB)")


if __name__ == "__main__":
    main()
