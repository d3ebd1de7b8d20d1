"""Planted-rank problems of the ARD tests (tests/test_ard.py, tests/test_gpu_ard.py): targets built from a few clearly
separated components plus a little noise, fitted from a generous rank, for which the float64 ARD oracle keeps exactly the
planted number of components above the bound after PLANTED_ITERS iterations at beta 1 with ARD(a=5)."""
import torch

from oracle import mu_oracle as orc

PLANTED_ITERS = 200


def planted_nmf(seed=0, N=80, C=64, rank=4, R=12, noise=0.05, scale=10.0):
    """V (N, C) fp32 = H* W*^T + noise, W* with disjoint channel blocks per component; (V, W0, H0), all fp32."""
    g = torch.Generator().manual_seed(seed)
    Hs = torch.rand(N, rank, generator=g, dtype=torch.float64) * scale
    Ws = torch.zeros(C, rank, dtype=torch.float64)
    for k in range(rank):
        Ws[k * C // rank:(k + 1) * C // rank, k] = torch.rand(C // rank, generator=g, dtype=torch.float64) + 0.5
    V = Hs @ Ws.t() + noise * torch.rand(N, C, generator=g, dtype=torch.float64)
    return V.float(), torch.rand(C, R, generator=g) + 0.1, torch.rand(N, R, generator=g) + 0.1


def planted_nmfd(seed=0, B=2, C=16, T=4, Lin=60, R=6, scale=10.0):
    """V (B, C, Lin + T - 1) fp32 from 2 planted kernels on disjoint channel halves with sparse activations; (V, W0, H0)."""
    g = torch.Generator().manual_seed(seed)
    Ws = torch.zeros(C, 2, T, dtype=torch.float64)
    Ws[:C // 2, 0] = torch.rand(C // 2, T, generator=g, dtype=torch.float64) + 0.5
    Ws[C // 2:, 1] = torch.rand(C // 2, T, generator=g, dtype=torch.float64) + 0.5
    Hs = torch.rand(B, 2, Lin, generator=g, dtype=torch.float64) * scale * (torch.rand(B, 2, Lin, generator=g) < 0.3)
    V = orc.nmfd_reconstruct(Hs, Ws) + 0.05 * torch.rand(B, C, Lin + T - 1, generator=g, dtype=torch.float64)
    return V.float(), torch.rand(C, R, T, generator=g) + 0.1, torch.rand(B, R, Lin, generator=g) + 0.1


def relevant(lam, bound, margin=1e-2):
    """The components whose relevance is clearly above the bound, as a sorted list of indices."""
    return [k for k, v in enumerate(lam.tolist()) if v > bound * (1 + margin)]
