"""Divergences of the reference's `torchnmf.metrics` surface (metrics.py:6-96): plain differentiable torch expressions,
used by user code and by the generic (autograd) path of `trainer.BetaMu`.  `fit` never calls these: its loss comes from
the fused kernels (`nmfb200_loss`).
"""
import torch

from .constants import eps

__all__ = ["kl_div", "euclidean", "is_div", "beta_div", "sparseness"]


def kl_div(input, target):
    """Generalised Kullback-Leibler divergence = beta-divergence at beta = 1 (metrics.py:6-22)."""
    t = target.reshape(-1)
    log_ratio = torch.log(target + eps) - torch.log(input + eps)
    return t @ log_ratio.reshape(-1) - target.sum() + input.sum()


def euclidean(input, target):
    """Half the squared Euclidean distance = beta-divergence at beta = 2 (metrics.py:25-39)."""
    d = input - target
    return 0.5 * (d * d).sum()


def is_div(input, target):
    """Itakura-Saito divergence = beta-divergence at beta = 0 (metrics.py:42-57)."""
    te, xe = target + eps, input + eps
    return (te / xe).sum() - torch.log(te).sum() + torch.log(xe).sum() - target.numel()


def beta_div(input, target, beta=2):
    """beta-divergence between the reconstruction `input` and `target` (metrics.py:60-96)."""
    if beta == 2:
        return euclidean(input, target)
    if beta == 1:
        return kl_div(input, target)
    if beta == 0:
        return is_div(input, target)
    x = input.reshape(-1) + eps
    t = target.reshape(-1)
    if beta < 0:
        t = t + eps
    bm = beta - 1
    return (t.pow(beta).sum() + bm * x.pow(beta).sum() - beta * (t @ x.pow(bm))) / (beta * bm)


def sparseness(x):
    """Hoyer's sparseness measure (sqrt(N) - |x|_1 / |x|_2) / (sqrt(N) - 1) of a tensor of any shape (metrics.py:99-115)."""
    n = x.numel() ** 0.5
    return (n - x.norm(1) / x.norm(2)) / (n - 1)
