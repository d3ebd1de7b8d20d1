"""Cases, float64 references and a priori bars of a sparse target's kernels at beta != 1, 2 (tests/test_gpu_sparse_beta.py;
checked on the CPU by tests/test_sparse_beta.py).

At such a beta (x = w_c . h_n + eps, nmf.py:621-636) the engine of nmfb200_nmf_set_target_sparse_any_beta forms
  * numerators at the stored entries only (csrc/sparse_nmf.cu, kSpBeta): num_H[n,:] = sum_{c in row n} v x^(beta-2) W[c,:],
    num_W[c,:] = sum_{n in col c} v x^(beta-2) H[n,:];
  * denominators over every cell without V (csrc/simt_nmf.cu, kVFree): den_H = (HW^T + eps)^(beta-1) W,
    den_W = ((HW^T + eps)^(beta-1))^T H -- the dense fp32 kernels' own denominators, bit for bit;
  * loss = V_norm + pos - neg, V_norm = sum_nnz v^beta / (beta (beta-1)), pos = sum_all x^beta / beta,
    neg = sum_nnz v x^(beta-1) / (beta-1): beta_div(HW^T, V, beta) summed over every cell.
The data helpers, patterns and dots are tests/sparse_cases.py's.
"""
import math

import torch

from f32_cases import U, gam
from sparse_cases import EPS, dots, gam64, seg_lengths, sparse_bar_data, sparse_tensor  # noqa: F401

BETAS = [0.5, 1.5, 3]

# (N, C, R, pattern): gather RPL 1, 2, 4, 8 and contraction RB 1, 2, 4, 8, 16 (R <= 16, 32, 64, 128, 256), both chunk plans of
# the V-free denominator (nch 1 and nch > 1 on each side), and the empty, edges and lines patterns
SPARSE_BETA = [
    (7, 9, 16, "edges"),           # RPL 1, RB 1, one chunk on both sides
    (33, 8, 31, "empty"),          # nnz = 0: numerators 0, denominators still every cell's
    (4096, 33, 64, "lines"),       # RPL 2, RB 4: a stored column of 4096; W side 32 chunks
    (33, 4096, 100, "lines"),      # RPL 4, RB 8: a stored row of 4096; H side 32 chunks
    (1050, 4000, 20, "random"),    # RPL 1, RB 2: 9 chunks of 2 tiles (H), the W side likewise
    (800, 800, 200, "random"),     # RPL 8, RB 16: the reference's sparse test shape
    (4097, 31, 256, "edges"),      # RPL 8, RB 16 at rank 256
]
# one update of each factor (l1, l2 > 0, gamma != 1) from the raw terms
SPARSE_BETA_RATIO = [(7, 9, 16, "edges"), (1050, 4000, 20, "random"), (800, 800, 200, "random")]


# ---- float64 restatement --------------------------------------------------------------------------------------------------
def recon_pow(W, H, p):
    """(H W^T + eps)^p over every cell."""
    return (H @ W.t() + EPS).pow(p)


def terms64(which, beta, rows, cols, vals, W, H):
    """(numerator, denominator) of the update of W (which 0) or H (which 1): the gradients of neg and pos of
    `_nmf_sp_recon_beta_pos_neg` (nmf.py:621-636)."""
    ratio = vals.to(W.dtype) * (dots(rows, cols, W, H) + EPS).pow(beta - 2)
    P = recon_pow(W, H, beta - 1)
    if which == 0:
        return torch.zeros_like(W).index_add_(0, cols, ratio[:, None] * H[rows]), P.t() @ H
    return torch.zeros_like(H).index_add_(0, rows, ratio[:, None] * W[cols]), P @ W


def v_norm(vals, beta):
    """`_get_V_norm` nmf.py:161-170 at beta != 1, 2."""
    return float(vals.double().pow(beta).sum() / beta / (beta - 1))


def loss_pieces64(beta, rows, cols, vals, W, H):
    """(v_norm, pos, neg): loss = v_norm + pos - neg (nmf.py:358)."""
    d = dots(rows, cols, W, H)
    v = vals.to(W.dtype)
    pos = float(recon_pow(W, H, beta).sum() / beta)
    neg = float(v @ (d + EPS).pow(beta - 1) / (beta - 1))
    return v_norm(vals, beta), pos, neg


def loss64(beta, rows, cols, vals, W, H):
    vn, pos, neg = loss_pieces64(beta, rows, cols, vals, W, H)
    return vn + pos - neg


# ---- a priori bars ----------------------------------------------------------------------------------------------------------
# powf: 4 ulp (CUDA Math API, single-precision table, "powf(x,y)"), i.e. 8u of its result
POWF = 8 * U


def num_bar(beta, R, n):
    """Relative bar of each numerator entry (n: its segment's length, a tensor).  Each term v x^(beta-2) w: the dot to gamma_R
    (non-negative terms, any order), the eps add u, so x to gamma_R + u, which the power amplifies by |beta - 2|; powf's
    8u; the product with v u (the fmaf with w is exact before its sum); the sum of the n terms gamma_n.  x 1.01 for the
    second-order products."""
    return 1.01 * (abs(beta - 2) * (gam(R) + U) + POWF + U + gam(n.double()))


def loss_bar(beta, rows, cols, vals, W, H):
    """Absolute bar of the loss from float64 factors.  pos: every cell's S to gamma_R + u (the eps add) through the power
    beta, powf's 8u, one thread's fp32 sum of 16 cells gamma_16.  neg: x to gamma_R + u through the power |beta - 1|, powf's
    8u, the product with v u.  V_norm: powf(v, beta)'s 8u.  The double sums add gamma64 of the number of terms of every
    piece."""
    N, C, R = H.shape[0], W.shape[0], W.shape[1]
    vn, pos, neg = loss_pieces64(beta, rows, cols, vals, W, H)
    pos_bar = abs(pos) * (beta * (gam(R) + U) + POWF + gam(16))
    neg_bar = abs(neg) * (abs(beta - 1) * (gam(R) + U) + POWF + U)
    vn_bar = abs(vn) * POWF
    nterms = rows.numel() + N * C + math.ceil(N / 8)
    return 1.01 * (pos_bar + neg_bar + vn_bar) + gam64(nterms) * (abs(vn) + abs(pos) + abs(neg))


# ---- fp32 emulation on the CPU --------------------------------------------------------------------------------------------------
def num32(which, beta, rows, cols, vals, W, H):
    """The numerator in fp32 arithmetic (dots, eps add, power, product, sums; in torch's order)."""
    ratio = vals * (dots(rows, cols, W, H) + torch.tensor(EPS, dtype=torch.float32)).pow(beta - 2)
    if which == 0:
        return torch.zeros_like(W).index_add_(0, cols, ratio[:, None] * H[rows])
    return torch.zeros_like(H).index_add_(0, rows, ratio[:, None] * W[cols])


def loss32(beta, rows, cols, vals, W, H):
    """The loss with fp32 terms and double sums: pos from fp32 S, neg and V_norm from fp32 powers."""
    eps = torch.tensor(EPS, dtype=torch.float32)
    pos = float((H @ W.t() + eps).pow(beta).double().sum()) / beta
    terms = vals.pow(beta).double() / (beta * (beta - 1)) - (vals * (dots(rows, cols, W, H) + eps).pow(beta - 1)).double() / (beta - 1)
    return float(terms.sum()) + pos


def den_bar(beta, R, nc, nch):
    """Relative bar of each V-free denominator entry (nc contracted cells, nch chunks): S to gamma_R + u through the power
    |beta - 1|, powf's 8u, the fmaf chain over a chunk gamma_nc and the chunk sum gamma_nch."""
    return 1.01 * (abs(beta - 1) * (gam(R) + U) + POWF + gam(nc) + gam(nch))
