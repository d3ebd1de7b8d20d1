"""Cases, data and float64 references of the sparse-target kernel tests (tests/test_gpu_sparse_terms.py), and what they must
cover (checked against the library's own launch plans on the CPU by tests/test_f32_plan_cover.py).

The sparse engine (csrc/sparse_nmf.cu) evaluates nmf.py:603-638 at the non-zeros of V only: one warp per row of the CSR form
(H update, loss) or of the CSC form (W update) gathers the other factor's rows; the beta-2 denominator is F (G^T G) with the
Gram matrix summed over per-block 32-row slabs.  Exact cases follow tests/f32_cases.py:
  * beta 2: integer factors in {0..fmax} and values in {0..fmax^2}: every numerator, Gram entry, denominator, dot and
    `v * dot` is an integer below 2^24 (`sparse_eu_bound`), so exact in any order; the loss pieces v_norm, pos and neg are
    sums of integers in double below 2^52, so the loss is exact too.
  * beta 1: factors in {2, 3} (distinct column sums) and V = Q (w . h) at the stored positions, Q in {0..3}: dot >= 4, so
    dot + eps rounds back to dot and v / (dot + eps) = q; the numerator is an integer sum, the denominator a column sum.
"""
import math

import torch

from f32_cases import EXACT, U, _gen, _ints, distinct_colsums, gam, nmf_bound, pick_range

EPS = 2.0 ** -23
EXACT_DOUBLE = 2 ** 52

# (N, C, R, pattern).  R covers RPL 1, 2, 4, 8 and Gram passes 1, 2, 3, 4, 5, 10, 16; N and C cover gather tails
# nseg % 8 in {0, 1, 7} and the Gram plans: one partial slab (<= 32 rows), 2 blocks with 1 row in the last (33), 128 blocks
# of 32 rows (4096), 64-row blocks with a 1-row last block (4097), and with a 63-row last block whose second slab is short
# (8191).
SPARSE_EXACT = [
    (1, 1, 1, "lines"),            # the one cell stored
    (7, 9, 31, "edges"),
    (8, 31, 32, "random"),
    (9, 32, 33, "random"),
    (31, 33, 64, "edges"),
    (32, 7, 65, "random"),
    (33, 8, 96, "empty"),          # nnz = 0
    (4096, 33, 128, "lines"),      # a stored column of 4096
    (33, 4096, 129, "lines"),      # a stored row of 4096
    (4097, 31, 200, "edges"),
    (9, 4097, 256, "lines"),
    (8191, 7, 256, "lines"),
    (1, 8191, 200, "random"),
    (8191, 4097, 65, "random"),
    (4097, 8191, 33, "edges"),
    (800, 800, 64, "random"),      # the reference's sparse test shape (tests/test_nmf_sparse.py)
    (800, 800, 200, "random"),
]
# random non-integer data, float64 bars
SPARSE_BAR = [(9, 32, 33, "random"), (7, 9, 31, "edges"), (4096, 33, 128, "lines"), (33, 4096, 129, "lines"),
              (4097, 31, 200, "edges"), (8191, 7, 256, "lines"), (800, 800, 64, "random"), (800, 800, 200, "random")]
# one update of each factor (l1, l2 > 0, gamma 2/3) from exact raw terms
SPARSE_RATIO = [(31, 33, 64, "edges"), (4097, 31, 200, "edges"), (800, 800, 200, "random")]

MAX_NNZ = 200_000                      # keeps the float64 references (nnz x R doubles) small


# ---- sparsity patterns ------------------------------------------------------------------------------------------------
def pattern(N, C, kind, g):
    """(rows, cols) of the stored entries, sorted by (row, col).  random: about 5 % (fewer on large shapes, MAX_NNZ);
    edges: the same with the first and last row and column empty; lines: the same plus one fully stored row and column;
    empty: none."""
    if kind == "empty":
        z = torch.zeros(0, dtype=torch.int64)
        return z, z
    p = min(0.05, MAX_NNZ / (N * C))
    mask = torch.rand(N, C, generator=g) < p
    if kind == "edges":
        mask[[0, -1], :] = False
        mask[:, [0, -1]] = False
    elif kind == "lines":
        mask[N // 2, :] = True
        mask[:, C // 2] = True
    idx = mask.nonzero()
    return idx[:, 0].contiguous(), idx[:, 1].contiguous()


def sparse_tensor(N, C, rows, cols, vals):
    """A coalesced COO tensor that keeps explicitly stored zeros."""
    return torch.sparse_coo_tensor(torch.stack([rows, cols]), vals, (N, C), check_invariants=True).coalesce()


# ---- exact data ---------------------------------------------------------------------------------------------------------
def sparse_eu_bound(N, C, R, fmax, vmax):
    """Largest full sum or product of the beta-2 terms (nmf_bound: numerators, Gram entries, denominators, dots) and of the
    loss's fp32 `v * dot`."""
    return max(nmf_bound(N, C, R, fmax, vmax), vmax * R * fmax * fmax)


def sparse_eu_loss_bound(N, C, R, fmax, vmax, nnz):
    """Largest double partial sum of the beta-2 loss: v_norm + pos (each Gram entry below C fmax^2 / N fmax^2) and neg."""
    return 0.5 * nnz * vmax ** 2 + 0.5 * R * R * (C * fmax ** 2) * (N * fmax ** 2) + nnz * vmax * R * fmax ** 2


def sparse_kl_bound(N, C, R):
    """beta 1, factors in {2, 3}, Q in {0..3}: v = q dot, numerators sum q w, column sums."""
    return max(3 * 9 * R, max(N, C) * 3 * 3)


def sparse_range(N, C, R):
    return pick_range(lambda f, v: sparse_eu_bound(N, C, R, f, v))


def sparse_eu_data(case, seed):
    """(rows, cols, vals, W, H): integer data, exact at beta 2."""
    N, C, R, kind = case
    g = _gen(seed)
    rows, cols = pattern(N, C, kind, g)
    fmax = sparse_range(N, C, R)
    return rows, cols, _ints((rows.numel(),), 0, fmax * fmax, g), _ints((C, R), 0, fmax, g), _ints((N, R), 0, fmax, g)


def sparse_kl_data(case, seed):
    """(rows, cols, vals, W, H, Q): vals = Q (w . h) exactly at the stored positions, factors in {2, 3}."""
    N, C, R, kind = case
    g = _gen(seed)
    rows, cols = pattern(N, C, kind, g)
    W, H = distinct_colsums(_ints((C, R), 2, 3, g)), distinct_colsums(_ints((N, R), 2, 3, g))
    Q = _ints((rows.numel(),), 0, 3, g)
    return rows, cols, (Q.double() * dots(rows, cols, W.double(), H.double())).float(), W, H, Q


def sparse_bar_data(case, seed):
    N, C, R, kind = case
    g = _gen(seed)
    rows, cols = pattern(N, C, kind, g)
    return (rows, cols, torch.rand(rows.numel(), generator=g) + 0.5, torch.rand(C, R, generator=g) + 0.5,
            torch.rand(N, R, generator=g) + 0.5)


# ---- float64 references: nmf.py:603-638 restated at the non-zeros --------------------------------------------------------
def dots(rows, cols, W, H):
    """w_c . h_n at every stored (n, c) (`_nmf_sparse_reconstruct`)."""
    return (W[cols] * H[rows]).sum(1)


def v_norm(vals, beta):
    """`_get_V_norm` nmf.py:161-170 as the engine computes it (0 log 0 = 0)."""
    v = vals.double()
    if beta == 2:
        return float((v * v).sum() * 0.5)
    pos = v[v > 0]
    return float((pos * pos.log()).sum() - v.sum())


def sp_terms64(which, beta, rows, cols, vals, W, H, ratio=None):
    """(numerator, denominator) of the update of W (which 0) or H (which 1): the gradients of `neg` and `pos` of
    `_nmf_sp_recon_beta_pos_neg`.  beta 2: neg = sum v (w . h), pos = 1/2 sum (H W^T W) o H; beta 1: neg = sum v log(w . h
    + eps), pos = colsum(W) . colsum(H).  `ratio`: the beta-1 v / (w . h + eps) per stored entry when it is known exactly
    (Q of the exact data, what fp32 computes)."""
    v = vals.to(W.dtype)
    if beta == 1:
        v = v / (dots(rows, cols, W, H) + EPS) if ratio is None else ratio.to(W.dtype)
    if which == 0:
        num = torch.zeros_like(W).index_add_(0, cols, v[:, None] * H[rows])
        return num, (H.sum(0) if beta == 1 else W @ (H.t() @ H))
    num = torch.zeros_like(H).index_add_(0, rows, v[:, None] * W[cols])
    return num, (W.sum(0) if beta == 1 else H @ (W.t() @ W))


def sp_loss_pieces64(beta, rows, cols, vals, W, H):
    """(v_norm, pos, neg): loss = v_norm + pos - neg (nmf.py:358, :398)."""
    d = dots(rows, cols, W, H)
    v = vals.to(W.dtype)
    if beta == 2:
        return v_norm(vals, 2), float(0.5 * ((W.t() @ W) * (H.t() @ H)).sum()), float(v @ d)
    return v_norm(vals, 1), float(W.sum(0) @ H.sum(0)), float(v @ (d + EPS).log())


def sp_loss64(beta, rows, cols, vals, W, H):
    vn, pos, neg = sp_loss_pieces64(beta, rows, cols, vals, W, H)
    return vn + pos - neg


# ---- a priori bars of the random-data cases ---------------------------------------------------------------------------------
def gam64(n):
    return n * 2.0 ** -53 / (1 - n * 2.0 ** -53)


def seg_lengths(which, rows, cols, N, C):
    """Stored entries per segment: per column of V (W update) or per row (H update)."""
    return torch.bincount(cols if which == 0 else rows, minlength=C if which == 0 else N)


def num_bar(beta, R, n):
    """Relative bar of each numerator entry (n: its segment's length, a tensor).  beta 1: f32_cases.terms_bar(1, R, n, 1)
    (dot to gamma_R, eps add u, division and product within 9u, the sum gamma_n); beta 2: gamma_n + u (the fmaf chain)."""
    g = n.double() * U / (1 - n.double() * U)
    if beta == 1:
        return 1.01 * ((gam(R) + U) + 9 * U + g + gam(1))
    return g + U


def den_bar(R, rpb, nb):
    """Relative bar of the beta-2 denominator F G: the Gram entries to gamma_rpb (slab fmaf chains and the slab sums of one
    block) + gamma_nb (the block sum), the R-term product gamma_R, plus u."""
    return gam(R) + gam(rpb) + gam(nb) + U


def loss_bar(beta, rows, cols, vals, W, H):
    """Absolute bar of the loss, in the style of f32_cases.loss_bar, from float64 factors.  pos: every colsum (beta 1) or
    Gram entry (beta 2) to gamma_rows, so each product to gamma_N + gamma_C.  neg: every dot to gamma_R; beta 2 the fp32
    v * dot adds u; beta 1 the eps add u, logf 1 ulp (2u of the result) and the fp32 product u.  The double sums add
    gamma64 of the number of terms of every piece."""
    N, C, R = H.shape[0], W.shape[0], W.shape[1]
    d = dots(rows, cols, W, H)
    v = vals.double()
    vn, pos, neg = sp_loss_pieces64(beta, rows, cols, vals, W, H)
    if beta == 2:
        neg_bar = float((v * d).sum()) * (gam(R) + U)
    else:
        neg_bar = float((v * (gam(R) + 2 * U + 3 * U * (d + EPS).log().abs())).sum())
    pos_bar = abs(pos) * (gam(N) + gam(C))
    nterms = rows.numel() + R * R + math.ceil(N / 8)
    return pos_bar + neg_bar + gam64(nterms) * (abs(vn) + abs(pos) + abs(neg))
