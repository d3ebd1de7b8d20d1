"""CPU oracle for the dense multiplicative-update (MU) NMF / NMFD hot path.

TEST INFRASTRUCTURE ONLY.  Nothing in the product package imports this file; only
``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` /
``--impl reference`` legs may.  It is the checker, never the thing shipped.

What it is: a closed-form fp32 restatement (plain torch CPU ops, NO autograd, NO
F.linear/F.conv1d) of the reference's autograd-derived update, written from the maths of

    torchnmf/nmf.py:52-92    _double_backward_update   (phi stage, two backward passes, ratio)
    torchnmf/nmf.py:122-131  _get_W_kl_positive / _get_H_kl_positive  (beta == 1 denominators)
    torchnmf/nmf.py:298-409  BaseComponent.fit          (gamma, l1/l2, loop order, stop rule)
    torchnmf/nmf.py:691-693  NMF.reconstruct            (WH = H @ W^T)
    torchnmf/nmf.py:776-779  NMFD.reconstruct           (WH[b,c,l] = sum_{r,t} W[c,r,t] H[b,r,l-t])
    torchnmf/metrics.py:6-96 kl_div / euclidean / is_div / beta_div
    torchnmf/constants.py:3  eps = float32 machine epsilon

Parity status: PINNED.  ``oracle/make_golden.py`` runs the real reference (imported from
oracle/_ref) from identical initial factors and stores its outputs
under ``tests/golden/``; ``tests/test_oracle.py`` checks this restatement against those vectors
(bit-exact for alpha == 0 on the build container's torch, <= 2e-6 relative otherwise).

Layout (reference layout, nmf.py:659-662): V (N, C), W (C, R), H (N, R), V ~= H @ W^T.
NMFD (nmf.py:743-750): V (B, C, L), W (C, R, T), H (B, R, L - T + 1).
"""
import math

import torch

# torchnmf/constants.py:3
EPS = float(torch.finfo(torch.float32).eps)


# --------------------------------------------------------------------------------------
# loss (torchnmf/metrics.py)
# --------------------------------------------------------------------------------------
def beta_div(WH, V, beta):
    """metrics.py:60-96 (dispatch) with kl_div :22, euclidean :39, is_div :56-57."""
    x = WH.reshape(-1)
    t = V.reshape(-1)
    if beta == 2:
        d = x - t
        return (d * d).sum() * 0.5
    if beta == 1:
        return t @ ((t + EPS).log() - (x + EPS).log()) - t.sum() + x.sum()
    if beta == 0:
        te, xe = t + EPS, x + EPS
        return (te / xe).sum() - te.log().sum() + xe.log().sum() - t.numel()
    x = x + EPS
    if beta < 0:
        t = t + EPS
    bm = beta - 1
    return (t.pow(beta).sum() + bm * x.pow(beta).sum() - beta * (t @ x.pow(bm))) / (beta * bm)


def fit_loss(WH, V, beta):
    """nmf.py:362 / :402 -- the quantity the stop rule looks at: sqrt(2 * beta_div)."""
    return math.sqrt(2.0 * float(beta_div(WH, V, beta)))


def gamma_of(beta):
    """nmf.py:341-346."""
    if beta < 1:
        return 1.0 / (2.0 - beta)
    if beta > 2:
        return 1.0 / (beta - 1.0)
    return 1.0


def phi(V, WH, beta):
    """nmf.py:61-74: (output_neg, output_pos); output_pos is None for beta == 1."""
    if beta == 2:
        return V, WH
    if beta == 1:
        return V / (WH + EPS), None
    if beta == 0:
        r = 1.0 / (WH + EPS)
        return r * r * V, r
    x = WH + EPS
    return x.pow(beta - 2) * V, x.pow(beta - 1)


def _ratio_update(param, neg, pos, gamma, l1_reg, l2_reg, pos_precomputed):
    """nmf.py:78-92.  `neg`/`pos` are the raw contractions (the autograd gradients)."""
    neg = neg.clamp_min(0) + EPS                      # :78  relu_().add_(eps)
    if not pos_precomputed:
        pos = pos.clamp_min(0) + EPS                  # :83
    if l1_reg > 0:
        pos = pos + l1_reg                            # :85-86
    if l2_reg > 0:
        pos = pos + l2_reg * param                    # :87-88 (pre-update factor)
    mult = neg / pos
    if gamma != 1:
        mult = mult.pow(gamma)                        # :90-91
    return param * mult                               # :92


# --------------------------------------------------------------------------------------
# NMF  (V (N,C) ~= H (N,R) @ W (C,R)^T)
# --------------------------------------------------------------------------------------
def nmf_reconstruct(H, W):
    """nmf.py:691-693."""
    return H @ W.t()


def nmf_w_contractions(V, W, H, beta):
    """Raw numerator / denominator of the W update before relu/eps/l1/l2 (linear in the rows of
    V and H, so row shards can be summed).  Returns (num (C,R), den (C,R) or colsum(H) (1,R))."""
    Pn, Pp = phi(V, nmf_reconstruct(H, W), beta)
    num = Pn.t() @ H
    den = H.sum(0, keepdim=True) if beta == 1 else Pp.t() @ H    # nmf.py:122-125
    return num, den


def nmf_update_w(V, W, H, beta, gamma=None, l1_reg=0.0, l2_reg=0.0):
    """nmf.py:367-378 for the dense NMF module; returns the new W."""
    gamma = gamma_of(beta) if gamma is None else gamma
    num, den = nmf_w_contractions(V, W, H, beta)
    return _ratio_update(W, num, den, gamma, l1_reg, l2_reg, beta == 1)


def nmf_update_h(V, W, H, beta, gamma=None, l1_reg=0.0, l2_reg=0.0):
    """nmf.py:380-391; returns the new H (W is the already-updated W)."""
    gamma = gamma_of(beta) if gamma is None else gamma
    Pn, Pp = phi(V, nmf_reconstruct(H, W), beta)
    num = Pn @ W
    den = W.sum(0, keepdim=True) if beta == 1 else Pp @ W        # nmf.py:128-131
    return _ratio_update(H, num, den, gamma, l1_reg, l2_reg, beta == 1)


# --------------------------------------------------------------------------------------
# NMFD  (V (B,C,L), W (C,R,T), H (B,R,Lin), L = Lin + T - 1)
# --------------------------------------------------------------------------------------
def nmfd_reconstruct(H, W):
    """nmf.py:776-779 restated as T shifted matrix products (docstring nmf.py:712-713)."""
    B, R, Lin = H.shape
    C, _, T = W.shape
    out = torch.zeros(B, C, Lin + T - 1, dtype=H.dtype)
    for t in range(T):
        out[:, :, t:t + Lin] += torch.matmul(W[:, :, t], H)      # (C,R) @ (B,R,Lin)
    return out


def nmfd_grad_w(G, H, T):
    """d<WH,G>/dW:  gW[c,r,t] = sum_{b,l} G[b,c,l] H[b,r,l-t]."""
    B, R, Lin = H.shape
    C = G.shape[1]
    gW = torch.zeros(C, R, T, dtype=H.dtype)
    for t in range(T):
        gW[:, :, t] = torch.matmul(G[:, :, t:t + Lin], H.transpose(1, 2)).sum(0)
    return gW


def nmfd_grad_h(G, W, Lin):
    """d<WH,G>/dH:  gH[b,r,j] = sum_{c,t} W[c,r,t] G[b,c,j+t]."""
    C, R, T = W.shape
    gH = torch.zeros(G.shape[0], R, Lin, dtype=W.dtype)
    for t in range(T):
        gH += torch.matmul(W[:, :, t].t(), G[:, :, t:t + Lin])
    return gH


def nmfd_update_w(V, W, H, beta, gamma=None, l1_reg=0.0, l2_reg=0.0):
    gamma = gamma_of(beta) if gamma is None else gamma
    T = W.shape[2]
    Pn, Pp = phi(V, nmfd_reconstruct(H, W), beta)
    num = nmfd_grad_w(Pn, H, T)
    den = H.sum((0, 2), keepdim=True) if beta == 1 else nmfd_grad_w(Pp, H, T)   # nmf.py:122-125 -> (1,R,1)
    return _ratio_update(W, num, den, gamma, l1_reg, l2_reg, beta == 1)


def nmfd_update_h(V, W, H, beta, gamma=None, l1_reg=0.0, l2_reg=0.0):
    gamma = gamma_of(beta) if gamma is None else gamma
    Lin = H.shape[2]
    Pn, Pp = phi(V, nmfd_reconstruct(H, W), beta)
    num = nmfd_grad_h(Pn, W, Lin)
    den = W.sum((0, 2), keepdim=True).squeeze(0) if beta == 1 else nmfd_grad_h(Pp, W, Lin)  # (R,1)
    return _ratio_update(H, num, den, gamma, l1_reg, l2_reg, beta == 1)


# --------------------------------------------------------------------------------------
# NMF2D / NMF3D  (V (B,C,*X), W (C,R,*K), H (B,R,*J), X = J + K - 1 per axis; nmf.py:782-942)
# The same three contractions as NMFD with a multi-index shift: one term per kernel offset.
# --------------------------------------------------------------------------------------
def _offsets(K):
    import itertools
    return itertools.product(*(range(k) for k in K))


def _window(t, J):
    return (slice(None), slice(None)) + tuple(slice(ti, ti + j) for ti, j in zip(t, J))


def nmfnd_reconstruct(H, W):
    """nmf.py:861-865 (conv2d) / :938-942 (conv3d), flipped kernel + full padding, restated as shifted products:
    WH[b,c,j+t] += sum_r W[c,r,t] H[b,r,j]."""
    J, K = H.shape[2:], W.shape[2:]
    out = torch.zeros(H.shape[0], W.shape[0], *(j + k - 1 for j, k in zip(J, K)), dtype=H.dtype)
    for t in _offsets(K):
        out[_window(t, J)] += torch.einsum("cr,br...->bc...", W[(slice(None), slice(None)) + t], H)
    return out


def nmfnd_grad_w(G, H, K):
    """gW[c,r,t] = sum_{b,j} G[b,c,j+t] H[b,r,j]."""
    J = H.shape[2:]
    gW = torch.zeros(G.shape[1], H.shape[1], *K, dtype=H.dtype)
    for t in _offsets(K):
        gW[(slice(None), slice(None)) + t] = torch.einsum("bc...,br...->cr", G[_window(t, J)], H)
    return gW


def nmfnd_grad_h(G, W, J):
    """gH[b,r,j] = sum_{c,t} W[c,r,t] G[b,c,j+t]."""
    K = W.shape[2:]
    gH = torch.zeros(G.shape[0], W.shape[1], *J, dtype=W.dtype)
    for t in _offsets(K):
        gH += torch.einsum("cr,bc...->br...", W[(slice(None), slice(None)) + t], G[_window(t, J)])
    return gH


def _sum_but_rank(x):
    dims = [d for d in range(x.dim()) if d != 1]
    return x.sum(dims, keepdim=True)                               # nmf.py:122-131


def nmfnd_update_w(V, W, H, beta, gamma=None, l1_reg=0.0, l2_reg=0.0):
    gamma = gamma_of(beta) if gamma is None else gamma
    K = tuple(W.shape[2:])
    Pn, Pp = phi(V, nmfnd_reconstruct(H, W), beta)
    num = nmfnd_grad_w(Pn, H, K)
    den = _sum_but_rank(H) if beta == 1 else nmfnd_grad_w(Pp, H, K)             # (1,R,1,..) broadcasts over W
    return _ratio_update(W, num, den, gamma, l1_reg, l2_reg, beta == 1)


def nmfnd_update_h(V, W, H, beta, gamma=None, l1_reg=0.0, l2_reg=0.0):
    gamma = gamma_of(beta) if gamma is None else gamma
    J = tuple(H.shape[2:])
    Pn, Pp = phi(V, nmfnd_reconstruct(H, W), beta)
    num = nmfnd_grad_h(Pn, W, J)
    den = _sum_but_rank(W).squeeze(0) if beta == 1 else nmfnd_grad_h(Pp, W, J)  # (R,1,..) broadcasts over H
    return _ratio_update(H, num, den, gamma, l1_reg, l2_reg, beta == 1)


# --------------------------------------------------------------------------------------
# fit loop (nmf.py:298-409)
# --------------------------------------------------------------------------------------
def fit(V, W, H, beta=1, tol=1e-4, max_iter=200, alpha=0, l1_ratio=0,
        trainable_W=True, trainable_H=True, kind="nmf"):
    """Restatement of BaseComponent.fit for dense V.  Returns (W, H, n_iter, losses) with
    `losses` = [loss_init, loss@9, loss@19, ...] exactly as the reference evaluates them."""
    assert bool(torch.all(V >= 0)), "Target should be non-negative."           # :329-330
    if float(V.min()) == 0 and beta <= 0:                                       # :332-336
        raise ValueError("When beta <= 0 and V contains zeros, the training process may diverge. "
                         "Please add small values to V, or use a positive beta value.")
    recon, upd_w, upd_h = {
        "nmf": (nmf_reconstruct, nmf_update_w, nmf_update_h),
        "nmfd": (nmfd_reconstruct, nmfd_update_w, nmfd_update_h),
        "nmf2d": (nmfnd_reconstruct, nmfnd_update_w, nmfnd_update_h),
        "nmf3d": (nmfnd_reconstruct, nmfnd_update_w, nmfnd_update_h),
    }[kind]
    gamma = gamma_of(beta)
    l1_reg = alpha * l1_ratio                                                   # :348
    l2_reg = alpha * (1 - l1_ratio)                                             # :349
    W, H = W.clone(), H.clone()
    loss_init = fit_loss(recon(H, W), V, beta)                                  # :360-362
    previous = loss_init
    losses = [loss_init]
    n_iter = -1
    for n_iter in range(max_iter):                                              # :366
        if trainable_W:
            W = upd_w(V, W, H, beta, gamma, l1_reg, l2_reg)                     # :367-378
        if trainable_H:
            H = upd_h(V, W, H, beta, gamma, l1_reg, l2_reg)                     # :380-391 (new W)
        if n_iter % 10 == 9:                                                    # :393
            loss = fit_loss(recon(H, W), V, beta)
            losses.append(loss)
            if (previous - loss) / loss_init < tol:                             # :405
                break
            previous = loss
    return W, H, n_iter + 1, losses                                             # :409
