"""CPU oracle of the masked PLCA fit: `PLCA.fit(V, ..., mask=M)` (and SIPLCA / SIPLCA2 / SIPLCA3), written from its
definition, in whatever dtype it is given (the tests run it in float64).

With O the observed cells (M True), q = reconstruct(H, W, Z) the model (summing to 1), q_O = sum_O q and Vn = V / sum_O V on
O, the fit maximises the observed-data log-likelihood sum_O Vn log(q / q_O) (plus the reference's Dirichlet priors) by EM
with the missing cells latent.  Each iteration materialises the completed target

    Vt = q_O Vn  on O,        Vt = q  off O                     (sum Vt = sum q = 1)

and takes the reference's EM step (torchnmf/plca.py:247-289, oracle/plca_oracle.py's loop body) on it, Vt normalised by its
sum as the reference's `fit(Vt, max_iter=1)` normalises its target.  The loss is
sqrt(2 sum_O [v (log(v + eps) - log(x + eps)) - v + x]) with v = V and x = q sum_O V / q_O, before the first iteration and
after every 10th, with the reference's stop rule; the fit returns sum_O V / q_O at the final factors as its norm.

Pinned by tests/golden/reference_masked_plca.npz (tools/make_golden_masked_plca.py, from the unmodified reference);
tests/test_masked_plca.py checks it.
"""
import math

import torch

from oracle import plca_oracle as po


def observed_mass(q, M):
    return torch.where(M, q, torch.zeros((), dtype=q.dtype)).sum()


def completed_target(Vn, M, q):
    """Vt of one iteration and q_O: the expected complete data given the observations and the model q."""
    qo = observed_mass(q, M)
    return torch.where(M, qo * Vn, q), qo


def em_step(Vt, W, H, Z, W_alpha=1., H_alpha=1., Z_alpha=1., trainable_W=True, trainable_H=True, trainable_Z=True,
            eps=po.EPS):
    """One reference EM step (plca.py:247-289) on the target Vt (normalised by its sum first), with the ratio's `eps`."""
    Vn = Vt / Vt.sum()
    P = Vn / (po.reconstruct(H, W, Z) + eps)
    dW, dH, dZ = po.gradients(P, H, W, Z)
    Z_prior = None
    if trainable_Z:
        Z = Z * dZ.clamp_min(0)
        Z_prior = Z.clone()
        Z = po._prior(Z, Z_alpha, False)
        Z = Z / Z.sum()
    if trainable_W:
        W = W * dW.clamp_min(0)
        if Z_prior is None:
            div = po.get_norm(W)
            Z_prior = div.squeeze()
        else:
            div = po._over(Z_prior, W)
        W = po._prior(W / div, W_alpha, True)
    if trainable_H:
        H = H * dH.clamp_min(0)
        div = po.get_norm(H) if Z_prior is None else po._over(Z_prior, H)
        H = po._prior(H / div, H_alpha, True)
    return W, H, Z


def loss(V, M, q, eps=po.EPS):
    """sqrt(2 kl_div(x[O], V[O])), x = q sum_O V / q_O (metrics.py:22's eps)."""
    v = V[M]
    x = (q * (v.sum() / observed_mass(q, M)))[M]
    d = float((v * (torch.log(v + eps) - torch.log(x + eps)) - v + x).sum())
    return math.sqrt(2.0 * d) if d >= 0 else float("nan")


def log_likelihood(V, M, W, H, Z):
    """sum_O Vn log(q / q_O), the objective (without priors) that EM never decreases at eps = 0 and alpha = 1."""
    q = po.reconstruct(H, W, Z)
    v = V[M]
    return float((v / v.sum() * torch.log(q[M] / observed_mass(q, M))).sum())


def fit_masked(V, M, W, H, Z, tol=1e-4, max_iter=200, W_alpha=1., H_alpha=1., Z_alpha=1., trainable_W=True,
               trainable_H=True, trainable_Z=True, eps=po.EPS, history=None):
    """Returns (W, H, Z, n_iter, norm, losses).  W, H, Z are the (already normalised) module parameters.  V is read on O only
    (NaN elsewhere is fine).  `eps` is the EM ratio's (the loss keeps the reference's).  `history`, a list, receives
    (W, H, Z) after every iteration."""
    V = torch.where(M, V, torch.zeros((), dtype=V.dtype))
    Vn = V / V.sum()
    kw = dict(W_alpha=W_alpha, H_alpha=H_alpha, Z_alpha=Z_alpha, trainable_W=trainable_W, trainable_H=trainable_H,
              trainable_Z=trainable_Z, eps=eps)
    loss_init = previous = loss(V, M, po.reconstruct(H, W, Z))
    losses = [loss_init]
    n_iter = -1
    for n_iter in range(max_iter):
        Vt, _ = completed_target(Vn, M, po.reconstruct(H, W, Z))
        W, H, Z = em_step(Vt, W, H, Z, **kw)
        if history is not None:
            history.append((W, H, Z))
        if n_iter % 10 == 9:
            cur = loss(V, M, po.reconstruct(H, W, Z))
            losses.append(cur)
            if (previous - cur) / loss_init < tol:
                break
            previous = cur
    norm = V.sum() / observed_mass(po.reconstruct(H, W, Z), M)
    return W, H, Z, n_iter, norm, losses
