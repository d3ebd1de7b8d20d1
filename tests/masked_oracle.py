"""CPU oracle of a fit on the observed cells of the target only (`fit(V, ..., mask=M)`).

TEST INFRASTRUCTURE ONLY, beside oracle/mu_oracle.py, whose closed-form pieces it reuses unchanged.  The masked fit
minimises beta_div(WH[M], V[M]) -- the missing cells dropped, not zeroed -- and every update is the reference's ratio
(nmf.py:78-92) of the two backward passes of that loss, which is what the reference's own `trainer.BetaMu` computes with the
closure `(V[M], model()[M])`:

    num = contraction of  M * V * (WH + eps)^(beta - 2)      (beta 2: M * V)
    den = contraction of  M * (WH + eps)^(beta - 1)          (beta 2: M * WH; beta 1: M itself, not the column sums)

both relu'd and eps-shifted.  The missing cells of V are replaced by zeros before any arithmetic, so a NaN there changes
nothing.  tests/golden/reference_masked.npz (tools/make_golden_masked.py, from the unmodified reference's BetaMu) pins it.
"""
import math

import torch

from oracle import mu_oracle as orc

# kind -> (reconstruct(H, W), d<WH,G>/dW (G, H, W), d<WH,G>/dH (G, W, H))
KINDS = {
    "nmf": (orc.nmf_reconstruct, lambda G, H, W: G.t() @ H, lambda G, W, H: G @ W),
    "nmfd": (orc.nmfd_reconstruct, lambda G, H, W: orc.nmfd_grad_w(G, H, W.shape[2]),
             lambda G, W, H: orc.nmfd_grad_h(G, W, H.shape[2])),
    "nmf2d": (orc.nmfnd_reconstruct, lambda G, H, W: orc.nmfnd_grad_w(G, H, tuple(W.shape[2:])),
              lambda G, W, H: orc.nmfnd_grad_h(G, W, tuple(H.shape[2:]))),
}
KINDS["nmf3d"] = KINDS["nmf2d"]


def masked_loss(WH, V, M, beta):
    """metrics.beta_div over the observed cells only."""
    return orc.beta_div(WH[M], V[M], beta)


def masked_phi(V, WH, M, beta):
    """(Pn, Pp) of nmf.py:61-74 on the observed cells, zero at the missing ones; Pp = M at beta 1."""
    zero = torch.zeros((), dtype=WH.dtype)
    Pn, Pp = orc.phi(torch.where(M, V, zero), WH, beta)
    if Pp is None:
        Pp = torch.ones_like(WH)
    return torch.where(M, Pn, zero), torch.where(M, Pp, zero)


def masked_terms(V, W, H, M, beta, which, kind="nmf"):
    """Raw (numerator, denominator) of the update of W (which = 0) or H (which = 1), each in the factor's shape."""
    recon, grad_w, grad_h = KINDS[kind]
    Pn, Pp = masked_phi(V, recon(H, W), M, beta)
    if which == 0:
        return grad_w(Pn, H, W), grad_w(Pp, H, W)
    return grad_h(Pn, W, H), grad_h(Pp, W, H)


def masked_update(V, W, H, M, beta, which, kind="nmf", gamma=None, l1_reg=0.0, l2_reg=0.0):
    gamma = orc.gamma_of(beta) if gamma is None else gamma
    num, den = masked_terms(V, W, H, M, beta, which, kind)
    return orc._ratio_update(W if which == 0 else H, num, den, gamma, l1_reg, l2_reg, False)


def fit(V, W, H, M, beta=1, tol=1e-4, max_iter=200, alpha=0, l1_ratio=0, trainable_W=True, trainable_H=True,
        kind="nmf"):
    """oracle/mu_oracle.py's fit on the observed cells.  Returns (W, H, n_iter, losses)."""
    Vo = V[M]
    assert Vo.numel() > 0, "no observed cell"
    assert bool(torch.all(Vo >= 0)), "Target should be non-negative."
    if float(Vo.min()) == 0 and beta <= 0:
        raise ValueError("When beta <= 0 and V contains zeros, the training process may diverge. "
                         "Please add small values to V, or use a positive beta value.")
    recon = KINDS[kind][0]
    gamma = orc.gamma_of(beta)
    l1_reg, l2_reg = alpha * l1_ratio, alpha * (1 - l1_ratio)
    W, H = W.clone(), H.clone()

    def loss():
        return math.sqrt(2.0 * float(masked_loss(recon(H, W), V, M, beta)))

    loss_init = previous = loss()
    losses = [loss_init]
    n_iter = -1
    for n_iter in range(max_iter):
        if trainable_W:
            W = masked_update(V, W, H, M, beta, 0, kind, gamma, l1_reg, l2_reg)
        if trainable_H:
            H = masked_update(V, W, H, M, beta, 1, kind, gamma, l1_reg, l2_reg)
        if n_iter % 10 == 9:
            cur = loss()
            losses.append(cur)
            if (previous - cur) / loss_init < tol:
                break
            previous = cur
    return W, H, n_iter + 1, losses
