"""CPU oracle of a fit with per-cell weights (`fit(V, ..., weight=Wt)`), in float64.

TEST INFRASTRUCTURE ONLY, beside tests/masked_oracle.py, whose kinds it reuses unchanged.  The weighted fit minimises
sum over the cells with w > 0 of w * d_beta(v | x), x = WH, and every update is the reference's ratio (nmf.py:78-92) of the
two backward passes of that loss:

    num = contraction of  w * V * (WH + eps)^(beta - 2)      (beta 2: w * V)
    den = contraction of  w * (WH + eps)^(beta - 1)          (beta 2: w * WH; beta 1: w itself, not the column sums)

both relu'd and eps-shifted.  The cells of weight 0 are dropped as the missing cells of a mask are: V is replaced by zeros
there before any arithmetic, so a NaN there changes nothing.  With integer weights this is what the reference's own
`trainer.BetaMu` computes with a closure that gathers each cell w times; tests/golden/reference_weighted.npz
(tools/make_golden_weighted.py) pins it.
"""
import math

import torch

from oracle import mu_oracle as orc
from masked_oracle import KINDS

EPS = orc.EPS


def cell_div(x, t, beta):
    """metrics.beta_div's term of every cell (metrics.py:22, :39, :56-57, :84-96), elementwise."""
    if beta == 2:
        d = x - t
        return 0.5 * d * d
    if beta == 1:
        return t * ((t + EPS).log() - (x + EPS).log()) - t + x
    if beta == 0:
        te, xe = t + EPS, x + EPS
        return te / xe - te.log() + xe.log() - 1
    x = x + EPS
    if beta < 0:
        t = t + EPS
    bm = beta - 1
    return (t.pow(beta) + bm * x.pow(beta) - beta * t * x.pow(bm)) / (beta * bm)


def weighted_loss(WH, V, Wt, beta):
    """sum over the cells with w > 0 of w * d_beta(v | x)."""
    on = Wt > 0
    return (Wt[on] * cell_div(WH[on], V[on], beta)).sum()


def weighted_phi(V, WH, Wt, beta):
    """(w Pn, w Pp) of nmf.py:61-74, zero where w == 0; w itself at beta 1."""
    on = Wt > 0
    zero = torch.zeros((), dtype=WH.dtype)
    Pn, Pp = orc.phi(torch.where(on, V, zero), WH, beta)
    if Pp is None:
        Pp = torch.ones_like(WH)
    return torch.where(on, Pn * Wt, zero), torch.where(on, Pp * Wt, zero)


def weighted_terms(V, W, H, Wt, beta, which, kind="nmf"):
    """Raw (numerator, denominator) of the update of W (which = 0) or H (which = 1), each in the factor's shape."""
    recon, grad_w, grad_h = KINDS[kind]
    Pn, Pp = weighted_phi(V, recon(H, W), Wt, beta)
    if which == 0:
        return grad_w(Pn, H, W), grad_w(Pp, H, W)
    return grad_h(Pn, W, H), grad_h(Pp, W, H)


def weighted_update(V, W, H, Wt, beta, which, kind="nmf", gamma=None, l1_reg=0.0, l2_reg=0.0):
    gamma = orc.gamma_of(beta) if gamma is None else gamma
    num, den = weighted_terms(V, W, H, Wt, beta, which, kind)
    return orc._ratio_update(W if which == 0 else H, num, den, gamma, l1_reg, l2_reg, False)


def fit(V, W, H, Wt, beta=1, tol=1e-4, max_iter=200, alpha=0, l1_ratio=0, trainable_W=True, trainable_H=True,
        kind="nmf"):
    """oracle/mu_oracle.py's fit on the weighted loss, in float64.  Returns (W, H, n_iter, losses) in float64."""
    V, W, H, Wt = V.double(), W.double(), H.double(), Wt.double()
    Vo = V[Wt > 0]
    assert Vo.numel() > 0, "every weight is zero"
    assert bool(torch.all(Vo >= 0)), "Target should be non-negative."
    if float(Vo.min()) == 0 and beta <= 0:
        raise ValueError("When beta <= 0 and V contains zeros, the training process may diverge. "
                         "Please add small values to V, or use a positive beta value.")
    recon = KINDS[kind][0]
    gamma = orc.gamma_of(beta)
    l1_reg, l2_reg = alpha * l1_ratio, alpha * (1 - l1_ratio)

    def loss():
        return math.sqrt(2.0 * float(weighted_loss(recon(H, W), V, Wt, beta)))

    loss_init = previous = loss()
    losses = [loss_init]
    n_iter = -1
    for n_iter in range(max_iter):
        if trainable_W:
            W = weighted_update(V, W, H, Wt, beta, 0, kind, gamma, l1_reg, l2_reg)
        if trainable_H:
            H = weighted_update(V, W, H, Wt, beta, 1, kind, gamma, l1_reg, l2_reg)
        if n_iter % 10 == 9:
            cur = loss()
            losses.append(cur)
            if (previous - cur) / loss_init < tol:
                break
            previous = cur
    return W, H, n_iter + 1, losses
