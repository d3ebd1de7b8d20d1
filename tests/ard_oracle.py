"""CPU oracle of an l1-ARD fit (`fit(V, ..., ard=ARD(...))`), in float64.

TEST INFRASTRUCTURE ONLY, built on oracle/mu_oracle.py's contractions and tests/masked_oracle.py's kinds.  Automatic
relevance determination with the l1 prior (Tan and Fevotte, TPAMI 2013) minimises

    J(W, H, lambda) = D(V | model) / phi + sum_k [(sum W[:, k] + sum H[:, k] + b) / lambda_k + c log lambda_k],
    c = n_W + n_H + a + 1,

D the divergence the plain fit minimises (every cell, the observed cells of a mask, or sum w d_beta for a weight).  Each
iteration: the MU update of W with l1_reg = phi / lambda_k on component k, the same for H with the new W, then lambda_k =
(sum W[:, k] + sum H[:, k] + b) / c.  The stop rule looks, every 10th iteration, at max_k |lambda_k - previous| / previous.
"""
import math

import torch

from oracle import mu_oracle as orc
from masked_oracle import KINDS
from weighted_oracle import cell_div

EPS = orc.EPS


def _rank_shape(x):
    """A view shape that broadcasts one value per component over x (components on axis 1)."""
    return (1, -1) + (1,) * (x.dim() - 2)


def comp_sums(X):
    """sum of every entry of each component (axis 1)."""
    return X.sum([d for d in range(X.dim()) if d != 1])


def init_lambda(W, H, b, c):
    return (comp_sums(W) + comp_sums(H) + b) / c


def default_b(a, mean_v, R, prod_k=1):
    return math.sqrt((a - 1.0) * (a - 2.0) * mean_v / (R * prod_k))


def constants(W, H, a):
    """c = n_W + n_H + a + 1."""
    R = W.shape[1]
    return W.numel() // R + H.numel() // R + a + 1.0


def _sel(S, V):
    """The per-cell weight of a selector: None (every cell, weight 1), a bool mask or a float weight."""
    return None if S is None else S.to(V.dtype)


def divergence(V, W, H, beta, kind="nmf", S=None):
    recon = KINDS[kind][0]
    WH = recon(H, W)
    if S is None:
        return float(orc.beta_div(WH, V, beta))
    on = S > 0
    return float((S[on] * cell_div(WH[on], V[on], beta)).sum())


def objective(V, W, H, lam, beta, b, c, phi, kind="nmf", S=None):
    return divergence(V, W, H, beta, kind, S) / phi + float(
        ((comp_sums(W) + comp_sums(H) + b) / lam + c * lam.log()).sum())


def terms(V, W, H, beta, which, kind="nmf", S=None):
    """(num, den, den_is_colsum) of one factor's update."""
    recon, grad_w, grad_h = KINDS[kind]
    WH = recon(H, W)
    if S is None:
        Pn, Pp = orc.phi(V, WH, beta)
    else:
        on = S > 0
        zero = torch.zeros((), dtype=WH.dtype)
        Pn, Pp = orc.phi(torch.where(on, V, zero), WH, beta)
        if Pp is None:
            Pp = torch.ones_like(WH)
        Pn, Pp = torch.where(on, Pn * S, zero), torch.where(on, Pp * S, zero)
    grad = (lambda G: grad_w(G, H, W)) if which == 0 else (lambda G: grad_h(G, W, H))
    other = H if which == 0 else W
    if Pp is None:                                   # beta 1, every cell: the column sums of the other factor
        den = comp_sums(other).view(_rank_shape(W if which == 0 else H))
        return grad(Pn), den, True
    return grad(Pn), grad(Pp), False


def ratio(X, num, den, gamma, pen, colsum):
    """nmf.py:78-92 with l1 = pen[k] on component k, l2 = 0."""
    neg = num.clamp_min(0) + EPS
    pos = den if colsum else den.clamp_min(0) + EPS
    pos = pos + pen.view(_rank_shape(X))
    mult = neg / pos
    if gamma != 1:
        mult = mult.pow(gamma)
    return X * mult


def step(V, W, H, lam, beta, b, c, phi, kind="nmf", S=None):
    """One ARD iteration: (W, H, lambda, change)."""
    gamma = orc.gamma_of(beta)
    pen = phi / lam
    num, den, cs = terms(V, W, H, beta, 0, kind, S)
    W = ratio(W, num, den, gamma, pen, cs)
    num, den, cs = terms(V, W, H, beta, 1, kind, S)
    H = ratio(H, num, den, gamma, pen, cs)
    new = init_lambda(W, H, b, c)
    change = float(((new - lam).abs() / lam).max())
    return W, H, new, change


def fit(V, W, H, beta=1, tol=1e-5, max_iter=200, a=5.0, b=None, phi=1.0, kind="nmf", S=None, mean_v=None,
        trace=None, dtype=torch.float64):
    """The whole ARD fit in `dtype` (float64 by default).  Returns (W, H, lambda, n_iter, b, c).  `trace` (a list):
    receives J after the initialisation and after every iteration."""
    V, W, H = V.to(dtype), W.to(dtype), H.to(dtype)
    S = _sel(S, V) if S is not None else None
    R = W.shape[1]
    if b is None:
        if mean_v is None:
            mean_v = float(V.double().mean()) if S is None else float(V.double()[S > 0].mean())
        b = default_b(a, mean_v, R, math.prod(W.shape[2:]))
    c = constants(W, H, a)
    lam = init_lambda(W, H, b, c)
    if trace is not None:
        trace.append(objective(V, W, H, lam, beta, b, c, phi, kind, S))
    it = -1
    for it in range(max_iter):
        W, H, lam, change = step(V, W, H, lam, beta, b, c, phi, kind, S)
        if trace is not None:
            trace.append(objective(V, W, H, lam, beta, b, c, phi, kind, S))
        if it % 10 == 9 and change < tol:
            break
    return W, H, lam, it + 1, b, c
