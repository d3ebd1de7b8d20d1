"""Float64 coordinate descent (HALS) at beta 2, written from its update formula (torchnmf_b200.nmf.NMF.fit, solver="cd").

Objective:  1/2 |V - H W^T|^2 + l1 (sum W + sum H) + l2 / 2 (|W|^2 + |H|^2).
One update of a factor X with A = V^T H, B = H^T H (X = W) or A = V W, B = W^T W (X = H), both taken once at its start:
    for k = 0 .. R-1:  X[:,k] <- max(0, X[:,k] + (A[:,k] - X B[:,k] - l1 - l2 X[:,k]) / (B[k,k] + l2))
with the columns j < k already updated; a column with B[k,k] + l2 == 0 is left as it is.
"""
import math

import torch


def objective(V, W, H, l1=0.0, l2=0.0):
    """The objective the solver descends, in float64."""
    V, W, H = V.double(), W.double(), H.double()
    E = V - H @ W.t()
    return float(0.5 * (E * E).sum() + l1 * (W.sum() + H.sum()) + 0.5 * l2 * ((W * W).sum() + (H * H).sum()))


def sweep(X, A, B, l1=0.0, l2=0.0, on_step=None):
    """One HALS sweep of X (rows x R) over its columns in order; returns the new X (float64).  on_step(k, X) is called after
    every column step, the skipped ones included."""
    X, A, B = X.double().clone(), A.double(), B.double()
    for k in range(X.shape[1]):
        hess = float(B[k, k]) + l2
        if hess != 0.0:
            step = (A[:, k] - X @ B[:, k] - l1 - l2 * X[:, k]) / hess
            X[:, k] = (X[:, k] + step).clamp_min(0.0)
        if on_step is not None:
            on_step(k, X)
    return X


def terms(V, W, H, which):
    """(A, B) of the update of W (which = 0) or H (which = 1), float64."""
    V, W, H = V.double(), W.double(), H.double()
    return (V.t() @ H, H.t() @ H) if which == 0 else (V @ W, W.t() @ W)


def update(V, W, H, which, l1=0.0, l2=0.0, on_step=None):
    """The new W (which = 0) or H (which = 1) after one HALS update."""
    A, B = terms(V, W, H, which)
    return sweep(W if which == 0 else H, A, B, l1, l2, on_step)


def gradient(V, W, H, which, l1=0.0, l2=0.0):
    """The objective's gradient with respect to W (which = 0) or H (which = 1), float64."""
    A, B = terms(V, W, H, which)
    X = (W if which == 0 else H).double()
    return X @ B - A + l1 + l2 * X


def frobenius(V, W, H):
    """fit()'s beta-2 divergence 1/2 |V - H W^T|^2 (no penalties), float64."""
    E = V.double() - H.double() @ W.double().t()
    return float(0.5 * (E * E).sum())


def fit(V, W, H, tol=1e-4, max_iter=200, l1=0.0, l2=0.0, train_w=True, train_h=True, loss=frobenius):
    """HALS under the reference's stop rule (nmf.py:393-405): the loss sqrt(2 loss(V, W, H)) every 10th iteration, stop when
    it fell by less than tol x the initial loss.  W and H keep their dtype: each update is cast back to it.
    Returns (W, H, n_iter, losses at every check)."""
    W, H = W.clone(), H.clone()
    loss_init = math.sqrt(2.0 * loss(V, W, H))
    previous, checks, n_iter = loss_init, [], -1
    for n_iter in range(max_iter):
        if train_w:
            W = update(V, W, H, 0, l1, l2).to(W.dtype)
        if train_h:
            H = update(V, W, H, 1, l1, l2).to(H.dtype)
        if n_iter % 10 == 9:
            cur = math.sqrt(2.0 * loss(V, W, H))
            checks.append(cur)
            if (previous - cur) / loss_init < tol:
                break
            previous = cur
    return W, H, n_iter + 1, checks
