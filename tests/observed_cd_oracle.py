"""Float64 coordinate descent at beta 2 on the observed cells, written naively from its update formula
(torchnmf_b200.nmf.NMF.fit, solver="cd" with a sparse mask or weight; include/nmf_b200.h: nmfb200_nmf_observed_cd_update).

Objective, with M the cells' weights (0: not observed, 1 for a mask):
    1/2 sum M (V - H W^T)^2 + l1 (sum W + sum H) + l2 / 2 (|W|^2 + |H|^2).
One update of a factor X with the other factor F fixed; every row s of X on its own, over its segment's cells; for k = 0 ..
R-1 in order, with the residual r = v - F x_s recomputed at the current x_s (entries j < k already updated):
    num = sum_j w_j r_j f_{j,k},  hess = sum_j w_j f_{j,k}^2 + l2,  if hess != 0: x_{s,k} <- max(0, x_{s,k} + (num - l1 -
    l2 x_{s,k}) / hess).
The rows are independent, so each column step is taken on every row at once, from the list of observed cells.  None
of the kernel's grouping is mirrored.
"""
import math

import torch


def dense_weights(O, weights=None):
    """(V, M) float64 of an observed-cell tensor O (sparse COO, the stored entries are the observed cells) and its entries'
    weights (None: 1): V holds O's values (0 elsewhere), M the weights (0 elsewhere)."""
    O = O.coalesce()
    V = torch.zeros(O.shape, dtype=torch.float64)
    M = torch.zeros(O.shape, dtype=torch.float64)
    rows, cols = O.indices().cpu()
    V[rows, cols] = O.values().cpu().double()
    M[rows, cols] = 1.0 if weights is None else weights.cpu().double()
    return V, M


def objective(V, M, W, H, l1=0.0, l2=0.0):
    W, H = W.double(), H.double()
    E = V - H @ W.t()
    return float(0.5 * (M * E * E).sum() + l1 * (W.sum() + H.sum()) + 0.5 * l2 * ((W * W).sum() + (H * H).sum()))


def loss(V, M, W, H):
    """fit()'s beta-2 divergence on the observed cells, 1/2 sum M (V - H W^T)^2 (no penalties), float64."""
    return objective(V, M, W, H)


def update(V, M, W, H, which, l1=0.0, l2=0.0, on_step=None):
    """The new W (which = 0) or H (which = 1), float64.  on_step(k, X) is called after every column step."""
    n, c = M.nonzero(as_tuple=True)                       # the observed cells
    v, w = V[n, c].double(), M[n, c].double()
    if which == 0:
        seg, oth, X, F = c, n, W.double().clone(), H.double()
    else:
        seg, oth, X, F = n, c, H.double().clone(), W.double()
    Fo = F[oth]                                           # f_j of every observed cell j
    for k in range(X.shape[1]):
        r = v - (X[seg] * Fo).sum(1)                      # at the current x_s: recomputed for every k
        num = torch.zeros(X.shape[0], dtype=torch.float64).index_add_(0, seg, w * r * Fo[:, k])
        hess = torch.zeros(X.shape[0], dtype=torch.float64).index_add_(0, seg, w * Fo[:, k] * Fo[:, k]) + l2
        live = hess != 0
        new = (X[:, k] + (num - l1 - l2 * X[:, k]) / torch.where(live, hess, torch.ones_like(hess))).clamp_min(0.0)
        X[:, k] = torch.where(live, new, X[:, k])
        if on_step is not None:
            on_step(k, X)
    return X


def gradient(V, M, W, H, which, l1=0.0, l2=0.0):
    """The objective's gradient with respect to W (which = 0) or H (which = 1), float64."""
    W, H = W.double(), H.double()
    E = M * (H @ W.t() - V)
    return (E.t() @ H + l1 + l2 * W) if which == 0 else (E @ W + l1 + l2 * H)


def fit(V, M, W, H, tol=1e-4, max_iter=200, l1=0.0, l2=0.0, train_w=True, train_h=True):
    """Observed-cell coordinate descent under the reference's stop rule (nmf.py:393-405): the loss sqrt(2 loss) every 10th
    iteration, stop when it fell by less than tol x the initial loss.  W and H keep their dtype: each update is cast back to
    it.  Returns (W, H, n_iter, losses at every check)."""
    W, H = W.clone(), H.clone()
    loss_init = math.sqrt(2.0 * loss(V, M, W, H))
    previous, checks, n_iter = loss_init, [], -1
    for n_iter in range(max_iter):
        if train_w:
            W = update(V, M, W, H, 0, l1, l2).to(W.dtype)
        if train_h:
            H = update(V, M, W, H, 1, l1, l2).to(H.dtype)
        if n_iter % 10 == 9:
            cur = math.sqrt(2.0 * loss(V, M, W, H))
            checks.append(cur)
            if (previous - cur) / loss_init < tol:
                break
            previous = cur
    return W, H, n_iter + 1, checks


class ObservedCdOracleEngine:
    """An engine for the `_engine_factory` hook of NMF.fit on a sparse mask or weight: it takes the observed-cell tensor O
    (and the entries' weights) the fit builds, and runs the two coordinate-descent calls and the loss on this oracle.  Every
    call is logged in `calls`, every tensor O it is given in `received` (class-level lists a test may reset)."""
    kind = "nmf"
    device = torch.device("cpu")
    precision = "f32"
    calls = []
    received = []

    def __init__(self, O, W, H, weights=None):
        assert O.is_sparse and O.is_coalesced() and O.dtype == torch.float32
        ObservedCdOracleEngine.received.append((O, weights))
        self.V, self.M = dense_weights(O, weights)
        self.W, self.H = W, H                              # the Parameter storages, updated in place

    def close(self):
        pass

    def minmax(self):
        vals = self.V[self.M > 0]
        return (float(vals.min()), float(vals.max())) if vals.numel() else (math.inf, -math.inf)

    def loss(self, beta):
        assert beta == 2
        d = loss(self.V, self.M, self.W, self.H)
        self.calls.append(("loss", d))
        return d

    def cd_update(self, which, l1, l2):
        self.calls.append(("cd_update", which, l1, l2))
        X = self.W if which == 0 else self.H
        X.copy_(update(self.V, self.M, self.W, self.H, which, l1, l2))

    def cd_iterate(self, n_iter, l1, l2):
        self.calls.append(("cd_iterate", n_iter, l1, l2))
        for _ in range(n_iter):
            self.W.copy_(update(self.V, self.M, self.W, self.H, 0, l1, l2))
            self.H.copy_(update(self.V, self.M, self.W, self.H, 1, l1, l2))
