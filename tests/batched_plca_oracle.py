"""A float64 CPU model of the batched PLCA engine (engine._BatchedEngine.plca_iterate / plca_losses), for the host logic of
the Batched*PLCA classes through their `_engine_factory` hook, and for the GPU tests' term-by-term checks of the EM step.

Each problem's EM step is oracle/plca_oracle.py's (the reference's plca.py:247-289) in float64, except that a frozen Z
with trainable W takes W's column sums as the prior as a rank vector at every rank (the reference squeezes it, which
leaves a 0-d prior at rank 1)."""
import torch

from oracle import plca_oracle as orc


def _per_problem(x):
    """The per-problem column sums of a factor (problems on axis 0, rank on axis 2), kept for broadcasting."""
    return x.sum([d for d in range(x.dim()) if d not in (0, 2)], keepdim=True)


def _rank(z, x):
    """A (P, R) tensor against the rank axis (2) of a batched factor."""
    return z.reshape(z.shape[0], 1, z.shape[1], *([1] * (x.dim() - 3)))


def _prior(x, alpha):
    if alpha is None:
        return x, False
    x = x + (alpha - 1)
    return torch.where(x > orc.EPS, x, torch.full_like(x, orc.EPS)), True


def em_step(W, H, Z, dW, dHz, train_w, train_h, train_z, W_alpha=None, H_alpha=None, Z_alpha=None):
    """One EM step of every problem from the raw numerators dW (W's shape) and dHz (H's shape): the new (W, H, Z), all
    batched (problems on axis 0).  Alphas: None (1) or tensors of the batched factor's shape."""
    Zo = Z
    dH = dHz * _rank(Zo, H)
    prior = None
    if train_z:                                                         # plca.py:256-262
        dZ = (H * dHz).sum([d for d in range(H.dim()) if d not in (0, 2)])
        Z = Z * dZ.clamp_min(0)
        prior = Z.clone()
        Z, _ = _prior(Z, Z_alpha)
        Z = Z / Z.sum(1, keepdim=True)
    if train_w:                                                         # plca.py:264-275
        W = W * dW.clamp_min(0)
        if prior is None:
            div = _per_problem(W)
            prior = div.reshape(W.shape[0], -1)
        else:
            div = _rank(prior, W)
        W, renorm = _prior(W / div, W_alpha)
        if renorm:
            W = W / _per_problem(W)
    if train_h:                                                         # plca.py:277-288
        H = H * dH.clamp_min(0)
        div = _per_problem(H) if prior is None else _rank(prior, H)
        H, renorm = _prior(H / div, H_alpha)
        if renorm:
            H = H / _per_problem(H)
    return W, H, Z


def raw_terms(Vn, W, Hz):
    """(dW, dHz) of every problem in float64: the contractions of Vn / (X + eps) with H Z and with W."""
    dWs, dHs = [], []
    for p in range(W.shape[0]):
        X = orc.reconstruct(Hz[p], W[p], torch.ones(W.shape[2], dtype=W.dtype))
        Pm = Vn[p] / (X + orc.EPS)
        if W.dim() == 3:
            dWs.append(Pm.t() @ Hz[p]); dHs.append(Pm @ W[p])
        else:
            dWs.append(orc.mu.nmfnd_grad_w(Pm, Hz[p], tuple(W.shape[3:])))
            dHs.append(orc.mu.nmfnd_grad_h(Pm, W[p], tuple(Hz.shape[3:])))
    return torch.stack(dWs), torch.stack(dHs)


def kl_loss(Vn, W, Hz, norm):
    """kl_div(norm_p X_p, norm_p Vn_p) of every problem, float64 (P,)."""
    out = []
    for p in range(W.shape[0]):
        X = orc.reconstruct(Hz[p], W[p], torch.ones(W.shape[2], dtype=W.dtype)) * norm[p]
        t = Vn[p] * norm[p]
        out.append(float((t * (torch.log(t + orc.EPS) - torch.log(X + orc.EPS))).sum() - t.sum() + X.sum()))
    return torch.tensor(out, dtype=torch.float64)


class BatchedPlcaOracleEngine:
    """The batched engine interface the Batched*PLCA fit uses (plca_iterate, plca_losses, set_active), every problem's EM
    iteration in float64 on the CPU.  Counts the EM steps each problem receives, so a test can see that a stopped problem
    is never touched again, and keeps the alpha buffers it was given."""
    kind = "plca_batched"
    device = torch.device("cpu")

    def __init__(self, Vn, W, Hz):
        P = W.shape[0]
        if Vn.dim() == W.dim() - 1:
            Vn = Vn.expand(P, *Vn.shape)
        self.Vn = Vn.double()
        self.W, self.H = W, Hz
        self.active = torch.ones(P, dtype=torch.bool)
        self.steps = [0] * P
        self.alphas = None
        self._last = torch.full((P,), float("nan"), dtype=torch.float64)

    def close(self):
        pass

    def check_health(self):
        pass

    def set_active(self, active):
        self.active = torch.as_tensor(active, dtype=torch.bool).clone()

    def plca_iterate(self, n_iter, H, Z, train_w, train_h, train_z, W_alpha=None, H_alpha=None, Z_alpha=None):
        self.alphas = (W_alpha, H_alpha, Z_alpha)
        a = self.active
        dbl = [x.double() if x is not None else None for x in (W_alpha, H_alpha, Z_alpha)]
        for _ in range(n_iter):
            W64, H64, Z64 = self.W.double(), H.double(), Z.double()
            dW, dHz = raw_terms(self.Vn, W64, self.H.double())
            Wn, Hn, Zn = em_step(W64, H64, Z64, dW, dHz, train_w, train_h, train_z, *dbl)
            self.W[a] = Wn[a].float(); H[a] = Hn[a].float(); Z[a] = Zn[a].float()
            self.H[a] = (H[a] * _rank(Z[a], H[a]))
            for p in range(len(self.steps)):
                self.steps[p] += int(a[p])

    def plca_losses(self, norm):
        d = kl_loss(self.Vn, self.W.double(), self.H.double(), norm.double())
        self._last[self.active] = d[self.active]
        return self._last.clone()
