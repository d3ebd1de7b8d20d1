"""Test-only engines that implement the engine interface of torchnmf_b200.engine with the CPU oracle.

They exist so the HOST logic (fit loop, validation, stop rule, sharded all-reduce protocol) can be
exercised on a machine with no GPU (`-m "not gpu"`, gloo).  They are never imported by the product.
"""
import torch

from oracle import hoyer_oracle as hoy
from oracle import mu_oracle as orc


class _OracleEngine:
    device = torch.device("cpu")
    precision = "oracle"

    def __init__(self, V, W, H):
        self.V, self.W, self.H = V, W, H      # W, H: the Parameter storages, updated in place

    def close(self):
        pass

    def sync(self):
        pass

    def minmax(self):
        return float(self.V.min()), float(self.V.max())

    def loss_tensor(self, beta):
        return orc.beta_div(self._recon(self.H, self.W), self.V, beta).double().reshape(1)

    def loss(self, beta):
        return float(self.loss_tensor(beta))

    # sparse_fit's extras (engine.py: project / loss_at / raw_terms)
    def project(self, x, dim, k1, k2):
        x.copy_(hoy.project_slices(x, dim, torch.as_tensor(k1), torch.as_tensor(k2)))
        return x

    def loss_at(self, W, H, beta):
        return float(orc.beta_div(self._recon(H, W), self.V, beta))

    def raw_terms(self, which, beta):
        """(raw numerator, raw denominator) of one factor's update; the denominator is (R,) for beta == 1."""
        Pn, Pp = orc.phi(self.V, self._recon(self.H, self.W), beta)
        contract = (lambda G: self._grad_w(G, self.H, self.W)) if which == 0 else (lambda G: self._grad_h(G, self.W, self.H))
        other = self.H if which == 0 else self.W
        den = other.sum([d for d in range(other.dim()) if d != 1]) if beta == 1 else contract(Pp)
        return contract(Pn), den


class OracleNmfEngine(_OracleEngine):
    kind = "nmf"
    _recon = staticmethod(orc.nmf_reconstruct)
    _grad_w = staticmethod(lambda G, H, W: G.t() @ H)
    _grad_h = staticmethod(lambda G, W, H: G @ W)

    def update_w(self, beta, gamma, l1, l2):
        self.W.copy_(orc.nmf_update_w(self.V, self.W, self.H, beta, gamma, l1, l2))

    def update_h(self, beta, gamma, l1, l2):
        self.H.copy_(orc.nmf_update_h(self.V, self.W, self.H, beta, gamma, l1, l2))

    # sharded pieces: same buffer layout as nmfb200_raw_terms(which = 0) (include/nmf_b200.h)
    def w_partial(self, beta):
        num, den = orc.nmf_w_contractions(self.V, self.W, self.H, beta)
        return torch.cat([num.reshape(-1), den.reshape(-1)]).contiguous()

    def w_apply(self, reduced, beta, gamma, l1, l2):
        C, R = self.W.shape
        num = reduced[:C * R].view(C, R)
        den = reduced[C * R:].view(1, R) if beta == 1 else reduced[C * R:].view(C, R)
        self.W.copy_(orc._ratio_update(self.W, num, den, gamma, l1, l2, beta == 1))


class OracleNmfdEngine(_OracleEngine):
    kind = "nmfd"
    _recon = staticmethod(orc.nmfd_reconstruct)
    _grad_w = staticmethod(lambda G, H, W: orc.nmfd_grad_w(G, H, W.shape[2]))
    _grad_h = staticmethod(lambda G, W, H: orc.nmfd_grad_h(G, W, H.shape[2]))

    def update_w(self, beta, gamma, l1, l2):
        self.W.copy_(orc.nmfd_update_w(self.V, self.W, self.H, beta, gamma, l1, l2))

    def update_h(self, beta, gamma, l1, l2):
        self.H.copy_(orc.nmfd_update_h(self.V, self.W, self.H, beta, gamma, l1, l2))


class OracleNmfndEngine(_OracleEngine):
    """One NMF2D / NMF3D problem on the CPU oracle (oracle/mu_oracle.py: nmfnd_*)."""
    kind = "nmfd"
    _recon = staticmethod(orc.nmfnd_reconstruct)

    def update_w(self, beta, gamma, l1, l2):
        self.W.copy_(orc.nmfnd_update_w(self.V, self.W, self.H, beta, gamma, l1, l2))

    def update_h(self, beta, gamma, l1, l2):
        self.H.copy_(orc.nmfnd_update_h(self.V, self.W, self.H, beta, gamma, l1, l2))
