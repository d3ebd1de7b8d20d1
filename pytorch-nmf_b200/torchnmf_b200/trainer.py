"""`BetaMu`: the multiplicative-update optimizer of the reference (torchnmf/trainer.py:7-121) with a fused fast path.

Surface and semantics are the reference's: `BetaMu(params, beta=1, l1_reg=0, l2_reg=0, orthogonal=0)`, and
`step(closure)` with `closure() -> (target, prediction)` updates every trainable parameter of every group ONE AT A TIME
(prediction re-evaluated before each), leaves `p.grad = positive - negative` gradient term (= the gradient of the
beta-divergence, the identity tests/test_trainer.py:54-73 of the reference checks) and multiplies
`p <- p * ((neg + eps) / (pos + l1 + l2 p + ortho (rowsum(p) - p) + eps)) ** gamma` (trainer.py:98-114).

Two ways to obtain the two gradient terms `neg = relu(d<WH, V (WH+eps)^(beta-2)>/dp)` and
`pos = relu(d<WH, (WH+eps)^(beta-1)>/dp)`:

* generic: two vector-Jacobian products through whatever graph the closure built (torch.autograd.grad) -- any
  composition of modules, CPU or GPU; this is the reference's algorithm.
* fused (GPU): when the prediction is the plain reconstruction of ONE `torchnmf_b200.NMF` module on a CUDA device and `p`
  is that module's W or H, both terms come from ONE launch of the fused wgmma contraction
  (`nmfb200_nmf_raw_terms`): neither WH nor the ratio matrices are materialised by the update.  The closure may
  return the module itself instead of its output (`return V, model`) to skip the forward pass as well.  The
  convolutive modules (`NMFD`, `NMF2D`, `NMF3D`) take the same route through `nmfb200_nmfd_raw_terms` (the sliding
  contractions of csrc/nmfd.cu / csrc/tc_nmfd.cu instead of two passes through cuDNN's convolution backward).

`SparsityProj` (trainer.py:124-190): Hoyer's projected-gradient step around a loss closure.  The gradient is the
closure's own (autograd); the projection of every slice of every parameter -- in the reference a Python loop over the
slices around the TorchScript `_proj_func`, one host synchronisation per round and slice -- is one
`nmfb200_hoyer_project` launch per parameter.
"""
import weakref

import torch
from torch.optim.optimizer import Optimizer

from .constants import eps
from . import engine as _engine

__all__ = ["BetaMu", "SparsityProj"]


def _gamma(beta):
    # trainer.py:63-68 (= nmf.py:341-346)
    if beta < 1:
        return 1.0 / (2.0 - beta)
    if beta > 2:
        return 1.0 / (beta - 1.0)
    return 1.0


def _phi(V, WH, beta):
    """(output_neg, output_pos) of trainer.py:79-90."""
    if beta == 2:
        return V, WH
    if beta == 1:
        return V / (WH + eps), torch.ones_like(WH)
    x = WH + eps
    if beta == 0:
        r = 1.0 / x
        return V * r * r, r
    return V * x.pow(beta - 2), x.pow(beta - 1)


class _FusedTerms:
    """Engine cache of the fused path: one `CudaNmfEngine` per (module, target) pair, rebuilt when either changes."""

    def __init__(self):
        self._key = None
        self._eng = None

    def close(self):
        if self._eng is not None:
            self._eng.close()
        self._eng, self._key = None, None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def terms(self, module, p, V, beta):
        """(neg_raw, pos_raw) for p in {module.W, module.H}, or None when the fused path does not apply."""
        W, H = module.W, module.H
        if W is None or H is None or (p is not W and p is not H):
            return None
        nd = W.dim() - 2                                  # convolved axes: 0 for NMF, 1..3 for NMFD / NMF2D / NMF3D
        if not (V.is_cuda and not V.is_sparse and V.dtype == torch.float32 and 0 <= nd <= 3 and V.dim() == W.dim()):
            return None
        if not (W.is_cuda and H.is_cuda and W.dtype == torch.float32 and H.dtype == torch.float32
                and W.device == V.device and H.device == V.device and H.dim() == W.dim()
                and W.data.is_contiguous() and H.data.is_contiguous()):
            return None
        if W.shape[1] != H.shape[1] or W.shape[1] > 256:
            return None
        want = (H.shape[0], W.shape[0]) + tuple(j + k - 1 for j, k in zip(H.shape[2:], W.shape[2:]))
        if tuple(V.shape) != want:
            return None
        Vc = V if V.is_contiguous() else V.contiguous()
        key = (id(module), Vc.data_ptr(), Vc._version, tuple(Vc.shape), W.data_ptr(), H.data_ptr())
        if key != self._key:
            self.close()
            make = _engine.CudaNmfEngine if nd == 0 else _engine.CudaNmfdEngine
            self._eng = make(Vc, W.data, H.data, "auto")
            self._key = key
            self._keep = Vc            # the engine borrows the target's storage
        else:
            self._eng.sync()           # W or H may have been changed by anyone since the last step
        which = 0 if p is W else 1
        num, den = self._eng.raw_terms(which, beta)
        if beta == 1:                  # trainer.py:83-84: backward of ones = column sums of the other factor
            den = den.view(1, -1, *([1] * nd)).expand_as(num) if nd else den.expand_as(num)
        return num, den


class BetaMu(Optimizer):
    """Multiplicative updater for NMF models minimising the beta-divergence (reference: trainer.py:7-34).

    Note:
        As in the reference, parameters and every gradient along the computational graph must be non-negative.

    Arguments:
        params: iterable of parameters or dicts defining parameter groups
        beta: the beta-divergence to minimise.  Default: 1
        l1_reg / l2_reg / orthogonal: L1, L2 (weight decay) and orthogonality penalties.  Default: 0
    """

    def __init__(self, params, beta=1, l1_reg=0, l2_reg=0, orthogonal=0):
        if not 0.0 <= l1_reg:
            raise ValueError("Invalid l1_reg value: {}".format(l1_reg))
        if not 0.0 <= l2_reg:
            raise ValueError("Invalid l2_reg value: {}".format(l2_reg))
        if not 0.0 <= orthogonal:
            raise ValueError("Invalid orthogonal value: {}".format(orthogonal))
        super().__init__(params, dict(beta=beta, l1_reg=l1_reg, l2_reg=l2_reg, orthogonal=orthogonal))
        self._fused = _FusedTerms()
        self.last_step_paths = []      # "fused" / "autograd" per updated parameter of the last step (introspection, tests)

    @torch.no_grad()
    def step(self, closure):
        """One pass over all trainable parameters.  `closure() -> (target, prediction)`; see the module docstring."""
        closure = torch.enable_grad()(closure)
        params = [p for g in self.param_groups for p in g["params"]]
        trainable = {id(p): p.requires_grad for p in params}
        for p in params:
            p.requires_grad = False
        self.last_step_paths = []
        try:
            for group in self.param_groups:
                beta, gamma = group["beta"], _gamma(group["beta"])
                l1_reg, l2_reg, ortho = group["l1_reg"], group["l2_reg"], group["orthogonal"]
                for p in group["params"]:
                    if not trainable[id(p)]:
                        continue
                    p.requires_grad = True
                    V, WH = closure()
                    neg = pos = None
                    module = WH if isinstance(WH, torch.nn.Module) else _source_module(WH)
                    if module is not None:
                        got = self._fused.terms(module, p, V, beta)
                        if got is not None:
                            neg, pos = got
                            self.last_step_paths.append("fused")
                    if neg is None:
                        if isinstance(WH, torch.nn.Module):
                            WH = WH()                  # the closure returned the module: evaluate it (generic path)
                        if not WH.requires_grad:       # trainer.py:75-77: p does not take part in the prediction
                            p.requires_grad = False
                            continue
                        out_neg, out_pos = _phi(V, WH, beta)
                        neg, = torch.autograd.grad(WH, p, out_neg, retain_graph=True)
                        pos, = torch.autograd.grad(WH, p, out_pos)
                        self.last_step_paths.append("autograd")
                    neg = neg.clamp_min(0)                                    # trainer.py:93
                    p.grad = pos - neg                                        # trainer.py:94-97: raw positive term - relu(negative)
                    pos = pos.clamp_min(0)
                    if l1_reg > 0:
                        pos = pos + l1_reg                                    # trainer.py:99-100
                    if l2_reg > 0:
                        pos = pos + l2_reg * p                                # trainer.py:101-102
                    if ortho > 0:
                        pos = pos + ortho * (p.sum(1, keepdim=True) - p)      # trainer.py:104-105
                    mult = (neg + eps) / (pos + eps)                          # trainer.py:107-109
                    if gamma != 1:
                        mult = mult.pow(gamma)                                # trainer.py:110-111
                    p.mul_(mult)                                              # trainer.py:113
                    p.requires_grad = False
        finally:
            for p in params:
                p.requires_grad = trainable[id(p)]
        return None


def _source_module(WH):
    """The NMF module whose plain reconstruction `WH` is (tagged by `NMF.forward`), else None."""
    ref = getattr(WH, "_nmf_b200_src", None)
    return ref() if isinstance(ref, weakref.ref) else None


def _get_norm(x, axis=1):
    """nmf.py:134-139."""
    dims = [d for d in range(x.dim()) if d != axis]
    return (x * x).sum(dims).sqrt()


def _project_slices_(p, dim, k1, k2):
    """Every slice of `p` along `dim` <- its Hoyer projection (nmf.py:21-49), in place, in the library.  A parameter that
    is not a contiguous fp32 CUDA tensor is staged through one (host buffers: through the current CUDA device, like `fit`)."""
    if p.is_cuda and p.dtype == torch.float32 and p.is_contiguous():
        _engine.hoyer_project_(p, dim, k1, k2)
        return
    if not (p.is_cuda or torch.cuda.is_available()):
        raise RuntimeError("SparsityProj needs a CUDA device (sm_90a) for the projection; there is no CPU fallback")
    dev = p.device if p.is_cuda else torch.device("cuda", torch.cuda.current_device())
    tmp = p.detach().to(dev, torch.float32).contiguous()
    _engine.hoyer_project_(tmp, dim, torch.as_tensor(k1).to(dev), torch.as_tensor(k2).to(dev))
    p.copy_(tmp)


class SparsityProj(Optimizer):
    """Sparseness-constrained gradient projection (Hoyer 2004; reference: trainer.py:124-147).

    Arguments:
        params: iterable of parameters or dicts defining parameter groups
        sparsity: the target sparseness of every slice of every parameter, 0 < sparsity < 1
        dim: the axis whose slices are the constrained vectors.  Default: 1
        max_iter: maximal number of loss evaluations per step.  Default: 10
    """

    def __init__(self, params, sparsity, dim=1, max_iter=10):
        if not 0.0 < sparsity < 1.:
            raise ValueError("Invalid sparsity value: {}".format(sparsity))
        super().__init__(params, dict(sparsity=sparsity, lr=1, dim=dim, max_iter=max_iter))

    @torch.no_grad()
    def step(self, closure):
        """One projected-gradient step per parameter group with a halving line search (trainer.py:150-190).
        `closure()` re-evaluates the model and returns the loss."""
        loss = None
        for group in self.param_groups:
            sparsity, lr, dim, max_iter = group["sparsity"], group["lr"], group["dim"], group["max_iter"]
            with torch.enable_grad():
                init_loss = closure()
                init_loss.backward()
            params = [(p, p.grad.clone()) for p in group["params"] if p.grad is not None]
            for _ in range(max_iter):
                for p, g in params:
                    norms = _get_norm(p, dim)                                  # trainer.py:173: of p BEFORE the step
                    p.add_(g, alpha=-lr)
                    n = p.numel() // p.shape[dim]
                    L1 = n ** 0.5 * (1 - sparsity) + sparsity
                    _project_slices_(p, dim, L1 * norms, norms * norms)        # trainer.py:176-181
                loss = closure()
                if loss <= init_loss:
                    break
                for p, g in params:
                    p.add_(g, alpha=lr)                                        # trainer.py:186-187
                lr *= 0.5
            lr *= 1.2
            group["lr"] = lr
        return loss
