"""PLCA / SIPLCA / SIPLCA2 / SIPLCA3 with the reference's module surface (torchnmf/plca.py:28-625) and an H100-native `fit`.

    V (N, C) / sum(V)  ~=  H (N, R) diag(Z (R,)) W (C, R)^T,     W, H column-normalised, Z a distribution.

The reference's EM iteration (plca.py:247-289) materialises WZH, takes ONE backward pass of V / (WZH + eps) through it and
updates Z, W and H simultaneously from the three gradients.  Here the two big contractions

    dW[c, r] = sum_n P[n, c] (H Z)[n, r],      dHz[n, r] = sum_c P[n, c] W[c, r],      P = V / ((H Z) W^T + eps)

are two launches of the fused wgmma KL contraction (`nmfb200_nmf_raw_terms` with the factor pair (W, H diag Z)): neither
WZH nor P reaches HBM.  dH = dHz * Z and dZ[r] = sum_n H[n, r] dHz[n, r] follow from them; everything after that is the
reference's sequence of small factor-sized operations (plca.py:256-289).

The shift-invariant models (plca.py:376-625) are the same EM step around the convolutive reconstruction
`sum_{r,t} W[c,r,t] Z[r] H[b,r,x-t]`: the factor pair handed to the library is (W, H Z) as well, and the two gradients are
the sliding contractions of `nmfb200_nmfd_raw_terms` (wgrad and dgrad of the ratio tile; csrc/nmfd.cu, csrc/tc_nmfd.cu).
"""
import math
from collections.abc import Iterable as _Iterable

import torch
import torch.nn.functional as F
from torch import Tensor
from torch.nn import Parameter

from .constants import eps
from . import engine as _engine

from torch.nn.modules.utils import _single, _pair, _triple

try:
    from tqdm import tqdm as _tqdm
except Exception:  # pragma: no cover
    _tqdm = None

__all__ = ["PLCA", "SIPLCA", "SIPLCA2", "SIPLCA3", "BaseComponent"]


@torch.no_grad()
def get_norm(x):
    """Sum over every dimension but the rank dimension (1), kept for broadcasting; the plain sum for a vector (plca.py:24-31)."""
    if x.ndim > 1:
        return x.sum([d for d in range(x.dim()) if d != 1], keepdim=True)
    return x.sum()


def _kl(x, t):
    # metrics.kl_div (metrics.py:22) on the de-normalised reconstruction / target, as plca.py:245,293 evaluates it
    return t.reshape(-1) @ (torch.log(t + eps) - torch.log(x + eps)).reshape(-1) - t.sum() + x.sum()


class BaseComponent(torch.nn.Module):
    """Base of the PLCA modules (reference: plca.py:34-184): W, H column-normalised probabilities, Z the latent prior."""

    def __init__(self, rank=None, W=None, H=None, Z=None, trainable_W=True, trainable_H=True, trainable_Z=True):
        super().__init__()
        inferred = None
        for name, spec, trainable in (("W", W, trainable_W), ("H", H, trainable_H)):
            if isinstance(spec, Tensor):
                assert torch.all(spec >= 0.), f"Tensor {name} should be non-negative."        # plca.py:101,116
                p = Parameter(torch.empty(*spec.size()), requires_grad=trainable)
                p.data.copy_(spec)
                self.register_parameter(name, p)
            elif isinstance(spec, _Iterable):
                self.register_parameter(name, Parameter(torch.randn(*tuple(spec)).abs()))   # plca.py:106,122
            else:
                self.register_parameter(name, None)
            p = getattr(self, name)
            if p is not None:
                p.data.div_(get_norm(p))                                                     # plca.py:110-112,126-128
                inferred = p.shape[1]
        if isinstance(Z, Tensor):
            assert Z.ndim == 1, "Z should be one dimensional."
            assert torch.all(Z >= 0.), "Tensor Z should be non-negative."
            rank = Z.numel()
            self.register_parameter("Z", Parameter(torch.empty(rank), requires_grad=trainable_Z))
            self.Z.data.copy_(Z)
        elif isinstance(rank, int):
            self.register_parameter("Z", Parameter(torch.ones(rank) / rank))                # plca.py:138-139
        else:
            self.register_parameter("Z", None)
        if self.Z is not None:
            self.Z.data.div_(get_norm(self.Z))
            inferred = self.Z.shape[0]
        if inferred is None:
            assert rank, "A rank should be given when W, H and Z are not available!"
        else:
            if self.Z is not None:
                assert self.Z.shape[0] == inferred, "Latent size of Z does not match with others!"
            if self.H is not None:
                assert self.H.shape[1] == inferred, "Latent size of H does not match with others!"
            if self.W is not None:
                assert self.W.shape[1] == inferred, "Latent size of W does not match with others!"
                self.out_channels = self.W.shape[0]
                if self.W.ndim > 2:
                    self.kernel_size = self.W.shape[2:]
            rank = inferred
        self.rank = rank

    def extra_repr(self):
        s = f"{self.rank}"
        if self.W is not None:
            s += f", out_channels={self.out_channels}"
            if hasattr(self, "kernel_size"):
                s += f", kernel_size={tuple(self.kernel_size)}"
        return s

    def forward(self, H=None, W=None, Z=None, norm=None):
        """Reconstruction (plca.py:164-183), scaled by `norm` when given."""
        H = self.H if H is None else H
        W = self.W if W is None else W
        Z = self.Z if Z is None else Z
        out = self.reconstruct(H, W, Z)
        return out if norm is None else out * norm

    @staticmethod
    def reconstruct(H, W, Z):
        raise NotImplementedError

    @torch.no_grad()
    def fit(self, V, tol=1e-4, max_iter=200, verbose=False, W_alpha=1., H_alpha=1., Z_alpha=1., *, precision="f32"):
        """EM fit of the PLCA model (reference: plca.py:193-304; same arguments, stop rule and return value
        `(n_iter, norm)`).  Runs on the parameters' CUDA device; host-resident modules are staged like `NMF.fit`.

        precision: "f32" (default: the fused fp32 CUDA-core contraction, matches the reference to 1e-5 on the fixtures) |
                   "f16" / "f16_split" (wgmma contraction: ~10x faster at large shapes; the EM recursion keeps the
                   fp16 operand rounding, measured 1.0-1.4e-3 relative after 30-50 iterations on the fixtures of
                   tests/golden/reference_next.npz -- outside the 1e-3 bar, hence opt-in)."""
        assert torch.all(V >= 0.), "Target should be non-negative."                         # plca.py:236
        W, H, Z = self.W, self.H, self.Z
        assert W is not None and H is not None and Z is not None, "fit() needs W, H and Z"
        if not torch.cuda.is_available():
            raise RuntimeError("torchnmf_b200.PLCA.fit needs a CUDA device (sm_90a); there is no CPU fallback")
        f32 = torch.float32
        on_gpu = W.device.type == "cuda"
        dev = W.device if on_gpu else torch.device("cuda", torch.cuda.current_device())
        norm = V.sum()
        Vn = (V.to(dev, f32).contiguous() / norm.to(dev, f32)).contiguous()                  # plca.py:241-242
        stage = not (on_gpu and all(t.dtype == f32 for t in (W, H, Z)))
        Wd = W.data.to(dev, f32).contiguous() if stage else W.data
        Hd = H.data.to(dev, f32).contiguous() if stage else H.data
        Zd = Z.data.to(dev, f32).contiguous() if stage else Z.data
        normd = norm.to(dev, f32)
        Vfull = Vn * normd

        def loss_now():
            WZH = self.reconstruct(Hd, Wd, Zd)
            d = float(_kl(WZH * normd, Vfull))
            return math.sqrt(2.0 * d) if d >= 0 else float("nan")                           # plca.py:245-246,293-294

        def over(z, x):                               # a rank vector against the rank dimension (1) of a factor
            return z[(slice(None),) + (None,) * (x.dim() - 2)]                               # plca.py:269-270,282-283

        Hz = (Hd * over(Zd, Hd)).contiguous()         # the engine's activation factor: H diag(Z)
        eng = self._engine(Vn, Wd, Hz, precision)
        try:
            loss_init = previous_loss = loss_now()
            bar = _tqdm(total=max_iter, disable=not verbose) if _tqdm is not None else None
            n_iter = -1
            for n_iter in range(max_iter):
                torch.mul(Hd, over(Zd, Hd), out=Hz)
                eng.sync()
                dW, _ = eng.raw_terms(0, 1.0)         # P contracted with H Z  = W.grad   (plca.py:252-253)
                dHz, _ = eng.raw_terms(1, 1.0)        # P contracted with W;  H.grad = dHz * Z,  Z.grad = sum H dHz
                dH = dHz * over(Zd, Hd)
                dZ = get_norm(Hd * dHz).reshape(-1)
                Z_prior = None
                if Z.requires_grad:                                                          # plca.py:256-262
                    Zd.mul_(dZ.clamp_min(0))
                    Z_prior = Zd.clone()
                    if not _is_one(Z_alpha):
                        Zd.add_(_as(Z_alpha, Zd) - 1)
                        F.threshold(Zd, eps, eps, True)
                    Zd.div_(Zd.sum())
                if W.requires_grad:                                                          # plca.py:264-275
                    Wd.mul_(dW.clamp_min(0))
                    if Z_prior is None:
                        W_div = get_norm(Wd)
                        Z_prior = W_div.squeeze()
                    else:
                        W_div = over(Z_prior, Wd)
                    Wd.div_(W_div)
                    if not _is_one(W_alpha):
                        Wd.add_(_as(W_alpha, Wd) - 1)
                        F.threshold(Wd, eps, eps, True)
                        Wd.div_(get_norm(Wd))
                if H.requires_grad:                                                          # plca.py:277-288
                    Hd.mul_(dH.clamp_min(0))
                    H_div = get_norm(Hd) if Z_prior is None else over(Z_prior, Hd)
                    Hd.div_(H_div)
                    if not _is_one(H_alpha):
                        Hd.add_(_as(H_alpha, Hd) - 1)
                        F.threshold(Hd, eps, eps, True)
                        Hd.div_(get_norm(Hd))
                if n_iter % 10 == 9:                                                         # plca.py:290-302
                    loss = loss_now()
                    if bar is not None:
                        bar.set_postfix(loss=loss)
                        bar.update(10)
                    if (previous_loss - loss) / loss_init < tol:
                        break
                    previous_loss = loss
            eng.check_health()
            self.last_fit_precision = eng.precision_for(1.0)
            if bar is not None:
                bar.close()
        finally:
            eng.close()
        if stage:
            W.data.copy_(Wd); H.data.copy_(Hd); Z.data.copy_(Zd)
        return n_iter, norm                                                                  # plca.py:304


    @staticmethod
    def _engine(Vn, W, Hz, precision):
        raise NotImplementedError


def _is_one(a):
    return not isinstance(a, Tensor) and a == 1


def _as(a, like):
    return a.to(like.device, like.dtype) if isinstance(a, Tensor) else a


class PLCA(BaseComponent):
    """Probabilistic latent component analysis  V / sum(V) ~= H diag(Z) W^T  (reference: plca.py:307-373).
    V (N, C), W (C, R), H (N, R), Z (R,)."""

    def __init__(self, Vshape=None, rank=None, **kwargs):
        if isinstance(Vshape, _Iterable):
            M, K = Vshape
            rank = rank if rank else K
            kwargs["W"] = (K, rank)
            kwargs["H"] = (M, rank)
        super().__init__(rank, **kwargs)

    @staticmethod
    def reconstruct(H, W, Z):
        return H @ (W * Z).t()                       # plca.py:371-373

    @staticmethod
    def _engine(Vn, W, Hz, precision):
        return _engine.CudaNmfEngine(Vn, W, Hz, precision)


class _ShiftInvariant(BaseComponent):
    """The shift-invariant models: V (B, C, *X), W (C, R, *K), H (B, R, *(X - K + 1)), Z (R,)."""

    @staticmethod
    def _engine(Vn, W, Hz, precision):
        return _engine.CudaNmfdEngine(Vn, W, Hz, precision)


def _flip_conv(conv, H, W, Z):
    # plca.py:453-455, :534-537, :621-625: full-padding convolution with the flipped kernel, the prior on the rank axis
    nd = W.dim() - 2
    kernel = W.flip(tuple(range(2, 2 + nd))) * Z.view(-1, *([1] * nd))
    return conv(H, kernel, padding=tuple(k - 1 for k in W.shape[2:]))


class SIPLCA(_ShiftInvariant):
    """Shift-invariant PLCA along one axis (reference: plca.py:376-455).
    V (B, C, L), W (C, R, T), H (B, R, L - T + 1), Z (R,):  P(b, c, l) ~= sum_z sum_t P(c, t | z) P(z) P(b, l - t | z)."""

    def __init__(self, Vshape=None, rank=None, T=1, **kwargs):
        if isinstance(Vshape, _Iterable):
            T, = _single(T)
            batch, K, M = Vshape
            rank = rank if rank else K
            kwargs["W"] = (K, rank, T)
            kwargs["H"] = (batch, rank, M - T + 1)
        super().__init__(rank, **kwargs)

    @staticmethod
    def reconstruct(H, W, Z):
        return _flip_conv(F.conv1d, H, W, Z)


class SIPLCA2(_ShiftInvariant):
    """Shift-invariant PLCA along two axes (reference: plca.py:458-537).
    V (B, C, L, M), W (C, R, k0, k1), H (B, R, L - k0 + 1, M - k1 + 1), Z (R,)."""

    def __init__(self, Vshape=None, rank=None, kernel_size=1, **kwargs):
        if isinstance(Vshape, _Iterable):
            kernel_size = _pair(kernel_size)
            k0, k1 = kernel_size
            batch, channel, K, M = Vshape
            rank = rank if rank else K
            kwargs["W"] = (channel, rank) + kernel_size
            kwargs["H"] = (batch, rank, K - k0 + 1, M - k1 + 1)
        super().__init__(rank, **kwargs)

    @staticmethod
    def reconstruct(H, W, Z):
        return _flip_conv(F.conv2d, H, W, Z)


class SIPLCA3(_ShiftInvariant):
    """Shift-invariant PLCA along three axes (reference: plca.py:540-625).
    V (B, C, L, M, O), W (C, R, k0, k1, k2), H (B, R, L - k0 + 1, M - k1 + 1, O - k2 + 1), Z (R,)."""

    def __init__(self, Vshape=None, rank=None, kernel_size=1, **kwargs):
        if isinstance(Vshape, _Iterable):
            kernel_size = _triple(kernel_size)
            k0, k1, k2 = kernel_size
            batch, channel, N, K, M = Vshape
            rank = rank if rank else K
            kwargs["W"] = (channel, rank) + kernel_size
            kwargs["H"] = (batch, rank, N - k0 + 1, K - k1 + 1, M - k2 + 1)
        super().__init__(rank, **kwargs)

    @staticmethod
    def reconstruct(H, W, Z):
        return _flip_conv(F.conv3d, H, W, Z)
