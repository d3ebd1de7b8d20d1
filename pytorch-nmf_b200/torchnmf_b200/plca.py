"""PLCA / SIPLCA / SIPLCA2 / SIPLCA3 with the reference's module surface (torchnmf/plca.py:28-625) and an H100-native `fit`.

    V (N, C) / sum(V)  ~=  H (N, R) diag(Z (R,)) W (C, R)^T,     W, H column-normalised, Z a distribution.

The reference's EM iteration (plca.py:247-289) materialises WZH, takes ONE backward pass of V / (WZH + eps) through it and
updates Z, W and H simultaneously from the three gradients.  Here the two big contractions

    dW[c, r] = sum_n P[n, c] (H Z)[n, r],      dHz[n, r] = sum_c P[n, c] W[c, r],      P = V / ((H Z) W^T + eps)

are two launches of the fused wgmma KL contraction (`nmfb200_raw_terms` with the factor pair (W, H diag Z)): neither
WZH nor P reaches HBM.  dH = dHz * Z and dZ[r] = sum_n H[n, r] dHz[n, r] follow from them; everything after that is the
reference's sequence of small factor-sized operations (plca.py:256-289).

The shift-invariant models (plca.py:376-625) are the same EM step around the convolutive reconstruction
`sum_{r,t} W[c,r,t] Z[r] H[b,r,x-t]`: the factor pair handed to the library is (W, H Z) as well, and the two gradients are
the sliding contractions of `nmfb200_raw_terms` (wgrad and dgrad of the ratio tile; csrc/nmfd.cu, csrc/tc_nmfd.cu).
"""
from collections.abc import Iterable as _Iterable

import torch
import torch.nn.functional as F
from torch import Tensor
from torch.nn import Parameter

from .constants import eps
from . import engine as _engine
from .nmf import (_batched_conv, _check_lengths, _checked_fixed_w, _fit_problems, _fit_single, _placed_factors,
                  _register_batched_factors)

from torch.nn.modules.utils import _single, _pair, _triple

__all__ = ["PLCA", "SIPLCA", "SIPLCA2", "SIPLCA3", "BaseComponent", "BatchedPLCA", "BatchedSIPLCA", "BatchedSIPLCA2",
           "BatchedSIPLCA3"]


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
    def fit(self, V, tol=1e-4, max_iter=200, verbose=False, W_alpha=1., H_alpha=1., Z_alpha=1., *, precision="f32",
            mask=None, group=None, fixed_W=None):
        """EM fit of the PLCA model (reference: plca.py:193-304; same arguments, stop rule and return value
        `(n_iter, norm)`).  Runs on the parameters' CUDA device; host-resident modules are staged like `NMF.fit`.

        precision: "f32" (default: the fused fp32 CUDA-core contraction, matches the reference to 1e-5 on the fixtures) |
                   "f16" / "f16_split" (wgmma contraction: ~10x faster at large shapes; the EM recursion keeps the
                   fp16 operand rounding, measured 1.0-1.4e-3 relative after 30-50 iterations on the fixtures of
                   tests/golden/reference_next.npz -- outside the 1e-3 bar, hence opt-in).  SIPLCA2 / SIPLCA3 at "f16"
                   run the tensor-core sliding GEMMs of NMFD with the outer axes (rank <= 256).
        mask:      (keyword-only, default None) a dense torch.bool tensor of V's shape, True where V is observed: the fit
                   maximises the observed-data log-likelihood sum_O Vn log(q / q_O) (plus the Dirichlet priors), with O the
                   observed cells, q the model (summing to 1), q_O = sum_O q and Vn = V / sum_O V, by EM over the missing
                   cells (Smaragdis, Raj and Shashanka's missing-data PLCA): every iteration is the reference's EM step on
                   the completed target q_O Vn on O and q off O.  Zeroing the missing cells instead would fit them as
                   observed zeros.  V is never read off O (NaN there is fine).  The loss and stop rule are the reference's
                   on O, with the model rescaled to the observed mass: sqrt(2 kl_div(x[O], V[O])), x = q sum_O V / q_O.
                   Returns `(n_iter, norm)` with norm = sum_O V / q_O at the final factors, so `model(norm=norm)`
                   reconstructs V at its own scale and `model(norm=norm)[~mask]` is the imputation.  fp32 kernels only
                   (precision "f32"); a dense V; rank <= 256 for the shift-invariant models.  ValueError for a mask that is
                   not a dense torch.bool tensor of V's shape, a sparse V, another precision, no observed cell or
                   sum_O V = 0.

        A sparse V (PLCA only; PLSA on a count matrix): a sparse COO tensor (N, C) of any floating dtype, on the host or
        the device, coalesced or not (duplicates sum, as in `coalesce()`), is fitted as `V.to_dense()` is -- same EM step,
        priors, frozen factors, stop rule and `(n_iter, norm)`, norm = V.sum() in V's dtype -- without forming anything
        of size N x C, at every rank: each EM step takes one ratio Vn / (q + eps) per stored entry in one gather over the
        rows, which also yields H's gradient, and one gather over the columns reuses it for W's; the loss takes the stored
        entries' terms from a gather over the rows and the model's mass from the factors' column sums.  The device holds
        O(nnz + (N + C) R).  fp32 kernels only (`last_fit_precision` "f32"); the summation order differs from the dense
        fit's, so the two agree to fp32 rounding, not bit for bit.  AssertionError for a negative stored value; ValueError
        for a target storing nothing or summing to 0, a sparse layout other than COO, precision "f16" / "f16_split" or an
        unknown precision, and a mask.  SIPLCA, SIPLCA2 and SIPLCA3 raise NotImplementedError for a sparse V.

        group:     (keyword-only, default None) a torch.distributed process group: a sharded fit, for a corpus or a set of
                   recordings that does not fit one GPU.  PLCA shards the rows: each rank passes its rows V[n_g, :] (dense or
                   sparse COO) and its module holds H[n_g, :]; SIPLCA / SIPLCA2 / SIPLCA3 shard the batch axis: V[b_g] and
                   H[b_g].  W and Z are replicated and must be identical on every rank at entry; an H_alpha tensor is this
                   rank's shard.  Shards may be uneven, but every size past the shard axis -- C, R and for the
                   shift-invariant models the kernel size and V's sizes past C -- must agree across ranks.  Each EM step
                   runs this rank's contractions on its own shard (the same kernels as the unsharded fit, at the same
                   precision) and sums W's and Z's gradients over the ranks in one all-reduce of C R prod(K) + R floats;
                   the Z and W updates then compute the same bits on every rank, so the replicas stay identical.  H's
                   update is local, apart from one R-float all-reduce of H's column sums where the update divides by
                   them (W and Z both frozen, or H_alpha != 1).  The loss is every shard's divergence summed in float64
                   by one scalar all-reduce every 10th iteration, so every rank takes the same stop decision.  Returns
                   `(n_iter, norm)` on every rank, norm = the sum of every shard's V.sum(), in V's dtype, by which each
                   rank normalises its shard.  A one-rank group gives the unsharded fit bit for bit.  V and H data never
                   move between ranks.  The checks that can fail on one rank only -- a shard that does not match the
                   module's H / W, a negative value (AssertionError), an empty shard (no row or clip; a sparse one storing no
                   entry) -- and the sizes
                   are agreed by every rank before any raises, so they raise on every rank together; so does a sparse
                   target whose shards all sum to 0.  ValueError for `mask` with `group`.  Not covered: masked fits,
                   the batched classes (which take no `group`), a peer-memory (NVLink) exchange, and (NMF) sharded
                   sparse targets without densifying.

        fixed_W:   (keyword-only, default None) a torch.bool tensor of R elements, on any device: the components k where it
                   is True keep W[:, k] (W[:, k, ...] for the shift-invariant models) at its value, for semi-supervised
                   separation (Smaragdis, Raj and Shashanka 2007): a dictionary learned for a known source stays fixed while
                   the free components learn the rest of the target.  Each EM step applies W's update -- the
                   multiplicative step, its normalisation and W_alpha's prior -- to the free components only, with the
                   same bits as without `fixed_W`; H and Z are learned for every component, Z from the gradient over all of
                   them.  Every component fixed is the fit of trainable_W=False; none fixed is the plain fit.  Dense,
                   sparse and masked targets alike.  ValueError, before any device work: a `fixed_W` that is not a dense
                   torch.bool tensor of shape (R,), a W that is not trainable, and `group`.
        """
        fixed_W = _checked_fixed_w(self.W, fixed_W, group)
        if mask is not None:
            if group is not None:
                raise ValueError(f"group: {type(self).__name__}.fit does not run masked fits sharded (mask with group)")
            return self._fit_masked(V, mask, tol, max_iter, verbose, W_alpha, H_alpha, Z_alpha, precision, fixed_W)
        if V.layout != torch.strided:
            return self._fit_sparse(V, tol, max_iter, verbose, W_alpha, H_alpha, Z_alpha, precision, group, fixed_W)
        if group is None:
            assert torch.all(V >= 0.), "Target should be non-negative."                     # plca.py:236
        W, H, Z = self.W, self.H, self.Z
        assert W is not None and H is not None and Z is not None, "fit() needs W, H and Z"
        no_cuda = "torchnmf_b200.PLCA.fit needs a CUDA device (sm_90a); there is no CPU fallback"
        with _placed_factors(self, (W, H, Z), no_cuda) as (dev, (Wd, Hd, Zd)):
            f32 = torch.float32
            norm = V.sum()
            ops = None
            if group is not None:
                ops = _engine.Collectives(group, dev)
                norm = self._agree_on_shards(ops, V, self._shape_mismatch(V), bool(torch.all(V >= 0.)), V.numel() > 0, norm)
            Vn = (V.to(dev, f32).contiguous() / norm.to(dev, f32)).contiguous()              # plca.py:241-242
            normd = norm.to(dev, f32)
            Vfull = Vn * normd

            def divergence(follows):
                return _total(ops, _kl(self.reconstruct(Hd, Wd, Zd) * normd, Vfull))      # plca.py:245-246,293-294

            Hz = (Hd * _over(Zd, Hd)).contiguous()        # the engine's activation factor: H diag(Z)
            buf = _terms_buffer(ops, Wd)
            wfix = _w_fixing(self.W, fixed_W, dev)
            eng = self._engine(Vn, Wd, Hz, precision) if self._engine_factory is None else self._engine_factory(Vn, Wd, Hz)
            try:
                def step(k):
                    for _ in range(k):
                        torch.mul(Hd, _over(Zd, Hd), out=Hz)
                        eng.sync()
                        dW, _ = eng.raw_terms(0, 1.0)     # P contracted with H Z  = W.grad   (plca.py:252-253)
                        dHz, _ = eng.raw_terms(1, 1.0)    # P contracted with W;  H.grad = dHz * Z,  Z.grad = sum H dHz
                        dW, dZ = _em_terms(ops, Hd, dW, dHz, buf)
                        self._em_update(Wd, Hd, Zd, dW, dHz, dZ, W_alpha, H_alpha, Z_alpha, ops, *wfix)

                n_iter = _fit_single(step, divergence, max_iter, tol, verbose)
                eng.check_health()
                self.last_fit_precision = eng.precision_for(1.0)
            finally:
                eng.close()
        return n_iter, norm                                                                  # plca.py:304

    def _target_shape(self):
        """The target's shape the factors model: (N, C) for PLCA, (B, C, *(J + K - 1)) for the shift-invariant models."""
        H, W = self.H, self.W
        return (H.shape[0], W.shape[0]) + tuple(j + k - 1 for j, k in zip(H.shape[2:], W.shape[2:]))

    def _shape_mismatch(self, V):
        """None when V has the shape the factors model, else the message of the mismatch."""
        if tuple(V.shape) == self._target_shape():
            return None
        return f"target shape {tuple(V.shape)} does not match H {tuple(self.H.shape)} / W {tuple(self.W.shape)}"

    def _agree_on_shards(self, ops, V, mismatch, nonneg, stored, norm):
        """A sharded fit's entry over the Collectives `ops`: this rank's checks -- `mismatch` (None or the message of a
        shard that does not match H / W), `nonneg` (no negative value) and `stored` (the shard holds a row or clip; a
        sparse one stores an entry) --
        agreed by every rank before any raises, so that no rank waits in a collective the others never reach; then the
        sizes past the shard axis, equal on every rank.  Returns the global norm, the sum of every shard's `norm`
        (float64 across ranks), in norm's dtype and on its device."""
        if not ops.all_ranks(mismatch is None):
            raise ValueError(mismatch or "sharded fit: the target shard of another rank does not match its H / W")
        nonneg = ops.all_ranks(nonneg)
        assert nonneg, "Target should be non-negative."                                     # plca.py:236, on any rank
        if not ops.all_ranks(stored):
            if stored:
                raise ValueError("sharded fit: the target shard of another rank is empty")
            raise ValueError("the sparse target stores no entry" if V.is_sparse
                             else f"sharded fit: this rank's target shard {tuple(V.shape)} is empty")
        K, X = tuple(self.W.shape[2:]), tuple(V.shape[2:])
        ops.check_same_sizes(["C", "R"] + [f"kernel_size[{i}]" for i in range(len(K))]
                             + [f"V.shape[{i + 2}]" for i in range(len(X))], [*self.W.shape[:2], *K, *X])
        total = ops.all_reduce_(norm.to(ops.device, torch.float64).reshape(1))
        return total[0].to(norm.device, norm.dtype)

    def _em_update(self, Wd, Hd, Zd, dW, dHz, dZ, W_alpha, H_alpha, Z_alpha, ops=None, train_w=None, fixed=None):
        """The Z, W and H updates of one EM step (plca.py:256-288) from the raw gradients dW, dHz (= H.grad / Z) and
        dZ (= Z.grad, `_em_terms`), in place on the working copies, each taken only where the module's factor is
        trainable (`train_w`, when given, in place of W's flag).  With `ops` (a sharded fit's Collectives: dW and dZ
        already summed over the ranks) the two divisions by H's column sums take them over every rank's rows, one R-float
        all-reduce each.  `fixed` (the indices of W's fixed components, on its device): those components keep their
        values; every step of W's update acts on each component alone, so the free ones take the bits they take without
        it, and the column masses H divides by with Z frozen are those of the whole step, as W's gradient gives them."""
        if train_w is None:
            train_w = self.W.requires_grad
        h_norm = get_norm if ops is None else (lambda x: ops.all_reduce_(get_norm(x)))
        dH = dHz * _over(Zd, Hd)
        Z_prior = None
        if self.Z.requires_grad:                                                             # plca.py:256-262
            Zd.mul_(dZ.clamp_min(0))
            Z_prior = Zd.clone()
            if not _is_one(Z_alpha):
                Zd.add_(_as(Z_alpha, Zd) - 1)
                F.threshold(Zd, eps, eps, True)
            Zd.div_(Zd.sum())
        if train_w:                                                                          # plca.py:264-275
            kept = Wd.index_select(1, fixed) if fixed is not None else None
            Wd.mul_(dW.clamp_min(0))
            if Z_prior is None:
                W_div = get_norm(Wd)
                Z_prior = W_div.squeeze()
            else:
                W_div = _over(Z_prior, Wd)
            Wd.div_(W_div)
            if not _is_one(W_alpha):
                Wd.add_(_as(W_alpha, Wd) - 1)
                F.threshold(Wd, eps, eps, True)
                Wd.div_(get_norm(Wd))
            if fixed is not None:
                Wd.index_copy_(1, fixed, kept)
        if self.H.requires_grad:                                                             # plca.py:277-288
            Hd.mul_(dH.clamp_min(0))
            H_div = h_norm(Hd) if Z_prior is None else _over(Z_prior, Hd)
            Hd.div_(H_div)
            if not _is_one(H_alpha):
                Hd.add_(_as(H_alpha, Hd) - 1)
                F.threshold(Hd, eps, eps, True)
                Hd.div_(h_norm(Hd))

    def _check_mask(self, V, mask, precision):
        """The masked fit's refusals, before any device work: (the mask on V's device, sum_O V in V's dtype)."""
        if not isinstance(mask, Tensor) or mask.dtype != torch.bool:
            raise ValueError(f"mask must be a torch.bool tensor (got {getattr(mask, 'dtype', type(mask))})")
        if mask.is_sparse:
            raise ValueError(f"mask: {type(self).__name__}.fit takes a dense mask only")
        if tuple(mask.shape) != tuple(V.shape):
            raise ValueError(f"mask shape {tuple(mask.shape)} does not match the target's {tuple(V.shape)}")
        if V.is_sparse:
            raise ValueError("mask: a masked fit needs a dense target")
        if precision != "f32":
            raise ValueError(f"mask: masked fits run on the fp32 kernels; precision must be 'f32' (got {precision!r})")
        M = mask.to(V.device)
        assert bool(torch.where(M, V >= 0., True).all()), "Target should be non-negative."   # plca.py:236, on O only
        if not bool(M.any()):
            raise ValueError("mask: no cell of the target is observed")
        norm_o = torch.where(M, V, torch.zeros((), dtype=V.dtype, device=V.device)).sum()
        if not bool(norm_o > 0):
            raise ValueError("mask: the observed cells of the target sum to 0")
        return M, norm_o

    def _fit_masked(self, V, mask, tol, max_iter, verbose, W_alpha, H_alpha, Z_alpha, precision, fixed_W=None):
        """fit(V, ..., mask=mask): EM with the missing cells latent (see fit)."""
        M, norm_o = self._check_mask(V, mask, precision)
        W, H, Z = self.W, self.H, self.Z
        assert W is not None and H is not None and Z is not None, "fit() needs W, H and Z"
        no_cuda = f"torchnmf_b200.{type(self).__name__}.fit needs a CUDA device (sm_90a); there is no CPU fallback"
        with _placed_factors(self, (W, H, Z), no_cuda) as (dev, (Wd, Hd, Zd)):
            f32 = torch.float32
            Md = M.to(dev).contiguous()
            normd = norm_o.to(dev, f32)
            # Vn on O and 0 off O: the kernels never meet what V holds at the missing cells
            Vn = (torch.where(Md, V.to(dev, f32), torch.zeros((), dtype=f32, device=dev)) / normd).contiguous()
            Vobs = Vn * normd

            def divergence(follows):
                # kl_div(x[O], V[O]) with the model scaled to the observed mass, x = q sum_O V / q_O; Vobs is 0 off O
                q = self.reconstruct(Hd, Wd, Zd)
                x = q * (normd / torch.where(Md, q, 0.).sum())
                return float(Vobs.reshape(-1) @ (torch.log(Vobs + eps) - torch.log(x + eps)).reshape(-1) - Vobs.sum()
                             + torch.where(Md, x, 0.).sum())

            Hz = (Hd * _over(Zd, Hd)).contiguous()
            qobs = torch.zeros(1, dtype=torch.float64, device=dev)
            wfix = _w_fixing(self.W, fixed_W, dev)
            eng = self._engine(Vn, Wd, Hz, precision) if self._engine_factory is None else self._engine_factory(Vn, Wd, Hz)
            try:
                eng.set_mask(Md)

                def step(k):
                    # the reference's EM step on the completed target q_O Vn (O) / q (off O): its gradients are q_O A + B
                    for _ in range(k):
                        torch.mul(Hd, _over(Zd, Hd), out=Hz)
                        eng.sync()
                        aW, bW = eng.plca_masked_terms(0, qobs)
                        aH, bH = eng.plca_masked_terms(1)
                        q = qobs.to(f32)
                        dHz = torch.addcmul(bH, aH, q)
                        dW, dZ = _em_terms(None, Hd, torch.addcmul(bW, aW, q), dHz)
                        self._em_update(Wd, Hd, Zd, dW, dHz, dZ, W_alpha, H_alpha, Z_alpha, None, *wfix)

                n_iter = _fit_single(step, divergence, max_iter, tol, verbose)
                eng.check_health()
                self.last_fit_precision = "f32"
            finally:
                eng.close()
            # the returned norm's q_O in float64 (the fp32 reconstruction may run on TF32 convolutions)
            q = self.reconstruct(Hd.double(), Wd.double(), Zd.double())
            qo = torch.where(Md, q, 0.).sum()
        return n_iter, (norm_o.double() / qo.to(norm_o.device)).to(norm_o.dtype)

    def _fit_sparse(self, V, tol, max_iter, verbose, W_alpha, H_alpha, Z_alpha, precision, group, fixed_W=None):
        raise NotImplementedError(f"{type(self).__name__}.fit takes dense targets only (PLCA fits sparse COO targets)")

    # test hook, as the NMF modules' (tests/test_plca.py): factory(Vn, W, Hz) stands in for `_engine`
    _engine_factory = None

    @staticmethod
    def _engine(Vn, W, Hz, precision):
        raise NotImplementedError


def _w_fixing(W, fixed_W, dev):
    """`_em_update`'s (train_w, fixed) for a fit's checked `fixed_W` (`_checked_fixed_w`): W's own flag and no fixed
    component; False when every component is fixed (the fit of trainable_W=False); else the indices of the fixed components
    on the device `dev`, found once per fit (indexing by the flags would synchronise with the host at every step)."""
    if fixed_W is None:
        return W.requires_grad, None
    if bool(fixed_W.all()):
        return False, None
    return True, fixed_W.nonzero().reshape(-1).to(dev)


def _over(z, x):
    """A rank vector against the rank dimension (1) of a factor (plca.py:269-270,282-283)."""
    return z[(slice(None),) + (None,) * (x.dim() - 2)]


def _terms_buffer(ops, Wd):
    """A sharded fit's flat [dW | dZ] buffer, W's size + R elements, allocated once per fit (None without `ops`)."""
    return None if ops is None else torch.empty(Wd.numel() + Wd.shape[1], dtype=Wd.dtype, device=Wd.device)


def _em_terms(ops, Hd, dW, dHz, buf=None):
    """(dW, dZ) of one EM step: Z's gradient dZ = sum H dHz beside W's dW; with `ops` (a sharded fit's Collectives) both
    copied into `buf` (`_terms_buffer`) and summed over the ranks in one all-reduce of it, returned as views of it."""
    dZ = get_norm(Hd * dHz).reshape(-1)
    if ops is None:
        return dW, dZ
    n = dW.numel()
    buf[:n].view(dW.shape).copy_(dW)
    buf[n:].copy_(dZ)
    ops.all_reduce_(buf)
    return buf[:n].view(dW.shape), buf[n:]


def _total(ops, d):
    """A divergence as a float: as it is without `ops`, else every rank's summed in float64 (one scalar all-reduce)."""
    if ops is None:
        return float(d)
    return float(ops.all_reduce_(torch.as_tensor(d, dtype=torch.float64).reshape(1).to(ops.device)))


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

    def _fit_sparse(self, V, tol, max_iter, verbose, W_alpha, H_alpha, Z_alpha, precision, group, fixed_W=None):
        """fit(V) for a sparse COO V: the EM fit of V.to_dense() without forming anything of size N x C (see `fit`)."""
        if V.layout != torch.sparse_coo:
            raise ValueError(f"PLCA.fit takes a dense or a sparse COO target (got layout {V.layout})")
        if precision != "f32":
            if precision in ("f16", "f16_split"):
                raise ValueError(f"a sparse target runs on the fp32 kernels: precision must be 'f32' (got {precision!r})")
            raise ValueError(f"unknown precision {precision!r}")
        W, H, Z = self.W, self.H, self.Z
        assert W is not None and H is not None and Z is not None, "fit() needs W, H and Z"
        mismatch = self._shape_mismatch(V)
        if mismatch is not None and group is None:
            raise ValueError(mismatch)
        Vc = V.coalesce()                                   # duplicates sum, as in V.to_dense()
        vals = Vc.values()
        nonneg = bool((vals >= 0.).all())
        if group is None:
            assert nonneg, "Target should be non-negative."                                 # plca.py:236
            if vals.numel() == 0:
                raise ValueError("the sparse target stores no entry")
        norm = vals.sum()                                                                    # V.sum(), in V's dtype
        if group is None and not bool(norm > 0):
            raise ValueError("the sparse target's values sum to 0")
        no_cuda = "torchnmf_b200.PLCA.fit needs a CUDA device (sm_90a); there is no CPU fallback"
        with _placed_factors(self, (W, H, Z), no_cuda) as (dev, (Wd, Hd, Zd)):
            ops = None
            if group is not None:
                ops = _engine.Collectives(group, dev)
                norm = self._agree_on_shards(ops, V, mismatch, nonneg, vals.numel() > 0, norm)
                if not bool(norm > 0):                      # the same global norm on every rank
                    raise ValueError("the sparse target's values sum to 0")
            ft = Wd.dtype                                   # fp32 on the device; the test hook's factors as they are
            normd = norm.to(dev, ft)
            Vn = torch.sparse_coo_tensor(Vc.indices().to(dev), vals.to(dev, ft) / normd, V.shape,
                                         is_coalesced=True)                                 # plca.py:241-242
            normf = float(normd)
            Hz = (Hd * _over(Zd, Hd)).contiguous()
            buf = _terms_buffer(ops, Wd)
            wfix = _w_fixing(self.W, fixed_W, dev)
            eng = _engine.CudaSparsePlcaEngine(Vn, Wd, Hz) if self._engine_factory is None else self._engine_factory(Vn, Wd, Hz)
            try:
                def divergence(follows):
                    torch.mul(Hd, _over(Zd, Hd), out=Hz)
                    return _total(ops, eng.loss(normf))     # kl_div(norm q, V) at the stored entries and the column sums

                def step(k):
                    for _ in range(k):
                        torch.mul(Hd, _over(Zd, Hd), out=Hz)
                        dW, dHz = eng.plca_terms(Hz)        # one ratio P per stored entry serves both gradients
                        dW, dZ = _em_terms(ops, Hd, dW, dHz, buf)
                        self._em_update(Wd, Hd, Zd, dW, dHz, dZ, W_alpha, H_alpha, Z_alpha, ops, *wfix)

                n_iter = _fit_single(step, divergence, max_iter, tol, verbose)
                eng.check_health()
                self.last_fit_precision = eng.precision_for(1.0)
            finally:
                eng.close()
        return n_iter, norm


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


# ---- many independent problems in one fit ---------------------------------------------------------------------------------

@torch.no_grad()
def _batched_norm(x):
    """get_norm of every problem of a batched factor (problems on axis 0, rank on axis 2), kept for broadcasting."""
    return x.sum([d for d in range(x.dim()) if d not in (0, 2)], keepdim=True)


def _alpha_buffer(alpha, like):
    """None for the scalar 1 (no prior), else alpha as one contiguous fp32 buffer of the batched factor's shape: a scalar, or
    a tensor that broadcasts to it (a single problem's alpha applies to every problem)."""
    if _is_one(alpha):
        return None
    a = torch.as_tensor(alpha).to(like.device, torch.float32)
    try:
        return torch.broadcast_to(a, like.shape).contiguous()
    except RuntimeError:
        raise ValueError(f"alpha of shape {tuple(a.shape)} does not broadcast to the factor's {tuple(like.shape)}") from None


class _BatchedPLCABase(BaseComponent):
    """Shared part of the batched PLCA classes: P independent problems of one model and one shape, fitted together.  W and H
    hold the problems on axis 0 and the rank on axis 2, Z is (P, R); problem p's W[p], H[p], Z[p] are those of the single
    model.  `fit` runs every problem's EM iteration on the fp32 CUDA-core kernels in the launches one problem takes, each
    with its own stop rule."""
    _ndim = 3
    _axes = "three axes (P, rows, rank)"
    _engine_cls = None
    _ragged = False                # fit(..., lengths=L): BatchedPLCA only

    def __init__(self, rank=None, W=None, H=None, Z=None, trainable_W=True, trainable_H=True, trainable_Z=True):
        torch.nn.Module.__init__(self)
        inferred, P = _register_batched_factors(self, W, H, trainable_W, trainable_H)
        for p in (self.W, self.H):
            if p is not None:
                p.data.div_(_batched_norm(p))
        if isinstance(Z, Tensor):
            if Z.dim() != 2:
                raise ValueError(f"Z must have two axes (P, rank); got shape {tuple(Z.shape)}")
            assert torch.all(Z >= 0.), "Tensor Z should be non-negative."
            z = Parameter(torch.empty(*Z.size()), requires_grad=trainable_Z)
            z.data.copy_(Z)
        elif P is not None and (inferred or rank):
            R = inferred or rank
            z = Parameter(torch.ones(P, R) / R)
        else:
            z = None
        self.register_parameter("Z", z)
        if z is not None:
            z.data.div_(z.data.sum(1, keepdim=True))
            if inferred is not None and z.shape[1] != inferred:
                raise ValueError("Latent size of Z does not match with others!")
            if P is not None and z.shape[0] != P:
                raise ValueError(f"Z holds {z.shape[0]} problems, W / H {P}")
            inferred = z.shape[1]
        if inferred is None:
            assert rank, "A rank should be given when W, H and Z are not available!"
        else:
            rank = inferred
        self.rank = rank

    def forward(self, H=None, W=None, Z=None, norm=None):
        """Every problem's reconstruction (P, *V's single shape), problem p scaled by norm[p] when `norm` is given."""
        H = self.H if H is None else H
        W = self.W if W is None else W
        Z = self.Z if Z is None else Z
        out = self.reconstruct(H, W, Z)
        return out if norm is None else out * torch.as_tensor(norm).reshape(-1, *([1] * (out.dim() - 1)))

    def _single_shape(self):
        raise NotImplementedError

    def _check_target_shape(self, V):
        """Whether V is one target shared by every problem (else it is stacked); ValueError if it is neither."""
        P = self.W.shape[0]
        single = self._single_shape()
        if tuple(V.shape) not in ((P,) + single, single):
            raise ValueError(f"target shape {tuple(V.shape)} does not match H {tuple(self.H.shape)} / W {tuple(self.W.shape)}: "
                             f"expected {(P,) + single} or {single}")
        return tuple(V.shape) == single

    def _length_range(self, V):
        """(lo, hi, name of hi) of the lengths of a ragged fit: rows of H in [1, N]."""
        return 1, self.H.shape[1], "N"

    @torch.no_grad()
    def fit(self, V, tol=1e-4, max_iter=200, verbose=False, W_alpha=1., H_alpha=1., Z_alpha=1., *, precision="f32",
            lengths=None):
        """Fit every problem by EM, as the single model's `fit(V[p], ...)` fits one, all of them in the same launches.

        V: the problems' targets stacked on a leading axis, or one target of the single model's shape shared by every
        problem (random restarts of one fit), of any floating dtype.  Each problem's target is normalised by its sum into
        one fp32 copy (a shared target once, read by every problem).  A sparse V raises NotImplementedError.

        Returns `(n_iter, norm)`: n_iter a torch.int64 tensor of P values, each what the single `fit` returns for that
        problem -- the loop index at its stop, or max_iter - 1 -- and norm the P sums V[p].sum() in V's dtype.  Problem p
        follows the reference's stop rule (plca.py:245-302) on its own: its loss sqrt(2 kl_div(norm_p X_p, V_p)) at the start
        and every 10th iteration, and it stops at the first check where (previous_p - loss_p) / init_p < tol; from then on
        every launch leaves its W, H and Z untouched while the others run on.  Each problem's EM step sums in an order fixed
        by its shape, so problem p's results do not depend on the other problems or on P.  The losses cost one
        synchronisation per 10 iterations for the whole batch.

        W_alpha / H_alpha / Z_alpha: the Dirichlet priors, each a scalar or a tensor broadcasting to the batched factor's
        shape (a single problem's alpha applies to every problem).  Frozen factors (trainable_W / _H / _Z) take the
        reference's branches.  precision: "f32" only ("f16" / "f16_split" and unknown strings raise ValueError), and so does
        a rank above 256 or a shape mismatch; `last_fit_precision` is "f32".  `mask`, `weight` and `group` are not
        parameters of this method (TypeError).  Host-resident and half or double modules are staged through fp32 device
        copies and written back.

        lengths: (keyword-only, default None; BatchedPLCA only) P ints in [1, N], as a sequence or an integer tensor of shape
        (P,) on any device: a ragged batch.  V (P, N, C) and H (P, N, R) stay padded, and problem p is the EM fit of
        V[p, :L_p] with W[p], H[p, :L_p] and Z[p]: n_iter[p], norm[p] = V[p, :L_p].sum(), W[p], H[p, :L_p] and Z[p] equal, bit
        for bit, those of this class's fit with P = 1 on V[p:p+1, :L_p] from W[p:p+1], H[p:p+1, :L_p] and Z[p:p+1], stop rule
        included: each problem runs the plan and summation order of its own row count.  The padding rows of V are never read
        by the fit (NaN there does not reach it), those of H are neither read nor written, even through a staged host, half
        or float64 module, the padding of an H_alpha tensor is ignored, and the non-negativity assertion looks at the real
        rows only.  The fit does not renormalise H: the constructor normalises H over all N rows, so pad H with zeros, or
        set the factors after construction, for each problem to start from its own normalised H[p, :L_p].  forward()[p, :L_p]
        is problem p's model (the rows of a PLCA model are independent).  Every alpha form, frozen factors and target dtype
        work as without lengths, and lengths all equal to N give the bits of lengths=None.  ValueError, before any device
        work: the wrong number of lengths, a length out of range, non-integer, bool or non-1-D lengths, a shared target, and
        lengths on BatchedSIPLCA / BatchedSIPLCA2 / BatchedSIPLCA3.
        """
        name = type(self).__name__
        if lengths is not None:
            assert self.W is not None and self.H is not None and self.Z is not None, "fit() needs W, H and Z"
            lengths = _check_lengths(self, V, lengths)
        if precision != "f32":
            if precision in ("f16", "f16_split"):
                raise ValueError(f"{name} runs on the fp32 kernels: precision must be 'f32' (got {precision!r})")
            raise ValueError(f"unknown precision {precision!r}")
        if V.is_sparse:
            raise NotImplementedError(f"{name} takes dense targets only")
        W, H, Z = self.W, self.H, self.Z
        assert W is not None and H is not None and Z is not None, "fit() needs W, H and Z"
        P, R = W.shape[0], W.shape[2]
        if R > 256:
            raise ValueError(f"{name} supports rank <= 256 (got {R})")
        shared = self._check_target_shape(V)
        real = None                # a ragged batch: the real rows of V and H, (P, N)
        if lengths is None:
            assert torch.all(V >= 0.), "Target should be non-negative."                     # plca.py:236
        else:
            real = torch.arange(H.shape[1]) < torch.tensor(lengths).unsqueeze(1)
            assert bool(torch.where(real.to(V.device).unsqueeze(2), V >= 0., True).all()), "Target should be non-negative."
        f32 = torch.float32
        no_cuda = f"torchnmf_b200.{name}.fit needs a CUDA device (sm_90a); there is no CPU fallback"
        with _placed_factors(self, (W, H, Z), no_cuda, real) as (dev, (Wd, Hd, Zd)):
            # every problem's norm as the single fit takes it (V[p].sum(), a ragged problem's V[p, :L_p].sum()), whatever P is
            if lengths is not None:
                norm = torch.stack([V[p, :n].sum() for p, n in enumerate(lengths)])
            else:
                norm = V.sum().reshape(1).expand(P).clone() if shared else torch.stack([V[p].sum() for p in range(P)])
            normd = norm.to(dev, f32)
            Vd = V.to(dev, f32).contiguous()
            Vn = (Vd / normd[0] if shared else Vd / normd.reshape(P, *([1] * (V.dim() - 1)))).contiguous()  # plca.py:241-242
            Hz = (Hd * Zd.reshape(P, 1, R, *([1] * (Hd.dim() - 3)))).contiguous()
            alphas = [_alpha_buffer(a, t) for a, t in ((W_alpha, Wd), (H_alpha, Hd), (Z_alpha, Zd))]
            ragged = {} if lengths is None else {"lengths": lengths}
            eng = (self._engine_cls if self._engine_factory is None else self._engine_factory)(Vn, Wd, Hz, **ragged)
            try:
                def step(k):                                                                 # plca.py:247-289, k times
                    eng.plca_iterate(k, Hd, Zd, W.requires_grad, H.requires_grad, Z.requires_grad, *alphas)

                # the single fit returns its loop index: one less than the iterations it ran (plca.py:304)
                n_iter = _fit_problems(eng, P, max_iter, tol, verbose, lambda: eng.plca_losses(normd), step) - 1
                self.last_fit_precision = "f32"
            finally:
                eng.close()
        return n_iter, norm


class BatchedPLCA(_BatchedPLCABase):
    """P independent PLCA problems of one shape:  V[p] / sum(V[p]) (N,C) ~= H[p] diag(Z[p]) W[p]^T,  W (P,C,R), H (P,N,R),
    Z (P,R).  Problem p is `PLCA(W=W[p], H=H[p], Z=Z[p])`.

    Args:
        Vshape: (P, N, C); W and H are then drawn as `PLCA` draws them, |randn| of (P, C, rank) and (P, N, rank), and every
            problem's factors normalised
        rank: size of the hidden dimension (default: C)
        W / H: a size (iterable of ints -> random non-negative init) or an initial non-negative Tensor
        Z: an initial non-negative (P, rank) Tensor (default: ones(P, rank) / rank), each row normalised
        trainable_W / trainable_H / trainable_Z: whether a *given tensor* is updated by `fit`

    `fit(V, ...)` takes V as (P, N, C), or as one (N, C) target shared by every problem.  Each problem's fit is
    `PLCA.fit(V[p], ..., precision="f32")`'s EM iteration.  Workspace (device memory, kept between fits of the same shape):
    that of `BatchedNMF` at this shape, plus per fit the raw numerators of W and H (the factors' size) and the EM step's
    scratch.  `fit(..., lengths=L)` fits a ragged batch: problem p is the EM fit of V[p, :L[p]] with W[p], H[p, :L[p]] and
    Z[p], V and H padded to N rows, each problem bit for bit its own fit with P = 1 (see `fit`); the workspace is then that
    of a ragged `BatchedNMF` with the same lengths plus the same per-fit buffers.
    """
    _engine_cls = _engine.CudaBatchedNmfEngine
    _ragged = True

    def __init__(self, Vshape=None, rank=None, *, W=None, H=None, Z=None, trainable_W=True, trainable_H=True,
                 trainable_Z=True):
        if isinstance(Vshape, _Iterable):
            P, N, C = Vshape
            rank = rank if rank else C
            W = (P, C, rank) if W is None else W
            H = (P, N, rank) if H is None else H
        super().__init__(rank, W, H, Z, trainable_W, trainable_H, trainable_Z)

    @staticmethod
    def reconstruct(H, W, Z):
        return H @ (W * Z.unsqueeze(1)).transpose(-1, -2)

    def _single_shape(self):
        return (self.H.shape[1], self.W.shape[1])


class _BatchedShiftInvariant(_BatchedPLCABase):
    """Shared part of BatchedSIPLCA / BatchedSIPLCA2 / BatchedSIPLCA3: P independent problems of the single model over `_nd`
    shifted axes, V (P,B,C,*X), W (P,C,R,*K), H (P,B,R,*(X-K+1)), Z (P,R); each problem's B clips share its W[p] and Z[p]."""
    _engine_cls = _engine.CudaBatchedNmfdEngine
    _conv = None

    @classmethod
    def reconstruct(cls, H, W, Z):
        return _batched_conv(H, W * Z.reshape(*Z.shape, *([1] * (W.dim() - 3))).unsqueeze(1), cls._conv)

    def _single_shape(self):
        B = self.H.shape[1]
        C, K, J = self.W.shape[1], self.W.shape[3:], self.H.shape[3:]
        return (B, C) + tuple(j + k - 1 for j, k in zip(J, K))


class BatchedSIPLCA(_BatchedShiftInvariant):
    """P independent SIPLCA problems of one shape: V[p] (B,C,L), W (P,C,R,T), H (P,B,R,L-T+1), Z (P,R).  Problem p is
    `SIPLCA(W=W[p], H=H[p], Z=Z[p])`; its B clips share W[p] and Z[p].

    Args:
        Vshape: (P, B, C, L); W and H are then drawn as `SIPLCA` draws them, |randn| of (P, C, rank, T) and
            (P, B, rank, L-T+1), and every problem's factors normalised
        rank: size of the hidden dimension (default: C)
        T: the kernel's length (an int or a 1-tuple)
        W / H: a size (iterable of ints -> random non-negative init) or an initial non-negative Tensor
        Z: an initial non-negative (P, rank) Tensor (default: ones(P, rank) / rank), each row normalised
        trainable_W / trainable_H / trainable_Z: whether a *given tensor* is updated by `fit`

    `fit(V, ...)` takes V as (P, B, C, L), or as one (B, C, L) target shared by every problem.  Workspace (device memory,
    kept between fits of the same shape): that of `BatchedNMFD` at this shape, plus per fit the raw numerators of W and H
    and the EM step's scratch.
    """
    _ndim = 4
    _axes = "four axes (P, rows, rank, T)"
    _conv = staticmethod(F.conv1d)

    def __init__(self, Vshape=None, rank=None, T=1, *, W=None, H=None, Z=None, trainable_W=True, trainable_H=True,
                 trainable_Z=True):
        if isinstance(Vshape, _Iterable):
            T, = _single(T)
            P, B, C, L = Vshape
            rank = rank if rank else C
            W = (P, C, rank, T) if W is None else W
            H = (P, B, rank, L - T + 1) if H is None else H
        super().__init__(rank, W, H, Z, trainable_W, trainable_H, trainable_Z)


class BatchedSIPLCA2(_BatchedShiftInvariant):
    """P independent SIPLCA2 problems of one shape: V[p] (B,C,X1,X2), W (P,C,R,k1,k2), H (P,B,R,X1-k1+1,X2-k2+1), Z (P,R).
    Problem p is `SIPLCA2(W=W[p], H=H[p], Z=Z[p])`; its B clips share W[p] and Z[p].

    Args:
        Vshape: (P, B, C, X1, X2); W and H are then drawn as `SIPLCA2` draws them (rank defaults to X1, as there)
        rank: size of the hidden dimension
        kernel_size: (k1, k2), or one int for both
        W / H: a size (iterable of ints -> random non-negative init) or an initial non-negative Tensor
        Z: an initial non-negative (P, rank) Tensor (default: ones(P, rank) / rank), each row normalised
        trainable_W / trainable_H / trainable_Z: whether a *given tensor* is updated by `fit`

    `fit(V, ...)` takes V as (P, B, C, X1, X2), or as one (B, C, X1, X2) target shared by every problem.  Workspace: that of
    `BatchedNMF2D` at this shape, plus per fit the raw numerators of W and H and the EM step's scratch.
    """
    _ndim = 5
    _axes = "five axes (P, rows, rank, k1, k2)"
    _conv = staticmethod(F.conv2d)

    def __init__(self, Vshape=None, rank=None, kernel_size=1, *, W=None, H=None, Z=None, trainable_W=True,
                 trainable_H=True, trainable_Z=True):
        if isinstance(Vshape, _Iterable):
            kernel_size = _pair(kernel_size)
            k1, k2 = kernel_size
            P, B, C, X1, X2 = Vshape
            rank = rank if rank else X1
            W = (P, C, rank) + tuple(kernel_size) if W is None else W
            H = (P, B, rank, X1 - k1 + 1, X2 - k2 + 1) if H is None else H
        super().__init__(rank, W, H, Z, trainable_W, trainable_H, trainable_Z)


class BatchedSIPLCA3(_BatchedShiftInvariant):
    """P independent SIPLCA3 problems of one shape: V[p] (B,C,X1,X2,X3), W (P,C,R,k1,k2,k3),
    H (P,B,R,X1-k1+1,X2-k2+1,X3-k3+1), Z (P,R).  Problem p is `SIPLCA3(W=W[p], H=H[p], Z=Z[p])`; its B clips share W[p]
    and Z[p].

    Args:
        Vshape: (P, B, C, X1, X2, X3); W and H are then drawn as `SIPLCA3` draws them (rank defaults to X2, as there)
        rank: size of the hidden dimension
        kernel_size: (k1, k2, k3), or one int for all three
        W / H: a size (iterable of ints -> random non-negative init) or an initial non-negative Tensor
        Z: an initial non-negative (P, rank) Tensor (default: ones(P, rank) / rank), each row normalised
        trainable_W / trainable_H / trainable_Z: whether a *given tensor* is updated by `fit`

    `fit(V, ...)` takes V as (P, B, C, X1, X2, X3), or as one (B, C, X1, X2, X3) target shared by every problem.  Workspace:
    that of `BatchedNMF3D` at this shape, plus per fit the raw numerators of W and H and the EM step's scratch.
    """
    _ndim = 6
    _axes = "six axes (P, rows, rank, k1, k2, k3)"
    _conv = staticmethod(F.conv3d)

    def __init__(self, Vshape=None, rank=None, kernel_size=1, *, W=None, H=None, Z=None, trainable_W=True,
                 trainable_H=True, trainable_Z=True):
        if isinstance(Vshape, _Iterable):
            kernel_size = _triple(kernel_size)
            k1, k2, k3 = kernel_size
            P, B, C, X1, X2, X3 = Vshape
            rank = rank if rank else X2
            W = (P, C, rank) + tuple(kernel_size) if W is None else W
            H = (P, B, rank, X1 - k1 + 1, X2 - k2 + 1, X3 - k3 + 1) if H is None else H
        super().__init__(rank, W, H, Z, trainable_W, trainable_H, trainable_Z)
