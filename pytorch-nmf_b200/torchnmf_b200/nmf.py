"""NMF / NMFD modules with the reference's surface and an H100-native `fit`.

Mirrors the module surface of torchnmf 0.3.5 (`torchnmf/nmf.py`): `BaseComponent` (:173-292),
`NMF` (:641-697), `NMFD` (:700-779) and `BaseComponent.fit` (:298-409).  Constructor arguments,
parameter shapes (`W (C,R[,T])`, `H (N,R)` / `(B,R,L_in)`), `forward`, `state_dict` keys and the
`fit` signature / return value / exceptions are the reference's.  What differs is the inside of the
iteration loop: instead of materialising `WH` and taking two autograd backward passes
(`_double_backward_update`, :52-92), every update is one call into libnmf_b200.so, whose fused
sm_90a kernels never write the (N x C) reconstruction or ratio matrices to HBM.

There is no CPU compute path: `fit` on CPU-resident modules copies V / W / H to the current CUDA
device, runs there, and copies the factors back into the same Parameter storages ("host buffer"
mode, the `e2e` number of bench.py).  Without a CUDA device or without the built library it raises.

`NMF2D` (:782-865) and `NMF3D` (:868-942) run the NMFD contractions with the last axis sliding and the outer axes as loops.
Sparse targets are accepted by `NMF` and run on the library's sparse kernels at every beta > 0 up to rank 256 (densified on the
device above that rank, for sharded fits and for `sparse_fit`).
`sparse_fit` (:411-599, Hoyer's sparseness-constrained projected gradient) runs on the same engine: gradients from the fused
raw-terms launch, line-search losses from the fused loss launch, every component projected by ONE
`nmfb200_hoyer_project` launch.  `trainer.BetaMu` / `SparsityProj` and `plca.*` live in their own modules.
"""
import contextlib
import dataclasses
import math
import numbers
import weakref
from collections.abc import Iterable as _Iterable

import torch
import torch.nn.functional as F
from torch import Tensor
from torch.nn import Parameter

from .constants import eps  # noqa: F401  (re-exported like torchnmf.nmf does)
from . import engine as _engine

try:
    from tqdm import tqdm as _tqdm
except Exception:  # pragma: no cover
    class _tqdm:
        """The progress bar where tqdm is not installed: shows nothing."""
        def __init__(self, *a, **k): pass
        def __enter__(self): return self
        def __exit__(self, *a): return False
        def set_postfix(self, **k): pass
        def update(self, n): pass

__all__ = ["BaseComponent", "NMF", "NMFD", "NMF2D", "NMF3D", "BatchedNMF", "BatchedNMFD", "BatchedNMF2D",
           "BatchedNMF3D", "ARD"]


def _gamma(beta):
    # nmf.py:341-346
    if beta < 1:
        return 1.0 / (2.0 - beta)
    if beta > 2:
        return 1.0 / (beta - 1.0)
    return 1.0


def _get_norm(x, axis=1):
    """L2 norm over every axis but `axis` (nmf.py:134-139)."""
    dims = [d for d in range(x.dim()) if d != axis]
    return (x * x).sum(dims).sqrt()


@torch.no_grad()
def _renorm(W, H, unit_norm="W"):
    """Move the component norms to the other factor, in place (nmf.py:142-159)."""
    if unit_norm == "W":
        unit, other = W, H
    elif unit_norm == "H":
        unit, other = H, W
    else:
        raise ValueError("Input type isn't valid!")
    n = _get_norm(unit)
    unit /= n[(slice(None),) + (None,) * (unit.dim() - 2)]
    other *= n[(slice(None),) + (None,) * (other.dim() - 2)]


def _proj_func(s, k1, k2):
    """Hoyer's projection of ONE vector (any shape) onto {v >= 0, |v|_1 = k1, |v|_2^2 = k2} (nmf.py:21-49); returns a new
    tensor.  Runs in the library (`nmfb200_hoyer_project`): CUDA tensors only."""
    out = s.detach().clone().reshape(1, 1, -1)
    _engine.hoyer_project_(out, 1, [float(k1)], [float(k2)])
    return out.view(s.shape)


def _sparse_engine_cls(sparse_kernels, beta, rank, group):
    """The engine of a sparse target, or None when the target is densified on the device: the sparse kernels serve rank <= 256
    on one device (`group is None`); beta 1 and 2 take their own gathers and Gram / column sums, every other beta > 0 the
    engine whose denominators and loss are V-free dense contractions."""
    if not sparse_kernels or group is not None or rank > 256 or not beta > 0:
        return None
    return _engine.CudaSparseNmfEngine if beta in (1, 2) else _engine.CudaSparseAnyBetaEngine


def _observed_cells(V, M, device):
    """The observed set of a sparse mask M on `device`: a coalesced fp32 sparse COO tensor of V's shape whose stored entries
    are exactly the cells where M stores True (each once, explicit zeros kept), holding V's value there -- a dense V's element,
    gathered at those cells only, or a sparse V's stored value (0 where V stores nothing).  Linear indices row * C + col in
    int64, so N * C beyond 2^31 is fine."""
    N, C = V.shape
    M = M.to(device)
    idx, keep = M._indices(), M._values()                      # uncoalesced masks too: duplicates collapse in unique()
    lin = torch.unique(idx[0][keep] * C + idx[1][keep])        # sorted: the COO tensor is coalesced as built
    return _cells_of(V, lin, device)


def _weighted_cells(Wt, C, device):
    """The observed set of a sparse weight Wt (N, C) on `device`: (sorted linear indices row * C + col, fp32 weights there)
    of the cells whose weight is > 0, and whether every weight is valid (`_weight_values_ok` over every stored entry as
    given, before duplicates are summed, and over the sums).  Duplicate coordinates add up, as in `Wt.to_dense()`; stored
    zeros are dropped."""
    Wt = Wt.to(device)
    Wc = Wt.coalesce()
    w = Wc.values().to(torch.float32)
    ok = _weight_values_ok(torch.cat([Wt._values().to(torch.float32), w]))
    keep = w > 0
    idx = Wc.indices()
    return idx[0][keep] * C + idx[1][keep], w[keep].contiguous(), ok


def _cells_of(V, lin, device):
    """A coalesced fp32 sparse COO tensor of V's shape storing V's value at the cells `lin` (sorted linear indices, each
    once; explicit zeros kept): a dense V's element, gathered there only, or a sparse V's stored value (0 where V stores
    nothing)."""
    N, C = V.shape
    rows, cols = lin // C, lin % C
    if V.is_sparse:
        Vc = V.coalesce()
        vlin = (Vc.indices()[0] * C + Vc.indices()[1]).to(device)
        vvals = Vc.values().to(device, torch.float32)
        vals = torch.zeros(lin.numel(), dtype=torch.float32, device=device)
        if vlin.numel():
            pos = torch.searchsorted(vlin, lin).clamp_(max=vlin.numel() - 1)
            hit = vlin[pos] == lin
            vals = torch.where(hit, vvals[pos], vals)
    else:
        vals = V[rows.to(V.device), cols.to(V.device)].to(device, torch.float32)
    return torch.sparse_coo_tensor(torch.stack([rows, cols]), vals, (N, C), is_coalesced=True, check_invariants=False)


def _weight_values_ok(w):
    """One reduction over a weight's values (fp32, on its device): whether every weight is finite and >= 0.  No value (an
    empty shard) is fine; a weight that is zero everywhere is refused by fit() after the (collective) min / max of V over
    the weighted cells, as a mask with nothing observed is."""
    if w.numel() == 0:
        return True
    lo, hi = torch.stack(torch.aminmax(w)).tolist()
    return lo >= 0 and hi < math.inf                         # NaN fails both


_NO_CUDA = "torchnmf_b200.fit needs a CUDA device (sm_90a); there is no CPU fallback"


def _checked_fixed_w(W, fixed_W, group):
    """The checks of a `fit(..., fixed_W=F)` argument for the module's W, before any device work: ValueError for a
    `fixed_W` that is not a dense torch.bool tensor of one flag per component, for a W that is not trainable and for
    `group`.  Returns None when no component is fixed (the plain fit), else `fixed_W` itself."""
    if fixed_W is None or W is None:                # no W: fit()'s own assertion reports it
        return None
    R = W.shape[1]
    if not isinstance(fixed_W, Tensor) or fixed_W.dtype != torch.bool or fixed_W.layout != torch.strided:
        raise ValueError(f"fixed_W must be a dense torch.bool tensor (got {getattr(fixed_W, 'dtype', type(fixed_W))})")
    if tuple(fixed_W.shape) != (R,):
        raise ValueError(f"fixed_W must hold one flag per component of W: shape ({R},) (got {tuple(fixed_W.shape)})")
    if not W.requires_grad:
        raise ValueError("fixed_W: W is not trainable (trainable_W=False); every component is already fixed")
    if group is not None:
        raise ValueError("fixed_W does not run sharded fits (group)")
    return fixed_W if bool(fixed_W.any()) else None


@dataclasses.dataclass(frozen=True)
class ARD:
    """Automatic relevance determination with the l1 prior (V. Y. F. Tan and C. Fevotte, "Automatic relevance determination
    in nonnegative matrix factorization with the beta-divergence", IEEE TPAMI 35(7), 2013): `fit(V, ..., ard=ARD())`.

    a:   shape of the inverse-gamma prior on each relevance lambda_k (default 5.0; must be > 2 when b is None).
    b:   its scale; None sets it by moment matching, b = sqrt((a - 1)(a - 2) mean(V) / (R prod(K))), with mean(V) over the
         cells the fit reads and prod(K) = 1 for NMF.
    phi: the dispersion: 1 for KL (Poisson), the noise variance at beta 2.
    """
    a: float = 5.0
    b: float = None
    phi: float = 1.0


def _finite_positive(x):
    return isinstance(x, numbers.Real) and not isinstance(x, bool) and math.isfinite(x) and x > 0


def _checked_ard(ard, W, H, alpha, solver, group, fixed_W):
    """The checks of a `fit(..., ard=...)` argument, before any device work: ValueError for anything that is not an `ARD`,
    a non-finite or non-positive a, b or phi, a <= 2 without b, and for alpha, solver="cd", group, fixed_W and a frozen
    factor, which ARD does not combine with.  Returns `ard` (None: the plain fit)."""
    if ard is None:
        return None
    if not isinstance(ard, ARD):
        raise ValueError(f"ard must be an ARD instance (got {type(ard).__name__})")
    for name in ("a", "phi") + (("b",) if ard.b is not None else ()):
        if not _finite_positive(getattr(ard, name)):
            raise ValueError(f"ARD.{name} must be finite and > 0 (got {getattr(ard, name)!r})")
    if ard.b is None and not ard.a > 2:
        raise ValueError(f"ARD.a must be > 2 to set b by moment matching (got {ard.a!r}); pass b")
    if alpha != 0:
        raise ValueError("ard: ARD replaces the alpha / l1_ratio penalty; alpha must be 0")
    if solver == "cd":
        raise ValueError("ard: ARD runs the multiplicative updates; solver='cd' is not supported")
    if group is not None:
        raise ValueError("ard does not run sharded fits (group)")
    if fixed_W is not None:
        raise ValueError("ard does not combine with fixed_W")
    if W is not None and H is not None and not (W.requires_grad and H.requires_grad):
        raise ValueError("ard: W and H must both be trainable")
    return ard


def _ard_mean(V, mask=None, weight=None):
    """mean(V) over the cells a fit reads, in float64: every cell of a dense target; the observed cells of a mask (NaN at the
    missing cells never enters); the cells of weight > 0, unweighted; the stored values of a sparse COO target over N x C."""
    f64 = torch.float64
    if weight is not None and weight.is_sparse:
        lin, _, _ = _weighted_cells(weight, V.shape[1], weight.device)
        vals = _cells_of(V, lin, weight.device).values()
        return float(vals.sum(dtype=f64)) / max(vals.numel(), 1)
    if mask is not None and mask.is_sparse:
        vals = _observed_cells(V, mask, mask.device).values()
        return float(vals.sum(dtype=f64)) / max(vals.numel(), 1)
    if weight is not None or mask is not None:
        on = (weight > 0) if weight is not None else mask
        on = on.to(V.device)
        total = torch.where(on, V, torch.zeros((), dtype=V.dtype, device=V.device)).sum(dtype=f64)
        return float(total) / max(int(on.sum()), 1)
    if V.is_sparse:
        return float(V._values().sum(dtype=f64)) / V.shape[0] / V.shape[1]
    return float(V.sum(dtype=f64)) / V.numel()


def _ard_constants(ard, V, W, H, mask=None, weight=None):
    """(b, c) of an ARD fit: c = n_W + n_H + a + 1, n_W and n_H the entries of one component of W and of H; b as given or
    by moment matching (`ARD`).  ValueError when that b is not positive (a target of mean 0)."""
    R = W.shape[1]
    n_w, n_h = W.numel() // R, H.numel() // R
    c = n_w + n_h + ard.a + 1.0
    b = ard.b
    if b is None:
        prod_k = math.prod(W.shape[2:])
        b = math.sqrt((ard.a - 1.0) * (ard.a - 2.0) * _ard_mean(V, mask, weight) / (R * prod_k))
        if not _finite_positive(b):
            raise ValueError(f"ard: moment matching gives b = {b!r} (the target's mean is not positive); pass ARD(b=...)")
    return float(b), float(c)


class BaseComponent(torch.nn.Module):
    """Base class of the NMF modules (reference: nmf.py:173-292).

    Args:
        rank: size of the hidden dimension
        W / H: a size (iterable of ints -> random non-negative init) or an initial non-negative Tensor
        trainable_W / trainable_H: whether a *given tensor* is updated by `fit`
    """

    def __init__(self, rank=None, W=None, H=None, trainable_W=True, trainable_H=True):
        super().__init__()
        inferred = None
        for name, spec, trainable in (("W", W, trainable_W), ("H", H, trainable_H)):
            if isinstance(spec, Tensor):
                assert torch.all(spec >= 0.), f"Tensor {name} should be non-negative."   # nmf.py:215,227
                p = Parameter(torch.empty(*spec.size()), requires_grad=trainable)
                p.data.copy_(spec)
                self.register_parameter(name, p)
                inferred = p.shape[1]
            elif isinstance(spec, _Iterable):
                spec = tuple(spec)
                self.register_parameter(name, Parameter(torch.randn(*spec).abs()))       # nmf.py:221,234
                inferred = spec[1]
            else:
                self.register_parameter(name, None)

        if inferred is None:
            assert rank, "A rank should be given when W and H are not available!"        # nmf.py:240
        else:
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

    def forward(self, H=None, W=None):
        """Reconstruction only (nmf.py:261-284); plain differentiable torch ops, not on the fit path."""
        own = H is None and W is None
        H = self.H if H is None else H
        W = self.W if W is None else W
        assert H is not None
        assert W is not None
        out = self.reconstruct(H, W)
        if own and type(self) in _BETAMU_FUSABLE:
            # the plain reconstruction of this module's own factors: lets trainer.BetaMu recognise a single-leaf graph
            # and take both update terms from the fused kernels instead of two backward passes through `out`
            out._nmf_b200_src = weakref.ref(self)
        return out

    @staticmethod
    def reconstruct(H, W):
        raise NotImplementedError

    # ---- engine selection -------------------------------------------------------------------
    _engine_cls = None

    def _check_target_shape(self, V):
        raise NotImplementedError

    # test hook (tests/oracle_engine.py): an engine class used instead of the CUDA engines, so the host logic of `fit`
    # can be tested on a GPU-less box.  Deliberately NOT a parameter of `fit`: its signature stays the reference's.
    _engine_factory = None
    _sparse_targets = False       # NMF only (nmf.py:603-638); the convolutive models raise, as in the reference
    _sparse_kernels = True        # a sparse target on the library's sparse kernels (False: densify)
    _strided_target = False       # the engine reads a row-strided (unit column stride) half-precision target as it is
    _cd_solver = False            # fit(..., solver="cd") at beta 2: NMF only

    def _checked_target(self, V, beta, mask=None, weight=None):
        """The checks of `fit` / `sparse_fit` that need no device pass, in the reference's order; returns the target, a
        sparse one coalesced."""
        observed = (mask is not None and mask.is_sparse) or (weight is not None and weight.is_sparse)
        sparse_target = V.is_sparse and not observed
        if sparse_target and not self._sparse_targets:
            raise NotImplementedError                      # nmf.py:294-295: only NMF derives the sparse update
        if sparse_target:
            # The reference's sparse derivation (nmf.py:95-119, :603-638: SDDMM at the non-zeros) is the same update as the
            # dense one on V.to_dense() -- its own tests/test_nmf_sparse.py:8-37 asserts exactly that.  The library's sparse
            # kernels take it at every beta > 0 (_sparse_engine_cls): the numerators at the non-zeros only, and for beta
            # != 1, 2 the denominators and the loss's sum (WH + eps)^beta from dense contractions that never read V, so the
            # device holds O(nnz + (N + C) R), not N x C.  Ranks above 256, sharded fits and `sparse_kernels=False` densify
            # the target ON THE DEVICE and take the fused dense kernels (memory = the dense size).
            V = V.coalesce()
            assert torch.all(V.values() >= 0.), "Target should be non-negative."            # nmf.py:329-330
            if beta <= 0:                                                                    # nmf.py:332-336
                raise ValueError("When beta <= 0 and V contains zeros, the training process may diverge. "
                                 "Please add small values to V, or use a positive beta value.")
        assert self.W is not None and self.H is not None, "fit() needs both W and H"
        self._check_target_shape(V)
        return V

    def _open_engine(self, V, dev, Wd, Hd, beta, precision, group, sparse_kernels, mask=None, weight=None):
        """The engine of `fit` / `sparse_fit` for the target V (`_checked_target`) on the device `dev`, updating the fp32
        factors Wd / Hd (`_placed_factors`).  A dense bf16 / fp16 target keeps its dtype, other target dtypes are staged
        through an fp32 device copy.  A `mask` (validated by `_check_mask`) is set on the engine: moved to its device and
        made contiguous, read there in place as one byte per cell.  A `weight` (validated by `_check_weight`) is set the
        same way as one fp32 per cell (other dtypes staged through one fp32 copy), after one reduction over its values
        (`_weight_values_ok`, agreed on by every rank with `group`, so that all of them raise together); a sparse one takes
        the observed-cell kernels."""
        wsparse = weight is not None and weight.is_sparse    # a sparse weight: the observed-cell kernels (NMF, _check_weight)
        observed = (mask is not None and mask.is_sparse) or wsparse
        sparse_target = V.is_sparse and not observed
        rank = Wd.shape[1]
        wok = True
        if self._engine_factory is None:
            f32 = torch.float32
            wv = None
            if observed:
                # the observed cells up to rank 256 (sharded or not); above it, scattered into a dense fp32 V and a dense
                # mask (or weight) on the device, for the dense masked (weighted) kernels
                if wsparse:
                    lin, wv, wok = _weighted_cells(weight, V.shape[1], dev)
                    O = _cells_of(V, lin, dev)
                else:
                    O = _observed_cells(V, mask, dev)
                if rank <= 256:
                    Vd, sparse_cls, mask, weight = O, _engine.CudaObservedNmfEngine, None, None
                else:
                    rows, cols = O.indices()
                    Vd = torch.zeros(O.shape, dtype=f32, device=dev)
                    Vd[rows, cols] = O.values()
                    if wsparse:
                        weight = torch.zeros(O.shape, dtype=f32, device=dev)
                        weight[rows, cols] = wv
                        wv = None
                    else:
                        mask = torch.zeros(O.shape, dtype=torch.bool, device=dev)
                        mask[rows, cols] = True
                    sparse_cls = None
            else:
                Vd = V.to(dev, non_blocking=True)
                sparse_cls = (_sparse_engine_cls(sparse_kernels and self._sparse_kernels, beta, rank, group)
                              if sparse_target else None)
                if not sparse_target and Vd.dtype in (torch.float16, torch.bfloat16):
                    # the kernels convert each element exactly where they load it: the fit is bit for bit that of V.float(),
                    # without the fp32 copy (4 bytes per element of V)
                    if not (self._strided_target and Vd.stride(-1) == 1 and Vd.stride(0) >= Vd.shape[1]):
                        Vd = Vd.contiguous()
                elif sparse_cls is None:
                    Vd = (Vd.to_dense() if sparse_target else Vd).to(f32).contiguous()
            if weight is not None and not wsparse:
                weight = weight.to(dev, f32).contiguous()
                wok = _weight_values_ok(weight)
            if wv is not None:
                eng = sparse_cls(Vd.coalesce(), Wd, Hd, weights=wv)
            elif sparse_cls is not None:
                eng = sparse_cls(Vd.coalesce(), Wd, Hd)
            else:
                eng = self._engine_cls(Vd, Wd, Hd, precision)
            Md = mask.to(dev).contiguous() if mask is not None else None
        else:
            if wsparse:
                lin, wv, wok = _weighted_cells(weight, V.shape[1], dev)
                eng, Md, weight = self._engine_factory(_cells_of(V, lin, dev), Wd, Hd, weights=wv), None, None
            elif observed:
                eng, Md = self._engine_factory(_observed_cells(V, mask, dev), Wd, Hd), None
            else:
                if weight is not None:
                    weight = weight.to(torch.float32).contiguous()
                    wok = _weight_values_ok(weight)
                eng = self._engine_factory(V.to_dense() if (sparse_target and not sparse_kernels) else V, Wd, Hd)
                Md = mask
        if group is not None:
            eng = _engine.ShardedEngine(eng, group)
            if eng.kind == "nmfd":
                # batch shards: the W terms' length depends on everything but B (ndim 1 to 3, padded with zeros to 3)
                nd = V.dim() - 2
                names = ["ndim", "C", "R"] + [f"kernel_size[{i}]" for i in range(3)] + [f"V.shape[{i + 2}]" for i in range(3)]
                pad = [0] * (3 - nd)
                try:
                    eng.check_same_sizes(names, [nd, V.shape[1], rank, *Wd.shape[2:], *pad, *V.shape[2:], *pad])
                except ValueError:
                    eng.close()
                    raise
            if wsparse or weight is not None:
                wok = eng.all_ranks(wok)          # collective: a bad weight on any rank makes every rank raise
        if not wok:
            eng.close()
            raise ValueError("weight: every weight must be finite and >= 0 (found a negative, NaN or Inf weight)")
        if Md is not None or weight is not None:
            try:
                if Md is not None:
                    eng.set_mask(Md)
                else:
                    eng.set_weight(weight)
            except Exception:
                eng.close()
                raise
        return eng

    @classmethod
    def _check_mask(cls, V, mask, precision):
        """fit()'s checks of a mask that need no device pass."""
        if not isinstance(mask, Tensor) or mask.dtype != torch.bool:
            raise ValueError(f"mask must be a torch.bool tensor (got {getattr(mask, 'dtype', type(mask))})")
        if mask.is_sparse:
            if not cls._sparse_targets:
                raise ValueError(f"mask: a sparse mask is supported by NMF only (got {cls.__name__}); pass a dense mask")
        elif V.is_sparse:
            raise ValueError("mask: a masked fit needs a dense target")
        if tuple(mask.shape) != tuple(V.shape):
            raise ValueError(f"mask shape {tuple(mask.shape)} does not match the target's {tuple(V.shape)}")
        if precision in ("f16", "f16_split"):
            raise ValueError(f"mask: masked fits run on the fp32 kernels; precision must be 'auto' or 'f32' (got {precision!r})")

    @classmethod
    def _check_weight(cls, V, weight, precision):
        """fit()'s checks of a weight that need no device pass (the values: `_weight_values_ok`)."""
        if not isinstance(weight, Tensor) or not weight.dtype.is_floating_point:
            raise ValueError(f"weight must be a floating-point tensor (got {getattr(weight, 'dtype', type(weight))})")
        if weight.is_sparse:
            if not cls._sparse_targets:
                raise ValueError(f"weight: a sparse weight is supported by NMF only (got {cls.__name__}); pass a dense weight")
        elif V.is_sparse:
            raise ValueError("weight: a dense weight needs a dense target (pass a sparse weight for a sparse target)")
        if tuple(weight.shape) != tuple(V.shape):
            raise ValueError(f"weight shape {tuple(weight.shape)} does not match the target's {tuple(V.shape)}")
        if precision in ("f16", "f16_split"):
            raise ValueError(f"weight: weighted fits run on the fp32 kernels; precision must be 'auto' or 'f32' "
                             f"(got {precision!r})")

    def _check_cd(self, beta, precision, group, mask, weight):
        """fit(solver="cd")'s refusals, before any device work."""
        if not self._cd_solver:
            raise ValueError(f"solver='cd' is supported by NMF only (got {type(self).__name__})")
        if beta != 2:
            raise ValueError(f"solver='cd' minimises the beta = 2 objective; beta must be 2 (got {beta!r})")
        for name, sel in (("mask", mask), ("weight", weight)):
            if isinstance(sel, Tensor) and not sel.is_sparse:
                raise ValueError(f"solver='cd' takes a sparse {name} only, fitted on its observed cells; pass "
                                 f"{name}.to_sparse()")
        if group is not None:
            raise ValueError("solver='cd' does not run sharded fits (group)")
        if precision in ("f16", "f16_split"):
            raise ValueError(f"solver='cd' runs on the fp32 kernels; precision must be 'auto' or 'f32' (got {precision!r})")
        rank = self.W.shape[1] if self.W is not None else self.rank
        if rank > 256:
            raise ValueError(f"solver='cd' supports rank <= 256 (got {rank})")

    @torch.no_grad()
    def fit(self, V, beta=1, tol=1e-4, max_iter=200, verbose=False, alpha=0, l1_ratio=0, *,
            precision="auto", group=None, **options):
        """Learn the model for `V` by minimising the beta-divergence with multiplicative updates.

        Positional arguments, defaults, return value (`n_iter`) and exceptions are those of
        `BaseComponent.fit` in the reference (nmf.py:298-409).  Keyword-only extras:

        precision: "auto" | "f32" | "f16" | "f16_split" -- arithmetic of the contraction kernels ("auto": fp16
                   tensor-core operands where the target fits their range, fp32 CUDA cores otherwise).  NMF2D / NMF3D:
                   "auto" and "f32" run the fp32 kernels; "f16" runs beta 1 on the tensor-core sliding GEMMs (rank <= 256)
                   and other betas on the fp32 kernels.  `last_fit_precision` reports what ran.
        group:     a torch.distributed process group; V and H are then this rank's shard and W is replicated, identical
                   on every rank at entry; one all-reduce per W update.  NMF shards the rows (rows of V <-> rows of H);
                   NMFD / NMF2D / NMF3D shard the batch axis (V (B_local,C,*X) <-> H (B_local,R,...)), and every rank
                   must have the same C, R, kernel size and sizes past the batch axis (ValueError otherwise).  Shards may
                   be uneven.  Each rank resolves precision="auto" from its own shard.

        dtype: the kernels keep fp32 master factors and fp32 accumulators.  The reference computes in the module's
        dtype (nmf.py:214-218).  Here a dense bfloat16 / float16 target is read as it is, with no fp32 copy (NMF also
        takes a row-strided view), and gives exactly the fit of `V.float()`; a float64 target is staged through an fp32
        copy.  A float64 / half module, or fp32 factors that are not contiguous, are staged through fp32 copies and the
        result is written back into the same Parameter storages in their own dtype and layout.

        sparse V (NMF, a COO tensor): fitted without densifying it at every beta > 0 up to rank 256 -- the update terms at
        the stored entries only and, for beta != 1, 2, the denominators and the loss's sum (WH + eps)^beta from dense
        contractions that never read V, so the device holds O(nnz + (N + C) R).  Above rank 256 or with `group`, the
        target is densified on the device.

        mask:      (keyword-only, default None; taken through **options so the named parameters stay the reference's
                   plus `precision` and `group`) a torch.bool tensor of V's shape, True where V is observed: the fit minimises beta_div(WH[mask],
                   V[mask]) -- the missing cells are dropped, not zeroed -- with every update the reference's ratio
                   (nmf.py:78-92) of the two backward passes of that loss, i.e. what `trainer.BetaMu` does with the closure
                   `(V[mask], model()[mask])`.  At beta 1 the denominator is therefore mask-weighted, not the column sums.
                   The missing cells of V are never read into arithmetic (NaN there is fine), and the non-negativity and
                   beta <= 0 checks look at the observed cells only.  A row or column with no observed cell leaves its row of
                   H or W unchanged when alpha = 0.  Dense targets only (any dtype or row stride V may have), on the fp32
                   kernels: precision "auto" resolves to "f32", "f16" / "f16_split" raise ValueError.  With `group`, each
                   rank passes the mask shard of its V shard.
                   NMF also takes a sparse COO torch.bool mask: the observed cells are the coordinates where it stores True
                   (a coordinate listed twice counts once; stored False entries are not observed), and V -- dense of any
                   dtype or row stride, or sparse COO (0 where it stores nothing; its entries outside the mask are ignored)
                   -- is read at those cells only.  The objective is the same; up to rank 256 every update and the loss
                   run on the observed cells alone, O(observed x R) per update and O(observed + (N + C) R) memory, for
                   matrix completion where few cells are observed.  Above rank 256 the observed values and the mask are
                   densified on the device.  With `group`, each rank passes the row shards of V and of the mask.  A
                   sparse mask also takes solver="cd" at beta 2 (see `solver`); a dense one does not.

        weight:    (keyword-only, default None, through **options like `mask`; exclusive with it -- fold a mask into the
                   weight) a floating-point tensor of V's shape holding one weight w >= 0 per cell: the fit minimises
                   sum over the cells with w > 0 of w * d_beta(v | WH), with every update the reference's ratio
                   (nmf.py:78-92) of the two backward passes of that loss (num = contraction of w V (WH + eps)^(beta-2),
                   den = of w (WH + eps)^(beta-1); at beta 1 den is the weighted contraction, not the column sums).  The
                   loss reported and used by the stop rule is sqrt(2 sum w d_beta), summed over ranks with `group`.
                   Confidence weights, per-bin reliabilities or inverse noise variances are the usual uses; weights in
                   {0, 1} give exactly the fit of the mask `weight > 0`.  Cells of weight 0 are dropped as missing cells
                   are for a mask: V is never read there, and the non-negativity and beta <= 0 checks look at the cells
                   with w > 0 only.  ValueError: a non-floating weight, a shape mismatch, any negative, NaN or Inf weight
                   (one reduction at entry; a sparse weight's stored entries are checked before duplicates are summed),
                   a weight that is zero everywhere, precision "f16" / "f16_split" ("auto" resolves to "f32").  A float32
                   weight is read in place (NMF: contiguous N x C whatever V's stride); float16, bfloat16 and float64
                   ones are staged through one fp32 copy on the device.  V is dense, of any
                   dtype (NMF: any row stride).  NMF also takes a sparse COO float weight: the observed cells are its
                   stored entries with w > 0 (duplicate coordinates add up, as in `weight.to_dense()`), V is dense or
                   sparse COO (0 where it stores nothing), and up to rank 256 every update and the loss run on those
                   cells alone, O(observed x R) per update; above rank 256 the weights and values are densified on the
                   device.  A dense weight on a sparse V and a sparse weight on NMFD / NMF2D / NMF3D raise ValueError.
                   A sparse weight also takes solver="cd" at beta 2 (see `solver`); a dense one does not.
                   With `group`, each rank passes the weight shard of its V shard; a shard may be zero everywhere (or,
                   sparse, store nothing), and the value check is agreed on by all ranks, so every rank raises together.

        solver:    (keyword-only, default "mu", through **options like `mask`) "mu" -- the multiplicative updates above -- or
                   "cd": coordinate descent (HALS, sklearn's `solver="cd"`) at beta 2, which usually reaches a given loss
                   in far fewer iterations.  It minimises 1/2 |V - H W^T|^2 + l1 (sum W + sum H) + l2 / 2 (|W|^2 + |H|^2),
                   l1 = alpha * l1_ratio and l2 = alpha * (1 - l1_ratio) as for "mu".  Each iteration updates W, then H
                   with the new W; each update is one sweep over the factor's columns k = 0 .. R-1 in order, every row c
                   at once:  X[c,k] <- max(0, X[c,k] + (A[c,k] - sum_j X[c,j] B[j,k] - l1 - l2 X[c,k]) / (B[k,k] + l2)),
                   with A = V^T H, B = H^T H for W and A = V W, B = W^T W for H, taken at the start of the update; a
                   column with B[k,k] + l2 == 0 (a dead component) is left as it is.  The floor is exactly 0, so the
                   objective never rises in exact arithmetic -- and a later "mu" fit cannot move an entry that is exactly
                   0.  Loss, stop rule and return value are those of "mu".  NMF only, on the fp32 kernels: precision
                   "auto" resolves to "f32" and `last_fit_precision` is "f32".  V dense (float32, float16 or bfloat16 read
                   in place at any row stride; float64 staged) or sparse COO; `alpha`, `l1_ratio`, frozen factors and
                   host or float64 modules work as for "mu".
                   With a sparse `mask` or `weight` (NMF, rank <= 256), "cd" fits the observed cells O alone:
                   1/2 sum_O w (v - h_n . w_c)^2 + the same penalties (w = 1 for a mask), by coordinate descent on O
                   (CCD++, Yu et al. 2012, made non-negative).  Each update is one exact sweep per row s of the factor
                   over the observed cells O_s of its segment (a column of V for W, a row for H): with f_j the other
                   factor's row of cell j and r = v - f_j . x_s at the current x_s, for k = 0 .. R-1 in order,
                   num = sum_{O_s} w r f_{j,k}, hess = sum_{O_s} w f_{j,k}^2 + l2, and if hess != 0,
                   x_{s,k} <- max(0, x_{s,k} + (num - l1 - l2 x_{s,k}) / hess).  O(observed x R) per update, device
                   memory O(observed + (N + C) R); the loss is the observed-cell loss "mu" reports.  Every cell observed
                   with unit weights gives the update above in exact arithmetic.  ValueError, before any device work:
                   beta != 2, a dense `mask` or `weight` (pass `mask.to_sparse()`: a dense one would need a Gram matrix
                   per row), `group`, precision "f16" / "f16_split", rank > 256, an unknown solver, and NMFD / NMF2D /
                   NMF3D.

        fixed_W:   (keyword-only, default None, through **options like `mask`) a torch.bool tensor of R elements, on any
                   device: the components k where it is True keep W[:, k] (W[:, k, ...] for NMFD / NMF2D / NMF3D) at its
                   value, for semi-supervised separation (Mysore and Smaragdis 2011): a dictionary learned for a known
                   source stays fixed while the free components learn the rest of the target.  The free components take
                   exactly the update they take without it, with the reconstruction formed from all R components: the
                   multiplicative ratio (`alpha` / `l1_ratio` penalise the free components only, since the fixed ones are
                   not updated), or with solver="cd" the sweep over k = 0 .. R-1 that skips each fixed k, so later columns
                   see its unchanged value (block coordinate descent on the free components).  H is learned for every
                   component.  Every component fixed is the fit of trainable_W=False, bit for bit; none fixed is the plain
                   fit.  Every target form, precision and solver above is covered.  ValueError, before any device work: a
                   `fixed_W` that is not a dense torch.bool tensor of shape (R,), a W that is not trainable, and `group`.

        ard:       (keyword-only, default None, through **options like `mask`) an `ARD(a=5.0, b=None, phi=1.0)`: choose the
                   rank during the fit by automatic relevance determination with the l1 prior (Tan and Fevotte, TPAMI
                   2013).  Fit with a generous R; component k gets a relevance lambda_k and the fit minimises
                     J = D / phi + sum_k [(sum W[:, k] + sum H[:, k] + b) / lambda_k + c log lambda_k],
                   c = n_W + n_H + a + 1 (n_W, n_H: the entries of one component of W and of H), D the divergence this fit
                   minimises without it (masked or weighted as given).  lambda starts at (sum W0[:, k] + sum H0[:, k] +
                   b) / c; each iteration updates W, then H, each by the multiplicative update with l1_reg = phi /
                   lambda_k on component k (the same exponent gamma(beta)), then sets lambda_k the same way from the new
                   factors.  J never increases in exact arithmetic; a component the data does not support shrinks to zero
                   and its lambda_k settles at the bound b / c.  b=None sets b by moment matching (`ARD`).  Stop rule: at
                   every 10th iteration, stop when max_k |lambda_k - its previous value| / its previous value < tol.
                   Afterwards `ard_lambda` holds lambda (float32, shape (R,), on the factors' device) and `ard_bound`
                   b / c.  The fit removes no component; keep the relevant ones with, for example,
                     keep = m.ard_lambda > m.ard_bound * (1 + 1e-3)
                     W, H = m.W.data[:, keep], m.H.data[:, keep]
                   NMF, NMFD, NMF2D and NMF3D on every target form and precision above.  ValueError, before any device
                   work: an `ard` that is not an `ARD`, a, b or phi not finite and > 0, a <= 2 with b=None, alpha != 0,
                   solver="cd", `group`, `fixed_W`, and a W or H that is not trainable.
        """
        mask = options.pop("mask", None)
        weight = options.pop("weight", None)
        solver = options.pop("solver", "mu")
        fixed_W = options.pop("fixed_W", None)
        ard = options.pop("ard", None)
        if options:
            raise TypeError(f"fit() got an unexpected keyword argument {next(iter(options))!r}")
        ard = _checked_ard(ard, self.W, self.H, alpha, solver, group, fixed_W)
        fixed_W = _checked_fixed_w(self.W, fixed_W, group)
        if solver not in ("mu", "cd"):
            raise ValueError(f"solver must be 'mu' or 'cd' (got {solver!r})")
        cd = solver == "cd"
        if cd:
            self._check_cd(beta, precision, group, mask, weight)
            precision = "f32"
        if mask is not None and weight is not None:
            raise ValueError("mask and weight are exclusive: fold the mask into the weight (weight * mask)")
        if mask is not None:
            self._check_mask(V, mask, precision)
            precision = "f32"
        if weight is not None:
            self._check_weight(V, weight, precision)
            precision = "f32"
        V = self._checked_target(V, beta, mask, weight)
        W, H = self.W, self.H
        with _placed_factors(self, (W, H), _NO_CUDA) as (dev, (Wd, Hd)):
            eng = self._open_engine(V, dev, Wd, Hd, beta, precision, group, True, mask, weight)
            try:
                vmin, vmax = eng.minmax()
                if mask is not None and vmin > vmax:                                       # +inf / -inf: nothing seen
                    raise ValueError("mask: no cell of the target is observed")
                if weight is not None and vmin > vmax:                                     # on every rank of a group
                    raise ValueError("weight: every weight is zero")
                assert vmin >= 0., "Target should be non-negative."                        # nmf.py:329-330
                if vmin == 0 and beta <= 0:                                                # nmf.py:332-336
                    raise ValueError("When beta <= 0 and V contains zeros, the training process may diverge. "
                                     "Please add small values to V, or use a positive beta value.")
                gamma = _gamma(beta)
                l1_reg = alpha * l1_ratio                                                  # nmf.py:348
                l2_reg = alpha * (1 - l1_ratio)                                            # nmf.py:349
                train_w, train_h = W.requires_grad, H.requires_grad
                if fixed_W is not None and bool(fixed_W.all()):
                    train_w = False                     # every component fixed: the fit of trainable_W=False
                elif fixed_W is not None:
                    eng.set_fixed_w(fixed_W.to(dev, torch.uint8).contiguous())

                def divergence(follows):
                    # a W update follows on these very factors: the engine may take the loss out of that update's own
                    # contraction pass (engine.loss_prefetch_w) instead of a pass over V of its own
                    if follows and train_w and group is None and hasattr(eng, "loss_prefetch_w"):
                        return eng.loss_prefetch_w(beta)
                    return eng.loss(beta)

                if ard is not None:
                    b, c = _ard_constants(ard, V, W, H, mask, weight)
                    eng.set_ard(b, c, ard.phi)
                    n_iter = _fit_ard(eng, beta, gamma, divergence, max_iter, tol, verbose)
                    self.ard_lambda = eng.ard_state()[0].to(W.device, copy=True)
                    self.ard_bound = b / c
                else:
                    step = _update_step(eng, cd, train_w, train_h, beta, gamma, l1_reg, l2_reg)
                    n_iter = _fit_single(step, divergence, max_iter, tol, verbose)
                if hasattr(eng, "check_health"):
                    eng.check_health()
                self.last_fit_precision = eng.precision_for(beta) if hasattr(eng, "precision_for") else eng.precision
                self.last_w_update_path = getattr(eng, "w_update_path", None)  # sharded fits: "peer" (NVLink P2P) or "nccl"
            finally:
                eng.close()
        return n_iter + 1                                                                  # nmf.py:409


    @torch.no_grad()
    def sparse_fit(self, V, beta=2, max_iter=200, verbose=False, sW=None, sH=None, *, precision="auto"):
        """Learn the model for `V` under Hoyer's sparseness constraints (reference: nmf.py:411-599).

        Positional arguments, defaults, return value and exceptions are the reference's: `sW` / `sH` in (0, 1) fix the
        sparseness of every component W[:, r] / H[:, r]; a factor without a constraint takes the multiplicative update
        (nmf.py:503-511), a constrained one a projected-gradient step with a halving line search (:513-538), and H is
        re-normalised to unit component norms after its update (:588).  No stop rule: `max_iter` iterations are run.

        On the engine: the gradient is `positive - negative` of ONE fused raw-terms launch (`nmfb200_raw_terms`), every
        line-search loss one fused loss launch on the trial factor, and the per-component Python loop around `_proj_func`
        (nmf.py:519-522: R x rounds x 7 ATen launches and one `.item()` per round) is one `nmfb200_hoyer_project` launch.

        precision: as in `fit`; "auto" resolves to "f32" when a constraint is active (the line search compares losses of
        nearly equal trial points).  Sparse targets are densified on the device.
        """
        constrained = ((sW is not None and self.W is not None and self.W.requires_grad)
                       or (sH is not None and self.H is not None and self.H.requires_grad))
        if precision == "auto" and constrained:
            precision = "f32"
        V = self._checked_target(V, beta)
        W, H = self.W, self.H
        with _placed_factors(self, (W, H), _NO_CUDA) as (dev, (Wd, Hd)):
            eng = self._open_engine(V, dev, Wd, Hd, beta, precision, None, False)
            try:
                vmin, vmax = eng.minmax()
                assert vmin >= 0., "Target should be non-negative."                        # nmf.py:447-448
                if vmin == 0 and beta <= 0:                                                # nmf.py:450-454
                    raise ValueError("When beta <= 0 and V contains zeros, the training process may diverge. "
                                     "Please add small values to V, or use a positive beta value.")
                train_w, train_h = W.requires_grad, H.requires_grad
                R = Wd.shape[1]
                L1a = L1s = None
                if sW is not None and train_w:                                             # nmf.py:459-467
                    L1a = Wd[:, 0].numel() ** 0.5 * (1 - sW) + sW
                    eng.project(Wd, 1, [L1a] * R, [1.0] * R)
                if sH is not None and train_h:                                             # nmf.py:469-477
                    L1s = Hd[:, 0].numel() ** 0.5 * (1 - sH) + sH
                    eng.project(Hd, 1, [L1s] * R, [1.0] * R)
                eng.sync()
                gamma = _gamma(beta)                                                       # nmf.py:479-484
                step = {0: 1.0, 1: 1.0}                                                    # nmf.py:490

                def projected_step(which, L1):
                    """nmf.py:513-538 (W) / :559-586 (H): gradient step, projection of every component, halving line
                    search."""
                    cur = Wd if which == 0 else Hd
                    loss = eng.loss(beta)
                    num, den = eng.raw_terms(which, beta)
                    if beta == 1:
                        den = den.view((1, -1) + (1,) * (cur.dim() - 2))                   # colsum of the other factor
                    grad = den - num
                    for _ in range(10):
                        new = cur - step[which] * grad
                        norms = _get_norm(new)
                        eng.project(new, 1, L1 * norms, norms * norms)
                        new_loss = eng.loss_at(new if which == 0 else Wd, Hd if which == 0 else new, beta)
                        if new_loss <= loss:
                            break
                        step[which] *= 0.5
                    step[which] *= 1.2
                    cur.copy_(new)
                    eng.sync()

                n_iter = -1
                with _tqdm(total=max_iter, disable=not verbose) as pbar:
                    for n_iter in range(max_iter):
                        if train_w:
                            if L1a is None:
                                eng.update_w(beta, gamma, 0.0, 0.0)                        # nmf.py:503-511
                            else:
                                projected_step(0, L1a)
                        if train_h:
                            if L1s is None:
                                eng.update_h(beta, gamma, 0.0, 0.0)                        # nmf.py:549-557
                            else:
                                projected_step(1, L1s)
                            _renorm(Wd, Hd, "H")                                           # nmf.py:588
                            eng.sync()
                        if n_iter % 10 == 9 and verbose:                                   # nmf.py:590-598 (display only)
                            d = eng.loss(beta)
                            pbar.set_postfix(loss=math.sqrt(2.0 * d) if d >= 0 else float("nan"))
                            pbar.update(10)
                if hasattr(eng, "check_health"):
                    eng.check_health()
                self.last_fit_precision = eng.precision_for(beta) if hasattr(eng, "precision_for") else eng.precision
            finally:
                eng.close()
        return n_iter + 1                                                              # nmf.py:599


class NMF(BaseComponent):
    """Non-negative matrix factorisation  V (N,C) ~= H (N,R) @ W (C,R)^T   (reference: nmf.py:641-697)."""
    _engine_cls = _engine.CudaNmfEngine
    _sparse_targets = True
    _strided_target = True
    _cd_solver = True

    def __init__(self, Vshape=None, rank=None, **kwargs):
        if isinstance(Vshape, _Iterable):
            M, K = Vshape                                  # wrong arity raises, as in the reference (:684)
            rank = rank if rank else K
            kwargs["W"] = (K, rank)
            kwargs["H"] = (M, rank)
        super().__init__(rank, **kwargs)

    @staticmethod
    def reconstruct(H, W):
        return F.linear(H, W)                              # H @ W^T, nmf.py:691-693

    def _check_target_shape(self, V):
        if V.dim() != 2 or V.shape[0] != self.H.shape[0] or V.shape[1] != self.W.shape[0]:
            raise RuntimeError(f"target shape {tuple(V.shape)} does not match H {tuple(self.H.shape)} / "
                               f"W {tuple(self.W.shape)}")


class NMFD(BaseComponent):
    """Non-negative matrix factor deconvolution (reference: nmf.py:700-779).

    V (B,C,L) ~= sum_t W[:,:,t] @ shift_t(H),  W (C,R,T), H (B,R,L-T+1).
    """
    _engine_cls = _engine.CudaNmfdEngine

    def __init__(self, Vshape=None, rank=None, T=1, **kwargs):
        if isinstance(Vshape, _Iterable):
            if isinstance(T, _Iterable):
                T, = T
            batch, K, M = Vshape                           # wrong arity raises, as in the reference (:769)
            rank = rank if rank else K
            kwargs["W"] = (K, rank, T)
            kwargs["H"] = (batch, rank, M - T + 1)
        super().__init__(rank, **kwargs)

    @staticmethod
    def reconstruct(H, W):
        return F.conv1d(H, W.flip(2), padding=W.shape[2] - 1)   # nmf.py:776-779

    def _check_target_shape(self, V):
        ok = (V.dim() == 3 and V.shape[0] == self.H.shape[0] and V.shape[1] == self.W.shape[0]
              and V.shape[2] == self.H.shape[2] + self.W.shape[2] - 1)
        if not ok:
            raise RuntimeError(f"target shape {tuple(V.shape)} does not match H {tuple(self.H.shape)} / "
                               f"W {tuple(self.W.shape)}")


# ---- what the fits share: factor registration (batched), placement, update step and stop rules -----------------------------

def _register_batched_factors(module, W, H, trainable_W, trainable_H):
    """Register W and H on a batched module (problems on axis 0, rank on axis 2): a Tensor is copied, an iterable of ints
    draws |randn| of that size, None registers None.  A factor without the class's `_ndim` axes, or W and H disagreeing on
    the rank or on the number of problems, raises ValueError.  Sets out_channels (and kernel_size, for a convolutive W)
    from W.  Returns (rank, number of problems) of the factors, None for each when neither is given."""
    rank = P = None
    for name, spec, trainable in (("W", W, trainable_W), ("H", H, trainable_H)):
        if isinstance(spec, Tensor):
            assert torch.all(spec >= 0.), f"Tensor {name} should be non-negative."
            p = Parameter(torch.empty(*spec.size()), requires_grad=trainable)
            p.data.copy_(spec)
        elif isinstance(spec, _Iterable):
            p = Parameter(torch.randn(*tuple(spec)).abs())
        else:
            p = None
        module.register_parameter(name, p)
        if p is not None:
            if p.dim() != module._ndim:
                raise ValueError(f"{name} must have {module._axes}; got shape {tuple(p.shape)}")
            if rank is not None and p.shape[2] != rank:
                raise ValueError("Latent size of H does not match with W")
            if P is not None and p.shape[0] != P:
                raise ValueError(f"W and H hold different numbers of problems ({P} and {p.shape[0]})")
            rank, P = p.shape[2], p.shape[0]
    if module.W is not None:
        module.out_channels = module.W.shape[1]
        if module.W.dim() > 3:
            module.kernel_size = module.W.shape[3:]
    return rank, P


@contextlib.contextmanager
def _placed_factors(module, factors, no_cuda, real=None):
    """Places a fit: yields (device, the fp32 contiguous tensors the engine updates, one per Parameter of
    `factors`).  They are the Parameters' own storages when every factor is fp32 and contiguous on a CUDA device, else
    device copies, written back into the Parameters when the block completes.  Without CUDA it raises
    RuntimeError(no_cuda).  With the `_engine_factory` test hook the storages are taken where they are.  `real` (a bool
    tensor over the leading axes of the second factor, or over all of them, or None): the cells of the second factor that
    are written back -- the real rows of a ragged BatchedNMF's H, the real positions of a ragged convolutive batch's H along
    its last axis; the others are left as they are (a ragged batch's padding)."""
    f32 = torch.float32
    if module._engine_factory is not None:
        dev, staged = factors[0].device, False
    else:
        if not torch.cuda.is_available():
            raise RuntimeError(no_cuda)
        on_gpu = factors[0].device.type == "cuda"
        dev = factors[0].device if on_gpu else torch.device("cuda", torch.cuda.current_device())
        staged = not (on_gpu and all(t.dtype == f32 and t.is_contiguous() for t in factors))
    placed = [t.data.to(dev, f32, non_blocking=True).contiguous() if staged else t.data for t in factors]
    yield dev, placed
    if staged:
        for i, (t, d) in enumerate(zip(factors, placed)):
            if i == 1 and real is not None:
                t.data[real.to(t.device)] = d[real.to(d.device)].to(t.device, t.dtype)
            else:
                t.data.copy_(d)


def _update_step(eng, cd, train_w, train_h, beta, gamma, l1_reg, l2_reg):
    """step(k) of `fit`: k iterations of the multiplicative updates (`cd`: of coordinate descent) of the trainable factors,
    W then H.  They run in one engine call when both factors train and the engine has it, else in one call per update."""
    fused = train_w and train_h and hasattr(eng, "cd_iterate" if cd else "iterate")

    def step(k):
        if fused and cd:
            eng.cd_iterate(k, l1_reg, l2_reg)
        elif fused:
            eng.iterate(k, beta, gamma, l1_reg, l2_reg)                                    # nmf.py:366-391, k times
        else:
            for _ in range(k):
                if train_w:
                    if cd:
                        eng.cd_update(0, l1_reg, l2_reg)
                    else:
                        eng.update_w(beta, gamma, l1_reg, l2_reg)                          # nmf.py:367-378
                if train_h:
                    if cd:
                        eng.cd_update(1, l1_reg, l2_reg)
                    else:
                        eng.update_h(beta, gamma, l1_reg, l2_reg)                          # nmf.py:380-391
    return step


def _fit_single(step, divergence, max_iter, tol, verbose):
    """The reference's stop rule (nmf.py:366-409, plca.py:245-302) for one problem: the loss sqrt(2 d) (NaN for d < 0) of
    the raw divergence d = `divergence(follows)` before the first iteration and after every 10th, stopping at the first
    check where (previous - loss) / initial < tol.  `follows` says whether iterations follow the check (False for the
    initial loss).  `step(k)` runs k iterations, at most 10 and never past a check.  Returns the last loop index: the
    iterations run, minus one."""
    def fit_loss(follows):
        d = divergence(follows)
        return math.sqrt(2.0 * d) if d >= 0 else float("nan")                              # nmf.py:362,402

    loss_init = previous = fit_loss(False)
    it = -1
    with _tqdm(total=max_iter, disable=not verbose) as pbar:
        while it + 1 < max_iter:
            k = min(10 - ((it + 1) % 10), max_iter - (it + 1))
            step(k)
            it += k
            if it % 10 == 9:                                                               # nmf.py:393
                loss = fit_loss(it + 1 < max_iter)
                pbar.set_postfix(loss=loss)
                pbar.update(10)
                if (previous - loss) / loss_init < tol:                                    # nmf.py:405
                    break
                previous = loss
    return it


def _fit_ard(eng, beta, gamma, divergence, max_iter, tol, verbose):
    """The loop of an ARD fit on `eng` (ARD registered): each iteration updates W, then H (the engine adds the penalties),
    then lambda -- one `iterate` call per run of iterations where the engine has it.  At every 10th iteration it stops when
    the largest relative change of lambda in that iteration is < tol (Tan and Fevotte's criterion), read from the engine
    there only.  With `verbose`, the progress bar shows the loss sqrt(2 d) of `divergence` at each check.  Returns the last
    loop index: the iterations run, minus one (`_fit_single`'s convention)."""
    fused = hasattr(eng, "iterate")

    def step(k):
        if fused:
            eng.iterate(k, beta, gamma, 0.0, 0.0)
            return
        for _ in range(k):
            eng.update_w(beta, gamma, 0.0, 0.0)
            eng.update_h(beta, gamma, 0.0, 0.0)
            eng.ard_update()

    it = -1
    with _tqdm(total=max_iter, disable=not verbose) as pbar:
        while it + 1 < max_iter:
            k = min(10 - ((it + 1) % 10), max_iter - (it + 1))
            step(k)
            it += k
            if it % 10 == 9:
                if verbose:
                    d = divergence(it + 1 < max_iter)
                    pbar.set_postfix(loss=math.sqrt(2.0 * d) if d >= 0 else float("nan"))
                pbar.update(10)
                if eng.ard_change() < tol:
                    break
    return it


def _fit_problems(eng, P, max_iter, tol, verbose, losses, step):
    """The reference's stop rule (nmf.py:366-409, plca.py:245-302) for each of P problems fitted together on `eng`: problem
    p's loss sqrt(2 d_p) (NaN for d_p < 0) from `losses()`, the P raw divergences, at the start and every 10th iteration,
    and it stops at the first check where (previous_p - loss_p) / init_p < tol; `eng.set_active` then freezes it while the
    others run on.  `step(k)` runs k iterations of every active problem, at most 10 and never past a check.  Returns the
    int64 iteration count of every problem: the iterations it ran, max_iter for one that never stopped."""
    def fit_losses():
        d = losses().to(torch.float64)
        return torch.where(d >= 0, torch.sqrt(2.0 * d.clamp(min=0)), float("nan"))

    loss_init = fit_losses()
    previous = loss_init.clone()
    n_iter = torch.full((P,), max_iter, dtype=torch.int64)
    active = torch.ones(P, dtype=torch.bool)
    it = -1
    with _tqdm(total=max_iter, disable=not verbose) as pbar:
        while it + 1 < max_iter and bool(active.any()):
            k = min(10 - ((it + 1) % 10), max_iter - (it + 1))
            step(k)
            it += k
            if it % 10 == 9:
                loss = fit_losses()
                stop = active & ((previous - loss) / loss_init < tol)
                n_iter[stop] = it + 1
                previous = torch.where(active & ~stop, loss, previous)
                pbar.set_postfix(active=int((active & ~stop).sum()))
                pbar.update(10)
                if bool(stop.any()):
                    active &= ~stop
                    eng.set_active(active)
    if hasattr(eng, "check_health"):
        eng.check_health()
    return n_iter


def _check_lengths(module, V, lengths, cd=False):
    """fit(..., lengths=L)'s checks for a batched module, before any device work: the lengths as a list of P Python ints in
    the module's `_length_range(V)`.  ValueError for a class without ragged fits (`_ragged` False), for `cd`, for a shared
    target (V without the problem axis), for lengths that are not a 1-D sequence or tensor of integers, and for a wrong
    count or a length out of range."""
    name = type(module).__name__
    if not module._ragged:
        raise ValueError(f"lengths is not supported by {name}")
    if cd:
        raise ValueError("lengths: solver='cd' does not fit ragged batches; use solver='mu'")
    B = module.H.shape[0]
    if V.dim() != module.H.dim():
        raise ValueError(f"lengths needs one target per problem, V with a leading axis of {B} problems; a shared "
                         f"target of shape {tuple(V.shape)} has one length")
    if isinstance(lengths, Tensor):
        if lengths.dtype.is_floating_point or lengths.dtype.is_complex or lengths.dtype == torch.bool:
            raise ValueError(f"lengths must hold integers (got {lengths.dtype})")
        if lengths.dim() != 1:
            raise ValueError(f"lengths must be 1-D (got shape {tuple(lengths.shape)})")
        lens = [int(n) for n in lengths.tolist()]
    elif isinstance(lengths, _Iterable) and not isinstance(lengths, (str, bytes)):
        lens = list(lengths)
        if not all(isinstance(n, numbers.Integral) and not isinstance(n, bool) for n in lens):
            raise ValueError("lengths must be a sequence of ints or an integer tensor")
        lens = [int(n) for n in lens]
    else:
        raise ValueError(f"lengths must be a sequence of ints or an integer tensor (got {type(lengths).__name__})")
    if len(lens) != B:
        raise ValueError(f"lengths holds {len(lens)} values for {B} problems")
    lo, hi, hi_name = module._length_range(V)
    bad = [n for n in lens if not lo <= n <= hi]
    if bad:
        raise ValueError(f"every length must be in [{lo}, {hi_name} = {hi}] (got {bad[0]})")
    return lens


class _BatchedComponent(BaseComponent):
    """Shared part of the batched classes: P independent problems of one model and one shape, fitted together.  W and H
    hold the problems on their leading axis and the rank on axis 2; problem p's factors W[p] / H[p] are those of the
    single model.  `fit` runs every problem on the fp32 CUDA-core kernels in the launches one problem takes, each with its
    own stop rule."""
    _ndim = 3                      # axes of W and of H
    _axes = "three axes (B, rows, rank)"
    _ragged = False                # fit(..., lengths=L): BatchedNMF and the convolutive batched models

    def __init__(self, rank=None, W=None, H=None, trainable_W=True, trainable_H=True):
        torch.nn.Module.__init__(self)
        inferred, _ = _register_batched_factors(self, W, H, trainable_W, trainable_H)
        if inferred is None:
            assert rank, "A rank should be given when W and H are not available!"
        else:
            rank = inferred
        self.rank = rank

    def _readable_in_place(self, Vd):
        """Whether the engine reads this device target (fp32, fp16 or bf16) as it is laid out."""
        raise NotImplementedError

    def sparse_fit(self, *args, **kwargs):
        raise NotImplementedError(f"{type(self).__name__} has no sparse_fit: fit each problem with the single model's sparse_fit")

    def _length_range(self, V):
        """(lo, hi, name of hi) of the lengths of a ragged fit: rows of H in [1, N]."""
        return 1, self.H.shape[1], "N"

    @torch.no_grad()
    def fit(self, V, beta=1, tol=1e-4, max_iter=200, verbose=False, alpha=0, l1_ratio=0, *, precision="auto", solver="mu",
            lengths=None):
        """Fit every problem by multiplicative updates, as the single model's `fit(V[p], ...)` fits one, all of them in the
        same launches.

        V: the problems' targets stacked on a leading axis, or one target of the single model's shape shared by every
        problem (random restarts of one fit).  Dense float32, float16 or bfloat16, read in place where the class's layout
        allows it (an expanded shared target is read once); float64 and other layouts are staged through one fp32 (or
        same-dtype contiguous) copy on the device.  A sparse V raises NotImplementedError.

        Returns a torch.int64 tensor of P iteration counts.  Problem p follows the reference's stop rule (nmf.py:366-409) on
        its own: its loss sqrt(2 d_p) at the start and every 10th iteration, and it stops at the first check where
        (previous_p - loss_p) / init_p < tol; from then on every kernel leaves its factors untouched while the others run
        on.  n_iter[p], W[p] and H[p] equal, bit for bit, those of the single model's
        `fit(V[p], ..., precision="f32")` from W0[p] / H0[p]: each problem keeps the single fit's tile plan and summation
        order.  The losses cost one synchronisation per 10 iterations for the whole batch.

        Every beta, `alpha` / `l1_ratio` and frozen factors (trainable_W / trainable_H) are supported, for 1 <= R <= 256,
        on the fp32 CUDA-core kernels: precision "auto" and "f32" run them (`last_fit_precision` is "f32"); "f16" and
        "f16_split" raise ValueError, as do R > 256 and shape mismatches.  Validation is the reference's over every problem:
        a negative V fails its assertion, and beta <= 0 with a zero anywhere in V raises ValueError.  `mask`, `weight` and
        `group` are not parameters of this method (TypeError).  Host or half-precision modules are staged through fp32
        device copies and written back, as by the single model's `fit`.  The workspace is P times one fp32 problem's (see
        the class).

        solver: "mu" (default) -- the multiplicative updates above -- or, BatchedNMF only, "cd": coordinate descent (HALS)
        at beta 2, each problem fitted as `NMF.fit(V[p], 2, ..., precision="f32", solver="cd")` fits it (see `NMF.fit`),
        bit for bit, with the same per-problem stop rule.  The iterations between two loss checks run in one call when both
        factors train; a frozen factor leaves the other's updates one call each.  ValueError, before any device work: an
        unknown solver, "cd" with beta != 2, and "cd" on the convolutive batched models.

        lengths: (keyword-only, default None) one int per problem, as a sequence or an integer tensor of shape (P,) on
        any device: a ragged batch.  BatchedNMF: B ints in [1, N], problem b being the fit of V[b, :lengths[b]] with W[b]
        and H[b, :lengths[b]]; V (B, N, C) and H (B, N, R) stay padded, and n_iter[b], W[b] and H[b, :L_b] equal, bit for
        bit, those of `NMF(W=W0[b], H=H0[b, :L_b]).fit(V[b, :L_b], ..., precision="f32")`.  BatchedNMFD / 2D / 3D: P ints
        in [K_last, X_last] (W's and V's last sizes) along the last convolved axis, problem p being the fit of
        V[p, ..., :L_p] with W[p] and H[p, ..., :L_p - K_last + 1]; V (P, B, C, *X) and H (P, B, R, *(X - K + 1)) stay
        padded, and n_iter[p], W[p] and those positions of H[p] equal, bit for bit, those of the single model's
        `(W=W0[p], H=H0[p, ..., :L_p - K_last + 1]).fit(V[p, ..., :L_p], ..., precision="f32")`; its B clips share W[p]
        and L_p.  The stop rule is included: each problem runs the tile plan of its own length.  The padding of V is never
        read (NaN there does not reach the fit) and that of H never written, even through a staged host or float64
        module; the non-negativity assertion and the beta <= 0 zero check look at the real cells only.  Every beta,
        alpha / l1_ratio, frozen factors, fp16 / bf16 (and, for BatchedNMF, strided) targets and host or float64 modules
        work as without it; lengths all at their maximum give the bits of lengths=None.  The workspace is the sum of the
        problems' single-problem workspaces.  ValueError, before any device work: the wrong number of lengths, a length
        out of range, a non-integer, bool or non-1-D lengths, a shared target (no problem axis), and solver="cd".
        """
        name = type(self).__name__
        if solver not in ("mu", "cd"):
            raise ValueError(f"solver must be 'mu' or 'cd' (got {solver!r})")
        cd = solver == "cd"
        if lengths is not None:
            assert self.W is not None and self.H is not None, "fit() needs both W and H"
            lengths = _check_lengths(self, V, lengths, cd)
        if cd:
            if not self._cd_solver:
                raise ValueError(f"solver='cd' is supported by BatchedNMF only (got {name})")
            if beta != 2:
                raise ValueError(f"solver='cd' minimises the beta = 2 objective; beta must be 2 (got {beta!r})")
        if precision not in ("auto", "f32"):
            if precision in ("f16", "f16_split"):
                raise ValueError(f"{name} runs on the fp32 kernels: precision must be 'auto' or 'f32' (got {precision!r})")
            raise ValueError(f"unknown precision {precision!r}")
        if V.is_sparse:
            raise NotImplementedError(f"{name} takes dense targets only")
        W, H = self.W, self.H
        assert W is not None and H is not None, "fit() needs both W and H"
        if W.shape[2] > 256:
            raise ValueError(f"{name} supports rank <= 256 (got {W.shape[2]})")
        self._check_target_shape(V)

        real = None                # a ragged batch: the real cells of H, the only ones written back from a staged copy
        if lengths is not None:
            real = self._real_cells(lengths)
        ragged = {} if lengths is None else {"lengths": lengths}
        with _placed_factors(self, (W, H), _NO_CUDA, real) as (dev, (Wd, Hd)):
            if self._engine_factory is None:
                Vd = V.to(dev, non_blocking=True)
                if Vd.dtype not in (torch.float32, torch.float16, torch.bfloat16):
                    Vd = Vd.to(torch.float32)
                if not self._readable_in_place(Vd):
                    Vd = Vd.contiguous()
                eng = self._engine_cls(Vd, Wd, Hd, **ragged)
            else:
                eng = self._engine_factory(V, Wd, Hd, **ragged)
            try:
                vmin, vmax = eng.minmax()
                assert vmin >= 0., "Target should be non-negative."                        # nmf.py:329-330
                if vmin == 0 and beta <= 0:                                                # nmf.py:332-336
                    raise ValueError("When beta <= 0 and V contains zeros, the training process may diverge. "
                                     "Please add small values to V, or use a positive beta value.")
                gamma = _gamma(beta)
                l1_reg = alpha * l1_ratio                                                  # nmf.py:348
                l2_reg = alpha * (1 - l1_ratio)                                            # nmf.py:349
                step = _update_step(eng, cd, W.requires_grad, H.requires_grad, beta, gamma, l1_reg, l2_reg)
                n_iter = _fit_problems(eng, W.shape[0], max_iter, tol, verbose, lambda: eng.losses(beta), step)
                self.last_fit_precision = "f32"
            finally:
                eng.close()
        return n_iter


class BatchedNMF(_BatchedComponent):
    """B independent NMF problems of one shape:  V[b] (N,C) ~= H[b] (N,R) @ W[b] (C,R)^T,  W (B,C,R), H (B,N,R).

    Args:
        Vshape: (B, N, C); W and H are then drawn as `NMF` draws them, |randn| of (B, C, rank) and (B, N, rank)
        rank: size of the hidden dimension (default: C); the last axis of W and H
        W / H: a size (iterable of ints -> random non-negative init) or an initial non-negative Tensor
        trainable_W / trainable_H: whether a *given tensor* is updated by `fit`

    `fit(V, ...)` takes V as (B, N, C), or as one (N, C) target shared by every problem; its columns must have unit stride
    to be read in place (rows and problems may be strided).  Each problem's fit is `NMF.fit(V[b], ..., precision="f32")`.
    Workspace (device memory, kept between fits of the same shape like `NMF.fit`'s): B times that of one fp32 NMF problem
    -- the chunked partial numerators and denominators, 8 R max(nch_w C, nch_h N) bytes with up to 32 chunks per
    contraction (`_capi.nmf_plan(N, C, R)`), plus the column sums and loss partials -- so it grows linearly with B.
    `fit(..., lengths=L)` fits a ragged batch: problem b is `NMF.fit(V[b, :L[b]], ..., precision="f32")` with W[b] and
    H[b, :L[b]], V and H padded to N rows, each problem on the tile plan of its own length (see `fit`); its workspace is the
    sum over the problems of one fp32 problem's of L[b] rows, not B times the largest.
    `fit(..., solver="cd")` fits each problem by coordinate descent (HALS) at beta 2, as `NMF.fit(V[b], 2, ...,
    precision="f32", solver="cd")`; it adds the Gram scratch, allocated at the first such fit, of 4 B (2 R^2 + max(nb(N),
    nb(C)) R^2) bytes, nb(rows) = ceil(rows / rpb) <= 128 Gram blocks of rpb = roundup(ceil(rows / 128), 32) rows
    (include/nmf_b200.h: nmfb200_nmf_sparse_plan).
    """
    _engine_cls = _engine.CudaBatchedNmfEngine
    _cd_solver = True
    _ragged = True

    def __init__(self, Vshape=None, rank=None, *, W=None, H=None, trainable_W=True, trainable_H=True):
        if isinstance(Vshape, _Iterable):
            B, N, C = Vshape
            rank = rank if rank else C
            W = (B, C, rank) if W is None else W
            H = (B, N, rank) if H is None else H
        super().__init__(rank, W, H, trainable_W, trainable_H)

    @staticmethod
    def reconstruct(H, W):
        return H @ W.transpose(-1, -2)

    def _check_target_shape(self, V):
        B, N, _ = self.H.shape
        C = self.W.shape[1]
        if tuple(V.shape) not in ((B, N, C), (N, C)):
            raise ValueError(f"target shape {tuple(V.shape)} does not match H {tuple(self.H.shape)} / W {tuple(self.W.shape)}: "
                             f"expected ({B}, {N}, {C}) or ({N}, {C})")

    def _readable_in_place(self, Vd):
        rows_ok = Vd.stride(-1) == 1 and Vd.stride(-2) >= Vd.shape[-1]
        return rows_ok and (Vd.dim() == 2 or Vd.stride(0) == 0 or Vd.stride(0) >= Vd.shape[1] * Vd.stride(1))

    def _real_cells(self, lengths):
        """The real rows of H, a bool (B, N) tensor."""
        return torch.arange(self.H.shape[1]) < torch.tensor(lengths).unsqueeze(1)


def _batched_conv(H, W, conv):
    """The reconstructions of P convolutive problems at once: problem p's H[p] (B,R,*J) convolved with its flipped W[p]
    (C,R,*K), full padding, as one grouped convolution; (P,B,C,*X)."""
    P, B, R = H.shape[:3]
    C, K = W.shape[1], W.shape[3:]
    x = H.transpose(0, 1).reshape(B, P * R, *H.shape[3:])
    w = W.flip(tuple(range(3, W.dim()))).reshape(P * C, R, *K)
    out = conv(x, w, padding=tuple(k - 1 for k in K), groups=P)
    return out.reshape(B, P, C, *out.shape[2:]).transpose(0, 1)


class _BatchedConvolutive(_BatchedComponent):
    """Shared part of BatchedNMFD / BatchedNMF2D / BatchedNMF3D: P independent problems of the single model over `_nd`
    convolved axes, V (P,B,C,*X), W (P,C,R,*K), H (P,B,R,*(X-K+1)); each problem's B clips share its W[p].

    `fit(V, ...)` takes V as (P, B, C, *X), or as one (B, C, *X) target shared by every problem.  It is read in place when
    every problem's block is contiguous and the blocks are at least B C prod(X) elements apart (or 0: an expanded shared
    target).  Workspace (device memory, kept between fits of the same shape): P times that of one fp32 problem of the
    single model -- the ratio tile of V's size (two at beta != 1), the wgrad / dgrad split partial slabs, 8 R max(nsw C
    prod(K), nsd B prod(X-K+1)) bytes with the splits of `_capi.nmfd_plan`, plus the column sums and loss partials -- so
    it grows linearly with P.  `fit(..., lengths=L)` fits a ragged batch along the last convolved axis: problem p is the
    single model's `fit(V[p, ..., :L[p]], ..., precision="f32")` with W[p] and H[p, ..., :L[p] - K_last + 1], V and H
    padded, each problem on the plan of its own length; its workspace is the sum of the problems' single-problem
    workspaces, not P times the largest."""
    _engine_cls = _engine.CudaBatchedNmfdEngine
    _ragged = True
    _nd = 1
    _conv = None

    @classmethod
    def reconstruct(cls, H, W):
        return _batched_conv(H, W, cls._conv)

    def _check_target_shape(self, V):
        P, B = self.H.shape[:2]
        C, K, J = self.W.shape[1], self.W.shape[3:], self.H.shape[3:]
        single = (B, C) + tuple(j + k - 1 for j, k in zip(J, K))
        if tuple(V.shape) not in ((P,) + single, single):
            raise ValueError(f"target shape {tuple(V.shape)} does not match H {tuple(self.H.shape)} / W {tuple(self.W.shape)}: "
                             f"expected {(P,) + single} or {single}")

    def _readable_in_place(self, Vd):
        if Vd.dim() == self._nd + 2:
            return Vd.is_contiguous()
        return Vd[0].is_contiguous() and (Vd.stride(0) == 0 or Vd.stride(0) >= Vd[0].numel())

    def _length_range(self, V):
        """A ragged fit's lengths run along the last convolved axis, from W's last size to V's."""
        return self.W.shape[-1], V.shape[-1], "X_last"

    def _real_cells(self, lengths):
        """The real cells of H (P, B, R, *J): positions below L_p - K_last + 1 of its last axis, a bool tensor of H's
        shape."""
        H = self.H
        lin = torch.tensor(lengths) - self.W.shape[-1] + 1
        real = torch.arange(H.shape[-1]) < lin.view(-1, *([1] * (H.dim() - 1)))
        return real.expand(H.shape)


class BatchedNMFD(_BatchedConvolutive):
    """P independent NMFD problems of one shape:  V[p] (B,C,L) ~= sum_t W[p][:,:,t] @ shift_t(H[p]),  W (P,C,R,T),
    H (P,B,R,L-T+1).  Problem p is `NMFD(W=W[p], H=H[p])`; its B clips share W[p].

    Args:
        Vshape: (P, B, C, L); W and H are then drawn as `NMFD` draws them, |randn| of (P, C, rank, T) and (P, B, rank, L-T+1)
        rank: size of the hidden dimension (default: C)
        T: the kernel's length (an int or a 1-tuple)
        W / H: a size (iterable of ints -> random non-negative init) or an initial non-negative Tensor
        trainable_W / trainable_H: whether a *given tensor* is updated by `fit`

    `fit(V, ...)` takes V as (P, B, C, *X), or as one (B, C, *X) target shared by every problem.  It is read in place when
    every problem's block is contiguous and the blocks are at least B C prod(X) elements apart (or 0: an expanded shared
    target).  Workspace (device memory, kept between fits of the same shape): P times that of one fp32 problem of the
    single model -- the ratio tile of V's size (two at beta != 1), the wgrad / dgrad split partial slabs, 8 R max(nsw C
    prod(K), nsd B prod(X-K+1)) bytes with the splits of `_capi.nmfd_plan`, plus the column sums and loss partials -- so
    it grows linearly with P.  `fit(..., lengths=L)` fits problems of different lengths along the clips' length L (the last axis),
    each bit for bit its own single fit on its real positions (see `fit`).
    """
    _nd = 1
    _ndim = 4
    _axes = "four axes (P, rows, rank, T)"
    _conv = staticmethod(F.conv1d)

    def __init__(self, Vshape=None, rank=None, T=1, *, W=None, H=None, trainable_W=True, trainable_H=True):
        if isinstance(Vshape, _Iterable):
            if isinstance(T, _Iterable):
                T, = T
            P, B, C, L = Vshape
            rank = rank if rank else C
            W = (P, C, rank, T) if W is None else W
            H = (P, B, rank, L - T + 1) if H is None else H
        super().__init__(rank, W, H, trainable_W, trainable_H)


class BatchedNMF2D(_BatchedConvolutive):
    """P independent NMF2D problems of one shape:  V[p] (B,C,X1,X2) ~= conv2d(H[p], flipped W[p], full padding),
    W (P,C,R,k1,k2), H (P,B,R,X1-k1+1,X2-k2+1).  Problem p is `NMF2D(W=W[p], H=H[p])`; its B clips share W[p].

    Args:
        Vshape: (P, B, C, X1, X2); W and H are then drawn as `NMF2D` draws them (rank defaults to X1, as there)
        rank: size of the hidden dimension
        kernel_size: (k1, k2), or one int for both
        W / H: a size (iterable of ints -> random non-negative init) or an initial non-negative Tensor
        trainable_W / trainable_H: whether a *given tensor* is updated by `fit`

    `fit(V, ...)` takes V as (P, B, C, *X), or as one (B, C, *X) target shared by every problem.  It is read in place when
    every problem's block is contiguous and the blocks are at least B C prod(X) elements apart (or 0: an expanded shared
    target).  Workspace (device memory, kept between fits of the same shape): P times that of one fp32 problem of the
    single model -- the ratio tile of V's size (two at beta != 1), the wgrad / dgrad split partial slabs, 8 R max(nsw C
    prod(K), nsd B prod(X-K+1)) bytes with the splits of `_capi.nmfd_plan`, plus the column sums and loss partials -- so
    it grows linearly with P.  `fit(..., lengths=L)` fits problems of different lengths along X2 (the last axis),
    each bit for bit its own single fit on its real positions (see `fit`).
    """
    _nd = 2
    _ndim = 5
    _axes = "five axes (P, rows, rank, k1, k2)"
    _conv = staticmethod(F.conv2d)

    def __init__(self, Vshape=None, rank=None, kernel_size=1, *, W=None, H=None, trainable_W=True, trainable_H=True):
        if isinstance(Vshape, _Iterable):
            kernel_size = _ntuple(kernel_size, 2)
            k1, k2 = kernel_size
            P, B, C, X1, X2 = Vshape
            rank = rank if rank else X1
            W = (P, C, rank) + kernel_size if W is None else W
            H = (P, B, rank, X1 - k1 + 1, X2 - k2 + 1) if H is None else H
        super().__init__(rank, W, H, trainable_W, trainable_H)


class BatchedNMF3D(_BatchedConvolutive):
    """P independent NMF3D problems of one shape:  V[p] (B,C,X1,X2,X3) ~= conv3d(H[p], flipped W[p], full padding),
    W (P,C,R,k1,k2,k3), H (P,B,R,X1-k1+1,X2-k2+1,X3-k3+1).  Problem p is `NMF3D(W=W[p], H=H[p])`; its B clips share W[p].

    Args:
        Vshape: (P, B, C, X1, X2, X3); W and H are then drawn as `NMF3D` draws them (rank defaults to X2, as there)
        rank: size of the hidden dimension
        kernel_size: (k1, k2, k3), or one int for all three
        W / H: a size (iterable of ints -> random non-negative init) or an initial non-negative Tensor
        trainable_W / trainable_H: whether a *given tensor* is updated by `fit`

    `fit(V, ...)` takes V as (P, B, C, *X), or as one (B, C, *X) target shared by every problem.  It is read in place when
    every problem's block is contiguous and the blocks are at least B C prod(X) elements apart (or 0: an expanded shared
    target).  Workspace (device memory, kept between fits of the same shape): P times that of one fp32 problem of the
    single model -- the ratio tile of V's size (two at beta != 1), the wgrad / dgrad split partial slabs, 8 R max(nsw C
    prod(K), nsd B prod(X-K+1)) bytes with the splits of `_capi.nmfd_plan`, plus the column sums and loss partials -- so
    it grows linearly with P.  `fit(..., lengths=L)` fits problems of different lengths along X3 (the last axis),
    each bit for bit its own single fit on its real positions (see `fit`).
    """
    _nd = 3
    _ndim = 6
    _axes = "six axes (P, rows, rank, k1, k2, k3)"
    _conv = staticmethod(F.conv3d)

    def __init__(self, Vshape=None, rank=None, kernel_size=1, *, W=None, H=None, trainable_W=True, trainable_H=True):
        if isinstance(Vshape, _Iterable):
            kernel_size = _ntuple(kernel_size, 3)
            k1, k2, k3 = kernel_size
            P, B, C, X1, X2, X3 = Vshape
            rank = rank if rank else X2
            W = (P, C, rank) + kernel_size if W is None else W
            H = (P, B, rank, X1 - k1 + 1, X2 - k2 + 1, X3 - k3 + 1) if H is None else H
        super().__init__(rank, W, H, trainable_W, trainable_H)


def _ntuple(x, n):
    """torch.nn.modules.utils._pair / _triple: an int repeats, an iterable is taken as is."""
    return tuple(x) if isinstance(x, _Iterable) else (x,) * n


class _NMFnD(BaseComponent):
    """Shared part of NMF2D / NMF3D: V (B,C,*X) ~= sum over the kernel offsets t of W[:,:,t] @ shift_t(H),
    W (C,R,*kernel_size), H (B,R,*(X - kernel_size + 1)).  `fit` runs the same three sliding contractions as NMFD with the
    last axis sliding and the outer axes as loops (csrc/nmfd.cu), in fp32, for every beta."""
    _engine_cls = _engine.CudaNmfdEngine
    _nd = 0

    def _check_target_shape(self, V):
        nd = self._nd
        ok = (V.dim() == nd + 2 and V.shape[0] == self.H.shape[0] and V.shape[1] == self.W.shape[0]
              and all(V.shape[2 + i] == self.H.shape[2 + i] + self.W.shape[2 + i] - 1 for i in range(nd)))
        if not ok:
            raise RuntimeError(f"target shape {tuple(V.shape)} does not match H {tuple(self.H.shape)} / "
                               f"W {tuple(self.W.shape)}")


class NMF2D(_NMFnD):
    """Non-negative matrix factor 2-D deconvolution (reference: nmf.py:782-865).

    V (B,C,L,M) ~= conv2d(H, flipped W, full padding),  W (C,R,k0,k1),  H (B,R,L-k0+1,M-k1+1).
    """
    _nd = 2

    def __init__(self, Vshape=None, rank=None, kernel_size=1, **kwargs):
        if isinstance(Vshape, _Iterable):
            kernel_size = _ntuple(kernel_size, 2)
            kh, kw = kernel_size
            batch, channel, K, M = Vshape                  # wrong arity raises, as in the reference (:852)
            rank = rank if rank else K
            kwargs["W"] = (channel, rank) + kernel_size
            kwargs["H"] = (batch, rank, K - kh + 1, M - kw + 1)
        super().__init__(rank, **kwargs)

    @staticmethod
    def reconstruct(H, W):
        return F.conv2d(H, W.flip((2, 3)), padding=(W.shape[2] - 1, W.shape[3] - 1))          # nmf.py:861-865


class NMF3D(_NMFnD):
    """Non-negative matrix factor 3-D deconvolution (reference: nmf.py:868-942).

    V (B,C,N,K,M) ~= conv3d(H, flipped W, full padding),  W (C,R,k0,k1,k2),  H (B,R,N-k0+1,K-k1+1,M-k2+1).
    """
    _nd = 3

    def __init__(self, Vshape=None, rank=None, kernel_size=1, **kwargs):
        if isinstance(Vshape, _Iterable):
            kernel_size = _ntuple(kernel_size, 3)
            kd, kh, kw = kernel_size
            batch, channel, N, K, M = Vshape               # wrong arity raises, as in the reference (:928)
            rank = rank if rank else K
            kwargs["W"] = (channel, rank) + kernel_size
            kwargs["H"] = (batch, rank, N - kd + 1, K - kh + 1, M - kw + 1)
        super().__init__(rank, **kwargs)

    @staticmethod
    def reconstruct(H, W):
        pad = (W.shape[2] - 1, W.shape[3] - 1, W.shape[4] - 1)
        return F.conv3d(H, W.flip((2, 3, 4)), padding=pad)                                     # nmf.py:938-942


# module types whose plain reconstruction trainer.BetaMu may replace by the fused kernels (exact types: a subclass with its
# own `reconstruct` is a different model)
_BETAMU_FUSABLE = frozenset({NMF, NMFD, NMF2D, NMF3D})
