"""Host-side engines: thin owners of an ``nmfb200_ctx`` plus the sharded W update.

An engine exposes exactly the operations ``BaseComponent.fit`` (nmf.py:366-407 in the reference)
needs from its loop body:

    minmax() -> (vmin, vmax)       fit()'s validation, nmf.py:329-336
    update_w / update_h            nmf.py:367-391
    loss(beta) -> float            metrics.beta_div of the current reconstruction, nmf.py:360-361,:400-401

`ShardedEngine` wraps any engine that also offers ``w_partial`` / ``w_apply`` / ``loss_tensor`` and
inserts the one collective per iteration that the row-sharded layout needs.  Its base, `Collectives`, holds the
collectives themselves; the sharded PLCA fits (plca.py) call them around unwrapped engines.
"""
import ctypes
import os

import torch

from . import _capi


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr())


def _stream(device):
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _device_index(device):
    """The CUDA ordinal the library is given for `device` (a bare "cuda": the current device)."""
    return device.index if device.index is not None else torch.cuda.current_device()


def _check_f32_cuda(t, name, device):
    if t.dtype != torch.float32:
        raise TypeError(f"{name} must be float32 (got {t.dtype}); the engine mirrors the reference's default dtype")
    if t.device != device:
        raise ValueError(f"{name} is on {t.device}, expected {device}")
    if not t.is_contiguous():
        raise ValueError(f"{name} must be contiguous")


def _check_target(V, device, strided_rows=False):
    """A dense target as the kernels read it: fp32, fp16 or bf16 (converted exactly where each element is loaded, so a
    half-precision V gives the results of V.float() without an fp32 copy) on the engine's device, contiguous -- or, for
    `strided_rows` (NMF), rows of unit column stride at a row stride >= the column count."""
    if V.dtype not in _capi.DTYPES:
        raise TypeError(f"V must be float32, float16 or bfloat16 (got {V.dtype})")
    if V.device != device:
        raise ValueError(f"V is on {V.device}, expected {device}")
    if not (V.is_contiguous() or (strided_rows and V.stride(1) == 1 and V.stride(0) >= V.shape[1])):
        raise ValueError("V must be contiguous" + (" or have unit column stride" if strided_rows else ""))


# Engine workspaces (the fp16 operand copies of V are the size of V) are kept across fit() calls of the same
# shape instead of being cudaMalloc'ed / cudaFree'd every time.  The memory is cudaMalloc'ed by the library, i.e. invisible
# to torch's caching allocator, so the cache is bounded by BYTES (estimated from the shapes): at most
# NMFB200_WORKSPACE_CACHE_MB (default 8192; 0 disables caching) are held between fits, in at most _MAX_WORKSPACES
# contexts.  release_workspaces() drops them all.
_WORKSPACES = {}
_MAX_WORKSPACES = 2
_CACHE_BYTES = int(float(os.environ.get("NMFB200_WORKSPACE_CACHE_MB", "8192")) * (1 << 20))


def _workspace_bytes(key):
    """Upper estimate of the device memory a cached context of this key holds."""
    if key[0] == "nmf":                   # ("nmf", device, N, C, R, precision): V16 + Vt16 + split partials + fp32 scratch
        _, _, N, C, R = key[:5]
        est = 4 * N * C + 64 * (N + C) * max(R, 64)
        if R > 256:                       # fp32 only: the chunked num / den partial slabs of the larger update
            p = _capi.nmf_plan(N, C, R)
            est += 8 * R * max(p["nch_w"] * C, p["nch_h"] * N)
        return est
    if key[0] == "nmf_batched":           # ("nmf_batched", device, B, N, C, R[, lengths]): B x the fp32 context of one problem
        _, _, B, N, C, R = key[:6]        # with the lengths of a ragged batch: the sum of each problem's own context

        def one(n):
            p = _capi.nmf_plan(n, C, R)
            return (8 * R * max(p["nch_w"] * C, p["nch_h"] * n) + 8 * R + 8 * p["loss_chunks"] * ((n + 63) // 64)
                    + 4 * R * max(p["colsum_blocks_n"], p["colsum_blocks_c"]))
        if len(key) > 6:
            return sum(one(n) for n in key[6]) + 88 * B + (1 << 14)
        return B * one(N) + (1 << 14)
    if key[0] == "nmfd_batched":          # ("nmfd_batched", device, P, B, C, X, R, K[, lengths]): P x the fp32 context of one
        _, _, P, B, C, X, R, K = key[:8]  # problem; with the lengths of a ragged batch the sum of each problem's own context

        def colsum_floats(outer, inner):      # update.cu: colsum_scratch_floats
            return R * (outer if inner > 1 else min(1024, max(1, (outer + 63) // 64)))

        def one(X):
            nx, nk, nh = 1, 1, 1
            for x, k in zip(X, K):
                nx, nk, nh = nx * x, nk * k, nh * (x - k + 1)
            p = _capi.nmfd_plan(B, C, X, R, K)
            loss_blocks = p["recon_grid"][0] * p["recon_grid"][1] * B
            return (8 * B * C * nx + 8 * R * max(p["wgrad_nsplit"] * C * nk, p["dgrad_nsplit"] * B * nh) + 8 * R
                    + 8 * loss_blocks + 4 * max(colsum_floats(C, nk), colsum_floats(B, nh)))
        if len(key) > 8:
            return sum(one(tuple(X[:-1]) + (n,)) for n in key[8]) + 96 * P + (1 << 14)
        return P * one(X) + (1 << 14)
    if key[0] == "nmfd":                  # ("nmfd", device, B, C, X, R, K, precision): ratio tiles + shifted operand copies
        _, _, B, C, X, R, K = key[:7]
        nx, nk = 1, 1
        for x in X:
            nx *= x
        for k in K:
            nk *= k
        est = 12 * B * C * nx + 64 * C * R * nk + 64 * B * R * nx
        if len(X) > 1 and key[7] == "f16":   # NMF2D / NMF3D fp16 copies: ratio tile lines, W (twice), H lines
            p = _capi.nmfnd_tc_plan(B, C, X, R, K)
            lines, klines, hlines = nx // X[-1], nk // K[-1], B * R
            for x, k in zip(X[:-1], K[:-1]):
                hlines *= x - k + 1
            est += 2 * p["Lq"] * B * C * lines + 4 * p["Cpad"] * R * klines * p["Tp"] + 2 * p["Lp"] * hlines
        return est
    return 0


def cached_workspace_bytes():
    """Estimated device memory currently parked in the workspace cache."""
    return sum(_workspace_bytes(k) for k in _WORKSPACES)



def hoyer_project_(x, dim, k1, k2):
    """Project every slice of `x` along `dim` onto {v >= 0, |v|_1 = k1[j], |v|_2^2 = k2[j]} IN PLACE: ONE launch of
    `nmfb200_hoyer_project` (include/nmf_b200.h) for what the reference does with a Python loop over the slices around
    `_proj_func` (nmf.py:21-49, :519-522; trainer.py:176-181).  x: contiguous fp32 CUDA tensor; k1 / k2: sequences or
    tensors of x.shape[dim] values (device tensors are used as they are: no host synchronisation)."""
    if not (isinstance(x, torch.Tensor) and x.is_cuda):
        raise TypeError("hoyer_project_: x must be a CUDA tensor (the library has no CPU path)")
    if x.dtype != torch.float32 or not x.is_contiguous():
        raise TypeError("hoyer_project_: x must be a contiguous float32 tensor")
    D = x.shape[dim]
    outer = 1
    for n in x.shape[:dim]:
        outer *= n
    inner = x.numel() // max(outer * D, 1)
    if x.numel() == 0:
        return x
    k1 = torch.as_tensor(k1, dtype=torch.float32, device=x.device).contiguous()
    k2 = torch.as_tensor(k2, dtype=torch.float32, device=x.device).contiguous()
    assert k1.numel() == D and k2.numel() == D
    zeroed = torch.empty(x.numel(), dtype=torch.uint8, device=x.device)
    lib = _capi.load()
    _capi.check(lib.nmfb200_hoyer_project(_device_index(x.device), _ptr(x), outer, D, inner, _ptr(k1), _ptr(k2), _ptr(zeroed),
                                          _stream(x.device)))
    return x


def release_workspaces():
    """Free every cached engine workspace (device memory held between fit() calls)."""
    lib = _capi.load()
    for ctx in _WORKSPACES.values():
        lib.nmfb200_destroy(ctx)
    _WORKSPACES.clear()


class _CudaEngine:
    kind = None

    def __init__(self):
        self._lib = _capi.load()
        self._ctx = ctypes.c_void_p()
        self._loss = None
        self._key = None
        self._wbuf = None
        self._mask = None
        self._weight = None

    def _acquire(self, key, create):
        """Take a cached context for `key` or create one with `create(ctx_ref)`."""
        self._key = key
        ctx = _WORKSPACES.pop(key, None)
        if ctx is not None:
            self._ctx = ctx
            return
        _capi.check(create(ctypes.byref(self._ctx)))

    def close(self):
        if self._ctx:
            mine = _workspace_bytes(self._key) if self._key is not None else 0
            if self._key is not None and mine <= _CACHE_BYTES:
                while _WORKSPACES and (len(_WORKSPACES) >= _MAX_WORKSPACES
                                       or cached_workspace_bytes() + mine > _CACHE_BYTES):
                    old = _WORKSPACES.pop(next(iter(_WORKSPACES)))
                    self._lib.nmfb200_destroy(old)
                _WORKSPACES[self._key] = self._ctx
            else:
                self._lib.nmfb200_destroy(self._ctx)
            self._ctx = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def precision(self):
        return _capi.PRECISION_NAMES[self._lib.nmfb200_precision(self._ctx)]

    def precision_for(self, beta):
        """Arithmetic the contraction kernels use for this beta ("f32" when the tensor-core path does not cover it)."""
        return _capi.PRECISION_NAMES[self._lib.nmfb200_precision_for_beta(self._ctx, float(beta))]

    def set_mask(self, M):
        """Fit only the observed cells of V from now on (include/nmf_b200.h: nmfb200_set_mask): M is a contiguous bool or
        uint8 tensor of V's shape on the engine's device, read in place (True = observed); None clears the mask.  The engine
        keeps a reference to M while it is set.  minmax() then covers the observed cells only."""
        if M is not None:
            if M.dtype not in (torch.bool, torch.uint8) or M.device != self.device or not M.is_contiguous():
                raise ValueError("the mask must be a contiguous bool tensor on the engine's device")
            if tuple(M.shape) != tuple(self.V.shape):
                raise ValueError(f"the mask's shape {tuple(M.shape)} does not match V's {tuple(self.V.shape)}")
        self._mask, self._weight = M, None
        _capi.check(self._lib.nmfb200_set_mask(self._ctx, _ptr(M) if M is not None else None, _stream(self.device)))

    def set_weight(self, Wt):
        """Fit with per-cell weights from now on (include/nmf_b200.h: nmfb200_set_weight): Wt is a contiguous float32 tensor
        of V's shape on the engine's device, read in place, every weight finite and >= 0 (fit() checks the values); None
        clears it.  Replaces a mask, and a mask replaces it.  The engine keeps a reference to Wt while it is set.  minmax()
        then covers the cells of non-zero weight only."""
        if Wt is not None:
            if Wt.dtype != torch.float32 or Wt.device != self.device or not Wt.is_contiguous():
                raise ValueError("the weight must be a contiguous float32 tensor on the engine's device")
            if tuple(Wt.shape) != tuple(self.V.shape):
                raise ValueError(f"the weight's shape {tuple(Wt.shape)} does not match V's {tuple(self.V.shape)}")
        self._mask, self._weight = None, Wt
        _capi.check(self._lib.nmfb200_set_weight(self._ctx, _ptr(Wt) if Wt is not None else None, _stream(self.device)))

    def set_fixed_w(self, fixed):
        """Hold the components k of W with fixed[k] != 0 at their values from now on (include/nmf_b200.h:
        nmfb200_set_fixed_w): fixed is a contiguous uint8 tensor of R elements on the engine's device, read in place by every
        later W update; None clears it.  The engine keeps a reference to it while it is set."""
        if fixed is not None:
            if fixed.dtype != torch.uint8 or fixed.device != self.device or not fixed.is_contiguous():
                raise ValueError("fixed must be a contiguous uint8 tensor on the engine's device")
            if fixed.numel() != self.W.shape[1]:
                raise ValueError(f"fixed has {fixed.numel()} elements for W's {self.W.shape[1]} components")
        self._fixed_w = fixed
        _capi.check(self._lib.nmfb200_set_fixed_w(self._ctx, _ptr(fixed) if fixed is not None else None,
                                                  _stream(self.device)))

    def set_ard(self, b, c, phi):
        """Register automatic relevance determination on the current factors (include/nmf_b200.h: nmfb200_set_ard): the
        relevances lambda_k = (sum W[:, k] + sum H[:, k] + b) / c and the penalties phi / lambda_k that every later W and H
        update adds to component k's denominators; `iterate` then runs the lambda update after each H update.  b=None
        clears it."""
        if b is None:
            _capi.check(self._lib.nmfb200_set_ard(self._ctx, None, None, 0.0, 0.0, 0.0, _stream(self.device)))
            return
        _capi.check(self._lib.nmfb200_set_ard(self._ctx, _ptr(self.W), _ptr(self.H), float(b), float(c), float(phi),
                                              _stream(self.device)))

    def ard_update(self):
        """The lambda update from the current factors (include/nmf_b200.h: nmfb200_ard_update)."""
        _capi.check(self._lib.nmfb200_ard_update(self._ctx, _ptr(self.W), _ptr(self.H), _stream(self.device)))

    def ard_state(self):
        """(lambda, pen) as float32 device tensors of R elements and the last lambda update's largest relative change, a
        float (include/nmf_b200.h: nmfb200_ard_read; synchronises)."""
        R = self.W.shape[1]
        buf = torch.empty(2 * R + 1, dtype=torch.float32, device=self.device)
        _capi.check(self._lib.nmfb200_ard_read(self._ctx, _ptr(buf), _ptr(buf[R:]), _ptr(buf[2 * R:]),
                                               _stream(self.device)))
        return buf[:R], buf[R:2 * R], float(buf[2 * R])

    def ard_change(self):
        """The last lambda update's largest relative change, max_k |lambda_k - previous| / previous (synchronises)."""
        change = ctypes.c_float()
        _capi.check(self._lib.nmfb200_ard_read(self._ctx, None, None, ctypes.byref(change), _stream(self.device)))
        return change.value

    def minmax(self):
        vmin, vmax = ctypes.c_float(), ctypes.c_float()
        _capi.check(self._lib.nmfb200_target_minmax(self._ctx, ctypes.byref(vmin), ctypes.byref(vmax),
                                                    _stream(self.device)))
        return vmin.value, vmax.value

    def loss(self, beta):
        val = float(self.loss_tensor(beta).item())
        self.check_health()
        return val

    def check_health(self):
        """Raise if a kernel of the library aborted an internal wait since the last check (synchronises)."""
        _capi.check(self._lib.nmfb200_ctx_check_health(self._ctx, _stream(self.device)))

    def sync(self):
        _capi.check(self._lib.nmfb200_sync_factors(self._ctx))

    def update_w(self, beta, gamma, l1_reg, l2_reg):
        _capi.check(self._lib.nmfb200_update_w(self._ctx, _ptr(self.W), _ptr(self.H), beta, gamma, l1_reg, l2_reg,
                                               _stream(self.device)))

    def update_h(self, beta, gamma, l1_reg, l2_reg):
        _capi.check(self._lib.nmfb200_update_h(self._ctx, _ptr(self.W), _ptr(self.H), beta, gamma, l1_reg, l2_reg,
                                               _stream(self.device)))

    def loss_tensor(self, beta):
        _capi.check(self._lib.nmfb200_loss(self._ctx, _ptr(self.W), _ptr(self.H), beta, _ptr(self._loss),
                                           _stream(self.device)))
        return self._loss

    def raw_terms(self, which, beta):
        """(numerator, denominator) of the update of W (which=0) or H (which=1) from the CURRENT factors, untouched: the
        numerator in the factor's shape; the denominator (R,) for beta == 1 without a mask or weight (the column sums of the
        other factor), else in the factor's shape.  What BetaMu.step and PLCA.fit are built from (include/nmf_b200.h:
        nmfb200_raw_terms)."""
        f = self.W if which == 0 else self.H
        buf = self._raw_terms_into(which, beta, None)
        num, den = buf[:f.numel()].view(f.shape), buf[f.numel():]
        return num, (den if beta == 1 and self._mask is None and self._weight is None else den.view(f.shape))

    def plca_masked_terms(self, which, qobs=None):
        """(A, B), each in the shape of W (which=0) or H (which=1), of one EM step of a PLCA fit on the observed cells of V
        (set_mask), from the current factors: with W and H = H diag(Z) the model q, its mass q_O on the observed cells and
        V the normalised observed target, the step's gradient of that factor is q_O A + B (include/nmf_b200.h:
        nmfb200_plca_masked_terms).  `qobs`: an optional float64 device tensor of one element that receives q_O."""
        f = self.W if which == 0 else self.H
        n = f.numel()
        buf = torch.empty(2 * n, dtype=torch.float32, device=self.device)
        _capi.check(self._lib.nmfb200_plca_masked_terms(self._ctx, _ptr(self.W), _ptr(self.H), int(which), _ptr(buf),
                                                        _ptr(qobs) if qobs is not None else None, _stream(self.device)))
        return buf[:n].view(f.shape), buf[n:].view(f.shape)

    def _raw_terms_into(self, which, beta, buf):
        """nmfb200_raw_terms flat into `buf`, or into a new buffer when `buf` is None or of another size; returns it."""
        n = int(self._lib.nmfb200_raw_terms_numel(self._ctx, int(which), float(beta)))
        if buf is None or buf.numel() != n:
            buf = torch.empty(n, dtype=torch.float32, device=self.device)
        _capi.check(self._lib.nmfb200_raw_terms(self._ctx, _ptr(self.W), _ptr(self.H), int(which), float(beta), _ptr(buf),
                                                _stream(self.device)))
        return buf

    # --- pieces of the sharded W update (ShardedEngine) ---------------------------------------
    def w_partial(self, beta):
        """This shard's raw W terms, raw_terms(0)'s layout flat, in one buffer per engine reused every iteration."""
        self._wbuf = self._raw_terms_into(0, beta, self._wbuf)
        return self._wbuf

    def w_apply(self, reduced, beta, gamma, l1_reg, l2_reg):
        _capi.check(self._lib.nmfb200_w_apply(self._ctx, _ptr(self.W), _ptr(reduced), beta, gamma, l1_reg, l2_reg,
                                              _stream(self.device)))

    # ---- what sparse_fit (nmf.py:411-599) needs beyond the MU updates ----
    def project(self, x, dim, k1, k2):
        """Hoyer projection of every slice of x along `dim`, in place (one launch)."""
        return hoyer_project_(x, dim, k1, k2)

    def loss_at(self, W, H, beta):
        """beta-divergence of the reconstruction from TRIAL factors (same shapes as the engine's own; a line search's
        candidate).  The engine's operand copies follow the trial factors: call sync() after committing or discarding."""
        keep = self.W, self.H
        self.W, self.H = W, H
        try:
            self.sync()
            return self.loss(beta)
        finally:
            self.W, self.H = keep


class CudaNmfEngine(_CudaEngine):
    """Dense NMF on one GPU: V (N,C) fp32, fp16 or bf16 (rows may be strided), W (C,R) and H (N,R) fp32, all CUDA tensors
    (W, H updated in place)."""
    kind = "nmf"

    def __init__(self, V, W, H, precision="auto"):
        super().__init__()
        self.device = W.device
        _check_target(V, self.device, strided_rows=True)
        for t, n in ((W, "W"), (H, "H")):
            _check_f32_cuda(t, n, self.device)
        N, C = V.shape
        R = W.shape[1]
        assert W.shape == (C, R) and H.shape == (N, R)
        self.V, self.W, self.H = V, W, H
        self.N, self.C, self.R = N, C, R
        dev_index = _device_index(self.device)
        self._acquire(("nmf", dev_index, N, C, R, precision),
                      lambda ref: self._lib.nmfb200_nmf_create(ref, dev_index, N, C, R, _capi.PRECISIONS[precision]))
        self._loss = torch.zeros(1, dtype=torch.float64, device=self.device)
        _capi.check(self._lib.nmfb200_nmf_set_target(self._ctx, _ptr(V), V.stride(0), _capi.DTYPES[V.dtype],
                                                     _stream(self.device)))
        self.sync()

    def iterate(self, n_iter, beta, gamma, l1_reg, l2_reg):
        """n_iter x (update_w; update_h) in one call."""
        _capi.check(self._lib.nmfb200_nmf_iterate(self._ctx, _ptr(self.W), _ptr(self.H), beta, gamma, l1_reg, l2_reg,
                                                  int(n_iter), _stream(self.device)))

    def cd_update(self, which, l1_reg, l2_reg):
        """One coordinate-descent (HALS) update at beta 2 of W (which=0) or H (which=1) in place: one sweep over its columns
        (include/nmf_b200.h: nmfb200_nmf_cd_update)."""
        _capi.check(self._lib.nmfb200_nmf_cd_update(self._ctx, _ptr(self.W), _ptr(self.H), int(which), float(l1_reg),
                                                    float(l2_reg), _stream(self.device)))

    def cd_iterate(self, n_iter, l1_reg, l2_reg):
        """n_iter x (cd_update(0); cd_update(1)) in one call."""
        _capi.check(self._lib.nmfb200_nmf_cd_iterate(self._ctx, _ptr(self.W), _ptr(self.H), float(l1_reg), float(l2_reg),
                                                     int(n_iter), _stream(self.device)))

    def loss_prefetch_w(self, beta):
        """The loss at the current factors, taken out of the NEXT W update's contraction pass where the library can fold it
        (beta 1 on the tensor-core path): that update then skips its contraction.  Same value as loss() (synchronises)."""
        _capi.check(self._lib.nmfb200_nmf_loss_prefetch_w(self._ctx, _ptr(self.W), _ptr(self.H), beta, _ptr(self._loss),
                                                          _stream(self.device)))
        val = float(self._loss.item())
        self.check_health()
        return val

    def contract_only(self, which, beta):
        """bench.py: launch only the fused contraction kernel (0 = W update's, 1 = H update's)."""
        _capi.check(self._lib.nmfb200_nmf_contract_only(self._ctx, _ptr(self.W), _ptr(self.H), which, beta,
                                                        _stream(self.device)))

    # ---- row-sharded W update over peer memory (include/nmf_b200.h: nmfb200_nmf_peer_*) ----
    def peer_supported(self, beta):
        return bool(self._lib.nmfb200_nmf_peer_supported(self._ctx, float(beta)))

    def peer_world(self):
        return int(self._lib.nmfb200_nmf_peer_world(self._ctx))

    def peer_alloc(self):
        h = (ctypes.c_ubyte * 64)()
        _capi.check(self._lib.nmfb200_nmf_peer_alloc(self._ctx, ctypes.cast(h, ctypes.c_void_p)))
        return bytes(h)

    def peer_connect(self, world, rank, handles):
        buf = (ctypes.c_ubyte * (64 * world)).from_buffer_copy(handles)
        return int(self._lib.nmfb200_nmf_peer_connect(self._ctx, int(world), int(rank), ctypes.cast(buf, ctypes.c_void_p)))

    def peer_release(self):
        self._lib.nmfb200_nmf_peer_release(self._ctx)

    def update_w_peer(self, beta, gamma, l1_reg, l2_reg):
        _capi.check(self._lib.nmfb200_nmf_update_w_peer(self._ctx, _ptr(self.W), _ptr(self.H), beta, gamma, l1_reg,
                                                        l2_reg, _stream(self.device)))


class _F32Engine(_CudaEngine):
    """An engine whose context runs the fp32 kernels only."""

    @property
    def precision(self):
        return "f32"

    def precision_for(self, beta):
        return "f32"


class _BatchedEngine(_F32Engine):
    """What the batched engines share: the problems are the leading axis of W and H, every launch runs the active ones, and
    the loss is one value per problem."""
    _set_active = None                     # the C ABI's set_active call of this context kind

    def __init__(self, V, W, H):
        """V stacked on a leading problem axis, or one target of a single problem's shape shared by every problem (read at
        problem stride 0), on W's device; W and H contiguous fp32.  Every problem starts active."""
        super().__init__()
        self.device = W.device
        if V.dim() == W.dim() - 1:
            V = V.unsqueeze(0).expand(W.shape[0], *V.shape)              # one target: problem stride 0
        if V.dtype not in _capi.DTYPES:
            raise TypeError(f"V must be float32, float16 or bfloat16 (got {V.dtype})")
        if V.device != self.device:
            raise ValueError(f"V is on {V.device}, expected {self.device}")
        for t, n in ((W, "W"), (H, "H")):
            _check_f32_cuda(t, n, self.device)
        self._loss = torch.zeros(W.shape[0], dtype=torch.float64, device=self.device)
        self._create(V, W, H, _device_index(self.device))
        self.V, self.W, self.H = V, W, H
        self.set_active(None)
        self.sync()

    def _create(self, V, W, H, dev_index):
        """Check the shapes, take a context for them and set V (problems on axis 0) as its target."""
        raise NotImplementedError

    def set_active(self, active):
        """Run only the problems whose flag is set from now on: `active` is a bool sequence or tensor of one flag per
        problem (None: all).  The others keep their factors and their slot of losses()."""
        if active is None:
            self._active = None
        else:
            self._active = torch.as_tensor(active).to(device=self.device, dtype=torch.uint8).contiguous()
            assert self._active.shape == (self.W.shape[0],)
        _capi.check(getattr(self._lib, self._set_active)(
            self._ctx, _ptr(self._active) if self._active is not None else None, _stream(self.device)))

    def losses(self, beta):
        """beta_div of every problem's reconstruction, one float64 value per problem, on the host (one synchronisation); an
        inactive problem's value is the last one computed for it."""
        val = self.loss_tensor(beta).cpu()
        self.check_health()
        return val

    def loss(self, beta):
        raise TypeError("a batched engine has one loss per problem: use losses()")

    def raw_terms(self, which, beta):
        """(numerator, denominator) of every problem's update of W (which=0) or H (which=1): the numerator in the factor's
        shape (problems, rows, R, ...); the denominator (problems, R) at beta 1 (the column sums of the other factor), else
        in the factor's shape."""
        f = self.W if which == 0 else self.H
        buf = self._raw_terms_into(which, beta, None)
        num, den = buf[:f.numel()].view(f.shape), buf[f.numel():]
        return num, (den.view(f.shape[0], f.shape[2]) if beta == 1 else den.view(f.shape))

    # ---- batched PLCA (include/nmf_b200.h: nmfb200_plca_iterate): the engine's factor pair is (W, Hz = H diag(Z)) ----
    def plca_iterate(self, n_iter, H, Z, train_w, train_h, train_z, W_alpha=None, H_alpha=None, Z_alpha=None):
        """n_iter EM iterations of every active problem in one call: the two raw-terms passes and one EM-step launch each.
        Updates self.W, H (H's shape), Z (P, R) and self.H (= H Z) in place; the alphas are None (1) or contiguous fp32
        tensors of the batched factor's shape."""
        if getattr(self, "_plca_work", None) is None:
            n = int(self._lib.nmfb200_plca_work_numel(self._ctx))
            self._plca_work = torch.empty(n, dtype=torch.float32, device=self.device)
        flags = (_capi.PLCA_TRAIN_W if train_w else 0) | (_capi.PLCA_TRAIN_H if train_h else 0) | (
            _capi.PLCA_TRAIN_Z if train_z else 0)
        alphas = [_ptr(a) if a is not None else None for a in (W_alpha, H_alpha, Z_alpha)]
        _capi.check(self._lib.nmfb200_plca_iterate(self._ctx, _ptr(self.W), _ptr(H), _ptr(Z), _ptr(self.H),
                                                   _ptr(self._plca_work), flags, *alphas, int(n_iter),
                                                   _stream(self.device)))

    def plca_losses(self, norm):
        """kl_div(norm[p] X_p, norm[p] V_p) of every problem (X_p from W and Hz, V_p the normalised target), one float64 value
        per problem, on the host (one synchronisation); an inactive problem's value is the last one computed for it.
        norm: (P,) fp32 on the engine's device."""
        _capi.check(self._lib.nmfb200_plca_loss(self._ctx, _ptr(self.W), _ptr(self.H), _ptr(norm), _ptr(self._loss),
                                                _stream(self.device)))
        val = self._loss.cpu()
        self.check_health()
        return val


class CudaBatchedNmfEngine(_BatchedEngine):
    """B independent dense NMF problems of one shape on one GPU (include/nmf_b200.h: nmfb200_nmf_batched_create), on the
    fp32 kernels: V (B,N,C) -- or (N,C), one target shared by every problem -- fp32, fp16 or bf16 with unit column stride,
    rows and problems strided; W (B,C,R) and H (B,N,R) contiguous fp32, updated in place.  Every update and loss launch
    runs all problems, and problem b's factors and loss are bit for bit those of CudaNmfEngine(V[b], W[b], H[b], "f32").

    `lengths` (B ints in [1, N], or None): a ragged batch (nmfb200_nmf_batched_create_ragged) -- problem b is the problem of
    V[b, :lengths[b]], W[b] and H[b, :lengths[b]], bit for bit CudaNmfEngine(V[b, :L], W[b], H[b, :L], "f32"); the rows
    past lengths[b] of V[b] are never read and those of H[b] never written.  plca_iterate / plca_losses serve it (problem b
    is then the PLCA problem of those rows, the padding rows of H and Hz neither read nor written); cd_update / cd_iterate
    do not."""
    kind = "nmf_batched"
    _set_active = "nmfb200_nmf_batched_set_active"

    def __init__(self, V, W, H, lengths=None):
        self._lengths = None if lengths is None else tuple(int(n) for n in lengths)
        super().__init__(V, W, H)

    def _create(self, V, W, H, dev_index):
        B, N, C = V.shape
        R = W.shape[2]
        assert W.shape == (B, C, R) and H.shape == (B, N, R)
        if not (V.stride(2) == 1 and V.stride(1) >= C and (V.stride(0) == 0 or V.stride(0) >= N * V.stride(1))):
            raise ValueError("V must have unit column stride, rows at least C apart and problems at least N rows apart")
        if self._lengths is None:
            self._acquire(("nmf_batched", dev_index, B, N, C, R),
                          lambda ref: self._lib.nmfb200_nmf_batched_create(ref, dev_index, B, N, C, R))
        else:
            if len(self._lengths) != B:
                raise ValueError(f"lengths holds {len(self._lengths)} values for {B} problems")
            lens = (ctypes.c_int64 * B)(*self._lengths)
            self._acquire(("nmf_batched", dev_index, B, N, C, R, self._lengths),
                          lambda ref: self._lib.nmfb200_nmf_batched_create_ragged(ref, dev_index, B, N, C, R, lens))
        _capi.check(self._lib.nmfb200_nmf_batched_set_target(self._ctx, _ptr(V), V.stride(1), V.stride(0),
                                                             _capi.DTYPES[V.dtype], _stream(self.device)))

    def iterate(self, n_iter, beta, gamma, l1_reg, l2_reg):
        """n_iter x (update_w; update_h) of every active problem in one call."""
        _capi.check(self._lib.nmfb200_nmf_iterate(self._ctx, _ptr(self.W), _ptr(self.H), beta, gamma, l1_reg, l2_reg,
                                                  int(n_iter), _stream(self.device)))

    def cd_update(self, which, l1_reg, l2_reg):
        """One coordinate-descent (HALS) update at beta 2 of W (which=0) or H (which=1) of every active problem, in place
        (include/nmf_b200.h: nmfb200_nmf_batched_cd_update)."""
        _capi.check(self._lib.nmfb200_nmf_batched_cd_update(self._ctx, _ptr(self.W), _ptr(self.H), int(which),
                                                            float(l1_reg), float(l2_reg), _stream(self.device)))

    def cd_iterate(self, n_iter, l1_reg, l2_reg):
        """n_iter x (cd_update(0); cd_update(1)) of every active problem in one call."""
        _capi.check(self._lib.nmfb200_nmf_batched_cd_iterate(self._ctx, _ptr(self.W), _ptr(self.H), float(l1_reg),
                                                             float(l2_reg), int(n_iter), _stream(self.device)))


class CudaBatchedNmfdEngine(_BatchedEngine):
    """P independent NMFD / NMF2D / NMF3D problems of one shape on one GPU (include/nmf_b200.h:
    nmfb200_nmfnd_batched_create), on the fp32 kernels: V (P,B,C,*X) -- or (B,C,*X), one target shared by every problem --
    fp32, fp16 or bf16, each problem's block contiguous and the blocks at least B C prod(X) elements apart; W (P,C,R,*K) and
    H (P,B,R,*(X-K+1)) contiguous fp32, updated in place.  Every update and loss launch runs all problems, and problem p's
    factors and loss are bit for bit those of CudaNmfdEngine(V[p], W[p], H[p], "f32").  No `iterate`: the fit loop calls
    update_w / update_h, as for a single NMFD engine.

    `lengths` (P ints in [K_last, X_last], or None): a ragged batch along the last axis
    (nmfb200_nmfnd_batched_create_ragged) -- problem p is the problem of V[p, ..., :lengths[p]], W[p] and
    H[p, ..., :lengths[p] - K_last + 1], bit for bit CudaNmfdEngine on those, "f32"; the positions past them of V[p] are
    never read and those of H[p] never written."""
    kind = "nmfd_batched"
    _set_active = "nmfb200_nmfd_batched_set_active"

    def __init__(self, V, W, H, lengths=None):
        self._lengths = None if lengths is None else tuple(int(n) for n in lengths)
        super().__init__(V, W, H)

    def _create(self, V, W, H, dev_index):
        P, C, R, *K = W.shape
        _, B, _, *X = V.shape
        nd = len(K)
        assert 1 <= nd <= 3 and len(X) == nd
        assert W.shape == (P, C, R, *K) and H.shape == (P, B, R, *(x - k + 1 for x, k in zip(X, K)))
        if not (V[0].is_contiguous() and (V.stride(0) == 0 or V.stride(0) >= V[0].numel())):
            raise ValueError("every problem's block of V must be contiguous, the blocks 0 or at least B C prod(X) apart")
        vd, kd = (ctypes.c_int64 * nd)(*X), (ctypes.c_int64 * nd)(*K)
        if self._lengths is None:
            self._acquire(("nmfd_batched", dev_index, P, B, C, tuple(X), R, tuple(K)),
                          lambda ref: self._lib.nmfb200_nmfnd_batched_create(ref, dev_index, P, B, C, nd, vd, R, kd))
        else:
            if len(self._lengths) != P:
                raise ValueError(f"lengths holds {len(self._lengths)} values for {P} problems")
            lens = (ctypes.c_int64 * P)(*self._lengths)
            self._acquire(("nmfd_batched", dev_index, P, B, C, tuple(X), R, tuple(K), self._lengths),
                          lambda ref: self._lib.nmfb200_nmfnd_batched_create_ragged(ref, dev_index, P, B, C, nd, vd, R, kd,
                                                                                   lens))
        _capi.check(self._lib.nmfb200_nmfd_batched_set_target(self._ctx, _ptr(V), V.stride(0), _capi.DTYPES[V.dtype],
                                                              _stream(self.device)))


def _compressed_forms(V, weights=None, with_order=False):
    """Both compressed forms of a coalesced sparse COO tensor V (N,C) on the device, built with torch (data-format plumbing):
    (crow, col, val) = CSR, (ccol, row, val_t) = CSC, int64 indices and fp32 values, all contiguous.  With `weights` (one
    per stored entry, in V's order) also (wt, wt_t): the weights in CSR and in CSC order.  With `with_order`, last, the CSR
    position of each CSC entry (int64, contiguous)."""
    N, C = V.shape
    vals = V.values().to(torch.float32).contiguous()
    rows, cols = V.indices()[0].contiguous(), V.indices()[1].contiguous()          # coalesced: sorted by (row, col)
    crow = torch.zeros(N + 1, dtype=torch.int64, device=vals.device)
    crow[1:] = torch.cumsum(torch.bincount(rows, minlength=N), 0)
    order = torch.argsort(cols * N + rows)                                         # the same entries sorted by (col, row)
    ccol = torch.zeros(C + 1, dtype=torch.int64, device=vals.device)
    ccol[1:] = torch.cumsum(torch.bincount(cols, minlength=C), 0)
    forms = (crow, cols, vals, ccol, rows[order].contiguous(), vals[order].contiguous())
    if weights is not None:
        wt = weights.to(torch.float32).contiguous()
        forms += (wt, wt[order].contiguous())
    return forms + (order.contiguous(),) if with_order else forms


class _SparseEngine(_F32Engine):
    """What the engines on a sparse target share: V is a coalesced sparse COO tensor (N,C) on the device of W (C,R) and
    H (N,R), both contiguous fp32.  The target's compressed forms (_compressed_forms of V, `weights` and `with_order`) are
    built here with torch (data-format plumbing) and kept alive for the context, which borrows them."""
    kind = "nmf"

    def __init__(self, V, W, H, h_name="H", weights=None, with_order=False):
        super().__init__()
        self.device = W.device
        for t, n in ((W, "W"), (H, h_name)):
            _check_f32_cuda(t, n, self.device)
        assert V.is_sparse and V.is_coalesced() and V.device == W.device
        N, C = V.shape
        R = W.shape[1]
        assert W.shape == (C, R) and H.shape == (N, R)
        self.W, self.H = W, H
        self.N, self.C, self.R = N, C, R
        if weights is not None:
            assert weights.shape == (V._nnz(),) and weights.device == W.device
        self._forms = _compressed_forms(V, weights, with_order)
        self._loss = torch.zeros(1, dtype=torch.float64, device=self.device)

    def _acquire_nmf(self):
        """Take a cached or new fp32 NMF context of the engine's shape: the sparse and observed-cell NMF targets run on it."""
        dev_index, N, C, R = _device_index(self.device), self.N, self.C, self.R
        self._acquire(("nmf", dev_index, N, C, R, "f32"),
                      lambda ref: self._lib.nmfb200_nmf_create(ref, dev_index, N, C, R, _capi.PRECISIONS["f32"]))


class CudaSparseNmfEngine(_SparseEngine):
    """NMF on a sparse target, beta 1 or 2 (reference: nmf.py:603-638): the update terms are evaluated at the non-zeros
    only by the library (include/nmf_b200.h: nmfb200_nmf_set_target_sparse)."""
    _set_target = "nmfb200_nmf_set_target_sparse"

    def __init__(self, V, W, H, precision="auto"):
        super().__init__(V, W, H)
        vals = self._forms[2]
        nnz = int(vals.numel())
        v64 = vals.double()
        pos = v64[v64 > 0]
        vnorm_kl = float((pos * pos.log()).sum() - v64.sum())                # nmf.py:166-167 (0 log 0 = 0)
        vnorm_eu = float((v64 * v64).sum() * 0.5)                            # nmf.py:164-165
        self._vmin = float(vals.min()) if nnz else 0.0
        self._vmax = float(vals.max()) if nnz else 0.0
        self._has_zeros = nnz < self.N * self.C
        self._acquire_nmf()
        _capi.check(getattr(self._lib, self._set_target)(self._ctx, nnz, *(_ptr(t) for t in self._forms), vnorm_kl,
                                                          vnorm_eu, _stream(self.device)))

    def minmax(self):
        return (min(self._vmin, 0.0) if self._has_zeros else self._vmin), self._vmax

    iterate = CudaNmfEngine.iterate
    cd_update = CudaNmfEngine.cd_update
    cd_iterate = CudaNmfEngine.cd_iterate


class CudaSparseAnyBetaEngine(CudaSparseNmfEngine):
    """NMF on a sparse target at every beta > 0, without densifying it (include/nmf_b200.h:
    nmfb200_nmf_set_target_sparse_any_beta): beta 1 and 2 as CudaSparseNmfEngine; any other beta takes its numerators at the
    non-zeros and its denominators and loss from V-free dense contractions, so the device holds O(nnz + (N + C) R)."""
    _set_target = "nmfb200_nmf_set_target_sparse_any_beta"


class CudaSparsePlcaEngine(_SparseEngine):
    """One EM step's gradients of a PLCA fit on a sparse target (include/nmf_b200.h: nmfb200_plca_sparse_*): Vn is a
    coalesced sparse COO tensor (N,C) of V / sum(V) with fp32 values on the device, W (C,R) and Hz = H diag(Z) (N,R)
    contiguous fp32 on the same device.  Its own context kind: the device holds O(nnz + (N + C) R), nothing of size N x C,
    at every rank."""
    kind = "plca_sparse"

    def __init__(self, Vn, W, Hz):
        super().__init__(Vn, W, Hz, h_name="Hz", with_order=True)
        crow, col, val, ccol, row, _, perm = self._forms
        self._forms = (crow, col, val, ccol, row, perm)          # the CSC values are not read: not kept
        N, C, R = self.N, self.C, self.R
        _capi.check(self._lib.nmfb200_plca_sparse_create(ctypes.byref(self._ctx), _device_index(self.device), N, C, R,
                                                         int(val.numel())))
        _capi.check(self._lib.nmfb200_plca_sparse_set_target(self._ctx, *(_ptr(t) for t in self._forms),
                                                             _stream(self.device)))
        self._out = torch.empty(C * R + N * R, dtype=torch.float32, device=self.device)

    def device_bytes(self):
        """Device bytes of the context's workspace (the compressed forms and the gradient buffer are torch tensors)."""
        return int(self._lib.nmfb200_plca_sparse_device_bytes(self._ctx))

    def plca_terms(self, Hz, norm=None):
        """(dW, dHz) of one EM step at self.W and Hz: P = Vn / (Hz W^T + eps) at the stored entries, dW = P^T Hz, dHz = P W,
        in a buffer the next call overwrites.  With `norm` (a float: the fp32 value of sum(V)) also the loss
        kl_div(norm q, norm Vn) from the same pass, as a float64 device tensor of one element: (dW, dHz, loss)."""
        _capi.check(self._lib.nmfb200_plca_sparse_terms(self._ctx, _ptr(self.W), _ptr(Hz), _ptr(self._out),
                                                        float(norm) if norm is not None else 0.0,
                                                        _ptr(self._loss) if norm is not None else None,
                                                        _stream(self.device)))
        C, N, R = self.C, self.N, self.R
        dW, dHz = self._out[:C * R].view(C, R), self._out[C * R:].view(N, R)
        return (dW, dHz) if norm is None else (dW, dHz, self._loss)

    def loss(self, norm):
        """kl_div(norm q, norm Vn) at self.W and self.H (= Hz), on the host (synchronises): one row-gather launch."""
        _capi.check(self._lib.nmfb200_plca_sparse_terms(self._ctx, _ptr(self.W), _ptr(self.H), None, float(norm),
                                                        _ptr(self._loss), _stream(self.device)))
        val = float(self._loss.item())
        self.check_health()
        return val


class CudaObservedNmfEngine(_SparseEngine):
    """NMF on the observed cells of a masked fit (include/nmf_b200.h: nmfb200_nmf_set_target_observed), rank <= 256: O is a
    coalesced fp32 sparse COO tensor (N,C) on the device whose stored entries are exactly the observed cells, explicit zeros
    included, with V's values there.  The fit minimises beta_div(WH[obs], V[obs]) at every beta; every update and the loss
    touch the observed cells only, O(observed x R) per update.  `weights` (optional, one positive fp32 weight per stored entry
    of O, in O's order): the fit minimises sum_obs w d_beta(v | WH) instead (nmfb200_nmf_set_target_observed_weighted)."""

    def __init__(self, O, W, H, precision="auto", weights=None):
        super().__init__(O, W, H, weights=weights)
        self._acquire_nmf()
        set_target = (self._lib.nmfb200_nmf_set_target_observed if weights is None
                      else self._lib.nmfb200_nmf_set_target_observed_weighted)
        _capi.check(set_target(self._ctx, int(self._forms[2].numel()), *(_ptr(t) for t in self._forms),
                               _stream(self.device)))

    def raw_terms(self, which, beta):
        """(numerator, denominator) of the update of W (which=0) or H (which=1), both in the factor's shape at every beta."""
        f = self.W if which == 0 else self.H
        buf = self._raw_terms_into(which, beta, None)
        return buf[:f.numel()].view(f.shape), buf[f.numel():].view(f.shape)

    def cd_update(self, which, l1_reg, l2_reg):
        """One coordinate-descent update at beta 2 of W (which=0) or H (which=1) in place on the observed cells: one exact
        sweep over its columns (include/nmf_b200.h: nmfb200_nmf_observed_cd_update)."""
        _capi.check(self._lib.nmfb200_nmf_observed_cd_update(self._ctx, _ptr(self.W), _ptr(self.H), int(which),
                                                             float(l1_reg), float(l2_reg), _stream(self.device)))

    def cd_iterate(self, n_iter, l1_reg, l2_reg):
        """n_iter x (cd_update(0); cd_update(1)) in one call."""
        _capi.check(self._lib.nmfb200_nmf_observed_cd_iterate(self._ctx, _ptr(self.W), _ptr(self.H), float(l1_reg),
                                                              float(l2_reg), int(n_iter), _stream(self.device)))

    iterate = CudaNmfEngine.iterate


class CudaNmfdEngine(_CudaEngine):
    """NMFD / NMF2D / NMF3D on one GPU: V (B,C,*X), W (C,R,*K), H (B,R,*(X-K+1)) over one to three convolved axes; V
    contiguous fp32, fp16 or bf16, W and H contiguous fp32."""
    kind = "nmfd"

    def __init__(self, V, W, H, precision="auto"):
        super().__init__()
        self.device = W.device
        _check_target(V, self.device)
        for t, n in ((W, "W"), (H, "H")):
            _check_f32_cuda(t, n, self.device)
        B, C, *X = V.shape
        _, R, *K = W.shape
        nd = len(X)
        assert 1 <= nd <= 3 and len(K) == nd
        assert W.shape == (C, R, *K) and H.shape == (B, R, *(x - k + 1 for x, k in zip(X, K)))
        self.V, self.W, self.H = V, W, H
        dev_index = _device_index(self.device)
        # "f16": beta 1 on the tensor-core sliding GEMMs; "auto" stays on the fp32 kernels for NMF2D / NMF3D
        vd, kd = (ctypes.c_int64 * nd)(*X), (ctypes.c_int64 * nd)(*K)
        self._acquire(("nmfd", dev_index, B, C, tuple(X), R, tuple(K), precision),
                      lambda ref: self._lib.nmfb200_nmfnd_create(ref, dev_index, B, C, nd, vd, R, kd,
                                                                 _capi.PRECISIONS[precision]))
        self._loss = torch.zeros(1, dtype=torch.float64, device=self.device)
        _capi.check(self._lib.nmfb200_nmfd_set_target(self._ctx, _ptr(V), _capi.DTYPES[V.dtype], _stream(self.device)))


class Collectives:
    """The collectives of a sharded fit's host code over a process group (None: the default group), on small tensors on
    `device` (a CUDA device for NCCL): a sum in place, agreement on a flag and agreement on sizes.  Every rank calls them
    in the same order."""

    def __init__(self, group, device):
        import torch.distributed as dist
        self._dist = dist
        self.group = group
        self.device = device
        self.world = dist.get_world_size(group)

    def _reduce_device(self):
        return self.device

    def all_reduce_(self, t):
        """Collective: `t` summed over the ranks, in place (one SUM all-reduce); returns t."""
        self._dist.all_reduce(t, op=self._dist.ReduceOp.SUM, group=self.group)
        return t

    def all_ranks(self, flag):
        """Collective: whether `flag` holds on every rank (one MIN all-reduce)."""
        t = torch.tensor([int(bool(flag))], dtype=torch.int32, device=self._reduce_device())
        self._dist.all_reduce(t, op=self._dist.ReduceOp.MIN, group=self.group)
        return bool(t.item())

    def check_same_sizes(self, names, sizes):
        """Collective: raise ValueError on every rank unless every rank passed the same `sizes` (ints; `names` label them
        in the message), so the W all-reduce never sums buffers of different lengths.  One MIN and one MAX all-reduce."""
        lo = torch.tensor(sizes, dtype=torch.int64, device=self._reduce_device())
        hi = lo.clone()
        self._dist.all_reduce(lo, op=self._dist.ReduceOp.MIN, group=self.group)
        self._dist.all_reduce(hi, op=self._dist.ReduceOp.MAX, group=self.group)
        lo, hi = lo.tolist(), hi.tolist()
        if lo != hi:
            differ = ", ".join(f"{n} from {a} to {b}" for n, a, b in zip(names, lo, hi) if a != b)
            mine = ", ".join(f"{n}={s}" for n, s in zip(names, sizes))
            raise ValueError(f"sharded fit: every rank must have the same sizes past the batch axis, but across ranks {differ} "
                             f"(this rank: {mine})")


class ShardedEngine(Collectives):
    """Sharded fit over a process group: every rank holds a shard of V and H and a replica of W -- NMF shards the rows
    (V[n_g,:], H[n_g,:]), NMFD / NMF2D / NMF3D the batch axis (V[b_g], H[b_g]).

    H update and phi stage are local.  The W update is `local raw contraction -> ONE sum-all-reduce ->
    identical ratio stage on every rank` (relu/eps/l1/l2/gamma are applied after the reduction because
    they are not linear).  The loss is one more scalar all-reduce every 10th iteration, and min/max
    for validation one at entry.  No V or H data ever moves.  NMF's W update may run over peer memory instead
    (`_peer_ready`); the convolutive models always take the all-reduce.
    """

    def __init__(self, local, group=None):
        dev = getattr(local, "device", None)
        super().__init__(group, dev if dev is not None else torch.device("cpu"))
        self.local = local
        self.kind = local.kind
        self._peer = {}                      # beta -> does the W update run over peer memory
        self.w_update_path = "nccl"

    @property
    def precision(self):
        return self.local.precision

    def precision_for(self, beta):
        return self.local.precision_for(beta) if hasattr(self.local, "precision_for") else self.local.precision

    def close(self):
        self.local.close()

    def sync(self):
        self.local.sync()

    def set_mask(self, M):
        """This rank's shard of the mask (the rows / batch elements of its V shard)."""
        self.local.set_mask(M)

    def set_weight(self, Wt):
        """This rank's shard of the weight (the rows / batch elements of its V shard)."""
        self.local.set_weight(Wt)

    def minmax(self):
        vmin, vmax = self.local.minmax()
        t = torch.tensor([-vmin, vmax], dtype=torch.float32, device=self._reduce_device())
        if vmin != vmin or vmax != vmax:          # NaN must survive the reduction
            t.fill_(float("nan"))
        self._dist.all_reduce(t, op=self._dist.ReduceOp.MAX, group=self.group)
        t = t.cpu()
        return -float(t[0]), float(t[1])

    def _peer_ready(self, beta):
        """Collective, once per (engine, beta): may the W update run over peer memory?  Every rank must answer the same, so
        each step is agreed with a MIN all-reduce.  Off with NMFB200_PEER=0, on another backend than NCCL, beyond 8 ranks, or
        when the CUDA IPC handles cannot be opened (ranks on different nodes): the NCCL all-reduce path is used then."""
        key = float(beta)
        if key in self._peer:
            return self._peer[key]
        dist, loc = self._dist, self.local
        ok = (os.environ.get("NMFB200_PEER", "1") != "0" and hasattr(loc, "peer_supported") and 2 <= self.world <= 8
              and dist.get_backend(self.group) == "nccl" and loc.peer_supported(beta))
        dev = self._reduce_device()
        connected = bool(ok) and loc.peer_world() == self.world
        t = torch.tensor([int(bool(ok)), int(connected)], dtype=torch.int32, device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MIN, group=self.group)
        ok, connected = bool(t[0].item()), bool(t[1].item())
        if ok and not connected:
            mine = torch.frombuffer(bytearray(loc.peer_alloc()), dtype=torch.uint8).to(dev)
            allh = torch.empty(self.world * 64, dtype=torch.uint8, device=dev)
            dist.all_gather_into_tensor(allh, mine, group=self.group)
            rc = loc.peer_connect(self.world, dist.get_rank(self.group), allh.cpu().numpy().tobytes())
            t = torch.tensor([int(rc == 0)], dtype=torch.int32, device=dev)
            dist.all_reduce(t, op=dist.ReduceOp.MIN, group=self.group)
            ok = bool(t[0].item())
            if not ok:
                loc.peer_release()
        self._peer[key] = ok
        self.w_update_path = "peer" if ok else "nccl"
        return ok

    def update_w(self, beta, gamma, l1_reg, l2_reg):
        if self._peer_ready(beta):
            self.local.update_w_peer(beta, gamma, l1_reg, l2_reg)     # contraction -> publish -> fused P2P sum + ratio stage
            return
        buf = self.local.w_partial(beta)
        self._dist.all_reduce(buf, op=self._dist.ReduceOp.SUM, group=self.group)
        self.local.w_apply(buf, beta, gamma, l1_reg, l2_reg)

    def update_h(self, beta, gamma, l1_reg, l2_reg):
        self.local.update_h(beta, gamma, l1_reg, l2_reg)

    def loss(self, beta):
        t = self.local.loss_tensor(beta).clone()
        self._dist.all_reduce(t, op=self._dist.ReduceOp.SUM, group=self.group)
        val = float(t.item())
        self.check_health()
        return val

    def check_health(self):
        if hasattr(self.local, "check_health"):
            self.local.check_health()
