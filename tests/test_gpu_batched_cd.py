"""`BatchedNMF.fit(V, beta=2, solver="cd")` on the GPU (include/nmf_b200.h: nmfb200_nmf_batched_cd_*).

* Every problem's n_iter, W and H equal, bit for bit, those of `NMF.fit(V[p], 2, ..., precision="f32", solver="cd")`: at the
  tile-plan edges, multi-chunk numerators, 1 / 2 / 4 / 8 components per lane, a multi-block Gram plan with a short last block,
  batches folded across many blocks, shared / half-precision / row-strided targets, alpha / l1_ratio, frozen factors, and
  problems that stop at different checks.
* Two runs are bit-identical; host and float64 modules give the CUDA fp32 module's bits.
* The ABI: inactive problems are not written, a dead component keeps its column, one batched update takes the launches of
  one single-problem update, and the refusals.
"""
import ctypes

import pytest
import torch

from f32_cases import NMF_CHUNKED, NMF_EDGE

pytestmark = pytest.mark.gpu


def _problems(B, N, C, R, seed, dtype=torch.float32, strided=False, shared=False, graded=False):
    """Targets (B, N, C) -- or one (N, C) shared target -- on the device and fp32 starting factors on the host.  graded:
    planted rank-R targets under noise growing with the problem, so their fits stop at different checks."""
    gen = torch.Generator().manual_seed(seed)
    shape = (N, C) if shared else (B, N, C)
    if graded:
        V = torch.rand(B, N, R, generator=gen) @ torch.rand(B, R, C, generator=gen)
        V += torch.logspace(-3, 0, B).view(B, 1, 1) * torch.rand(B, N, C, generator=gen)
    else:
        V = torch.rand(*shape[:-1], shape[-1] + (3 if strided else 0), generator=gen)
    V = V.to(dtype).cuda()
    if strided:
        V = V[..., :C]
    W0 = torch.rand(B, C, R, generator=gen) + 0.1
    H0 = torch.rand(B, N, R, generator=gen) + 0.1
    return V, W0, H0


def _batched(V, W0, H0, tol=1e-4, max_iter=20, alpha=0.0, l1_ratio=0.0, cuda=True, double=False, **fr):
    from torchnmf_b200 import BatchedNMF
    m = BatchedNMF(W=W0, H=H0, **fr)
    m = m.cuda() if cuda else m
    m = m.double() if double else m
    n = m.fit(V, 2, tol, max_iter, False, alpha, l1_ratio, solver="cd")
    assert m.last_fit_precision == "f32"
    return n, m.W.data, m.H.data


def _assert_each_is_its_single_fit(V, W0, H0, tol=1e-4, max_iter=20, alpha=0.0, l1_ratio=0.0, **fr):
    from torchnmf_b200 import NMF
    n, W, H = _batched(V, W0, H0, tol, max_iter, alpha, l1_ratio, **fr)
    counts = []
    for p in range(W0.shape[0]):
        m = NMF(W=W0[p], H=H0[p], **fr).cuda()
        n_p = m.fit(V if V.dim() == 2 else V[p], 2, tol, max_iter, False, alpha, l1_ratio, precision="f32", solver="cd")
        counts.append(n_p)
        assert int(n[p]) == n_p, p
        assert torch.equal(W[p], m.W.data), p
        assert torch.equal(H[p], m.H.data), p
    return counts


# ---- bit for bit per problem -------------------------------------------------------------------------------------------

@pytest.mark.parametrize("N,C,R", NMF_EDGE + NMF_CHUNKED[:4])
def test_each_problem_equals_its_single_fit(N, C, R):
    V, W0, H0 = _problems(3, N, C, R, seed=N * 7 + C * 3 + R)
    _assert_each_is_its_single_fit(V, W0, H0, alpha=0.1, l1_ratio=0.3)


def test_multi_block_gram_with_a_short_last_block():
    # 5000 rows: sparse_gram_plan gives 79 blocks of 64 rows, the last one of 8
    V, W0, H0 = _problems(3, 5000, 300, 33, seed=5)
    _assert_each_is_its_single_fit(V, W0, H0, max_iter=10)


def test_many_problems_fold_across_blocks():
    V, W0, H0 = _problems(300, 65, 40, 17, seed=6)
    _assert_each_is_its_single_fit(V, W0, H0, tol=1e-3, max_iter=30)


@pytest.mark.parametrize("kind", ["shared", "f16", "bf16", "strided"])
def test_targets(kind):
    dtype = {"f16": torch.float16, "bf16": torch.bfloat16}.get(kind, torch.float32)
    V, W0, H0 = _problems(4, 129, 191, 65, seed=7, dtype=dtype, strided=kind == "strided", shared=kind == "shared")
    _assert_each_is_its_single_fit(V, W0, H0, alpha=0.2, l1_ratio=0.5)


@pytest.mark.parametrize("alpha,l1_ratio", [(0.5, 0.0), (0.5, 1.0), (1.0, 0.25)])
def test_penalties(alpha, l1_ratio):
    V, W0, H0 = _problems(3, 200, 150, 20, seed=8)
    _assert_each_is_its_single_fit(V, W0, H0, alpha=alpha, l1_ratio=l1_ratio)


@pytest.mark.parametrize("frozen", ["W", "H"])
def test_frozen_factor(frozen):
    V, W0, H0 = _problems(3, 190, 130, 24, seed=9)
    fr = dict(trainable_W=frozen != "W", trainable_H=frozen != "H")
    _assert_each_is_its_single_fit(V, W0, H0, alpha=0.1, l1_ratio=0.5, **fr)
    _, W, H = _batched(V, W0, H0, **fr)
    assert torch.equal((W if frozen == "W" else H).cpu(), W0 if frozen == "W" else H0)


def test_problems_stop_at_different_iterations():
    V, W0, H0 = _problems(8, 120, 90, 6, seed=10, graded=True)
    counts = _assert_each_is_its_single_fit(V, W0, H0, tol=5e-4, max_iter=200)
    assert len(set(counts)) >= 3, counts


# ---- runs and staging ------------------------------------------------------------------------------------------------------

def test_runs_and_staged_modules_are_bit_identical():
    V, W0, H0 = _problems(4, 300, 200, 16, seed=11)
    n, W, H = _batched(V, W0, H0, max_iter=30)
    n2, W2, H2 = _batched(V, W0, H0, max_iter=30)
    assert torch.equal(n, n2) and torch.equal(W, W2) and torch.equal(H, H2)
    nh, Wh, Hh = _batched(V.cpu(), W0, H0, max_iter=30, cuda=False)
    assert Wh.device.type == "cpu" and torch.equal(nh, n) and torch.equal(Wh, W.cpu()) and torch.equal(Hh, H.cpu())
    nd, Wd, Hd = _batched(V.double(), W0, H0, max_iter=30, double=True)
    assert Wd.dtype == torch.float64 and torch.equal(nd, n)
    assert torch.equal(Wd, W.double()) and torch.equal(Hd, H.double())


# ---- the ABI -----------------------------------------------------------------------------------------------------------------

def _lib():
    from torchnmf_b200 import _capi
    return _capi, _capi.load()


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _batched_ctx(lib, capi, B, N, C, R, V, ctxs):
    c = ctypes.c_void_p()
    assert lib.nmfb200_nmf_batched_create(ctypes.byref(c), torch.cuda.current_device(), B, N, C, R) == 0
    ctxs.append(c)
    if V is not None:
        assert lib.nmfb200_nmf_batched_set_target(c, _p(V), V.stride(1), V.stride(0), capi.DTYPE_F32, _stream()) == 0
    return c


def test_inactive_problems_are_not_written():
    capi, lib = _lib()
    B, N, C, R = 3, 150, 100, 12
    V, W0, H0 = _problems(B, N, C, R, seed=12)
    W, H = W0.cuda(), H0.cuda()
    active = torch.tensor([1, 0, 1], dtype=torch.uint8, device="cuda")
    ctxs = []
    try:
        c = _batched_ctx(lib, capi, B, N, C, R, V, ctxs)
        assert lib.nmfb200_nmf_batched_set_active(c, _p(active), _stream()) == 0
        assert lib.nmfb200_nmf_batched_cd_iterate(c, _p(W), _p(H), 0.1, 0.1, 3, _stream()) == 0
        torch.cuda.synchronize()
    finally:
        for c in ctxs:
            lib.nmfb200_destroy(c)
    assert torch.equal(W[1].cpu(), W0[1]) and torch.equal(H[1].cpu(), H0[1])
    assert not torch.equal(W[0].cpu(), W0[0]) and not torch.equal(H[2].cpu(), H0[2])


def test_dead_component_keeps_its_column():
    capi, lib = _lib()
    B, N, C, R = 3, 150, 100, 12
    V, W0, H0 = _problems(B, N, C, R, seed=13)
    H0[1, :, 5] = 0.0                      # problem 1: (H^T H)[5,5] = 0, and l2 = 0
    W, H = W0.cuda(), H0.cuda()
    ctxs = []
    try:
        c = _batched_ctx(lib, capi, B, N, C, R, V, ctxs)
        assert lib.nmfb200_nmf_batched_cd_update(c, _p(W), _p(H), 0, 0.0, 0.0, _stream()) == 0
        torch.cuda.synchronize()
    finally:
        for c in ctxs:
            lib.nmfb200_destroy(c)
    assert torch.isfinite(W).all()
    assert torch.equal(W[1, :, 5].cpu(), W0[1, :, 5])
    assert not torch.equal(W[0, :, 5].cpu(), W0[0, :, 5])


@pytest.mark.parametrize("which", [0, 1])
def test_one_batched_update_takes_the_launches_of_one_single_update(which):
    capi, lib = _lib()
    B, N, C, R = 64, 600, 300, 40
    V, W0, H0 = _problems(B, N, C, R, seed=14)
    W, H = W0.cuda(), H0.cuda()
    Ws, Hs = W[0].clone(), H[0].clone()
    ctxs = []
    try:
        c = _batched_ctx(lib, capi, B, N, C, R, V, ctxs)
        s = ctypes.c_void_p()
        assert lib.nmfb200_nmf_create(ctypes.byref(s), torch.cuda.current_device(), N, C, R, capi.PREC_F32) == 0
        ctxs.append(s)
        assert lib.nmfb200_nmf_set_target(s, _p(V[0]), C, capi.DTYPE_F32, _stream()) == 0
        counts = []
        for call in (lambda: lib.nmfb200_nmf_cd_update(s, _p(Ws), _p(Hs), which, 0.0, 0.0, _stream()),
                     lambda: lib.nmfb200_nmf_batched_cd_update(c, _p(W), _p(H), which, 0.0, 0.0, _stream())):
            assert call() == 0                      # the first call allocates the Gram scratch
            before = lib.nmfb200_launch_count()
            assert call() == 0
            counts.append(lib.nmfb200_launch_count() - before)
        torch.cuda.synchronize()
    finally:
        for c in ctxs:
            lib.nmfb200_destroy(c)
    assert counts[0] == counts[1] == 4, counts


def test_abi_refusals():
    from torchnmf_b200.engine import CudaObservedNmfEngine, CudaSparseNmfEngine
    capi, lib = _lib()
    dev, st = torch.cuda.current_device(), _stream()
    B, N, C, R = 2, 70, 50, 8
    V = torch.rand(N, C, device="cuda")
    W, H = torch.rand(B, C, R, device="cuda"), torch.rand(B, N, R, device="cuda")
    ctxs = []

    def both(c, Wt=W, Ht=H, which=0, n_iter=1):
        return (lib.nmfb200_nmf_batched_cd_update(c, _p(Wt), _p(Ht), which, 0.0, 0.0, st),
                lib.nmfb200_nmf_batched_cd_iterate(c, _p(Wt), _p(Ht), 0.0, 0.0, n_iter, st))

    try:
        c = _batched_ctx(lib, capi, B, N, C, R, None, ctxs)
        assert both(c) == (3, 3)                                              # NMFB200_ERR_STATE before set_target
        assert lib.nmfb200_nmf_batched_set_target(c, _p(V), C, 0, capi.DTYPE_F32, st) == 0
        assert both(c) == (0, 0)
        assert lib.nmfb200_nmf_batched_cd_update(c, _p(W), _p(H), 2, 0.0, 0.0, st) == 1      # bad which
        assert lib.nmfb200_nmf_batched_cd_iterate(c, _p(W), _p(H), 0.0, 0.0, -1, st) == 1    # bad n_iter
        assert lib.nmfb200_nmf_batched_cd_update(c, None, _p(H), 0, 0.0, 0.0, st) == 1       # null factor
        # the single cd calls keep refusing a batched context
        assert lib.nmfb200_nmf_cd_update(c, _p(W), _p(H), 0, 0.0, 0.0, st) == 1
        s = ctypes.c_void_p()
        assert lib.nmfb200_nmf_create(ctypes.byref(s), dev, N, C, R, capi.PREC_F32) == 0
        ctxs.append(s)
        assert lib.nmfb200_nmf_set_target(s, _p(V), C, capi.DTYPE_F32, st) == 0
        assert both(s, W[0], H[0]) == (1, 1)                                  # NMFB200_ERR_INVALID: a single dense NMF
        Vn = torch.rand(2, 6, 20, device="cuda")
        vd, kd = (ctypes.c_int64 * 1)(20), (ctypes.c_int64 * 1)(4)
        d = ctypes.c_void_p()
        assert lib.nmfb200_nmfnd_create(ctypes.byref(d), dev, 2, 6, 1, vd, 3, kd, capi.PREC_F32) == 0
        ctxs.append(d)
        assert lib.nmfb200_nmfd_set_target(d, _p(Vn), capi.DTYPE_F32, st) == 0
        assert both(d, torch.rand(6, 3, 4, device="cuda"), torch.rand(2, 3, 17, device="cuda")) == (1, 1)      # NMFD
        bd = ctypes.c_void_p()
        assert lib.nmfb200_nmfnd_batched_create(ctypes.byref(bd), dev, 2, 2, 6, 1, vd, 3, kd) == 0
        ctxs.append(bd)
        assert lib.nmfb200_nmfd_batched_set_target(bd, _p(Vn), 0, capi.DTYPE_F32, st) == 0
        assert both(bd, torch.rand(2, 6, 3, 4, device="cuda"), torch.rand(2, 2, 3, 17, device="cuda")) == (1, 1)  # batched NMFD
        Vs = (V * (V > 0.5)).to_sparse().coalesce()
        for cls in (CudaSparseNmfEngine, CudaObservedNmfEngine):             # sparse and observed-cell targets
            eng = cls(Vs, W[0].clone(), H[0].clone())
            try:
                assert both(eng._ctx, W[0], H[0]) == (1, 1)
            finally:
                eng.close()
        assert both(None) == (1, 1)                                           # null context
    finally:
        for c in ctxs:
            lib.nmfb200_destroy(c)
