"""bfloat16 and float16 targets read in place by the kernels (no fp32 copy of V), on the H100.

A half-precision value converts to fp32 exactly, and every kernel converts V where it loads it, so a fit from a half
target must be the fit from `V.float()` bit for bit: the same W and H (torch.equal), the same n_iter, the same
last_fit_precision.  Every case below fits both from identical initial factors and compares them, over the tensor-core and
fp32 paths of NMF, NMFD, NMF2D / NMF3D, sparse_fit, host staging and a one-rank sharded fit; then the engine calls
(minmax, loss), the errors of fit's validation, the device memory a fit takes, and the C ABI's rejections.
"""
import ctypes

import pytest
import torch

from torchnmf_b200 import NMF, NMF2D, NMF3D, NMFD, _capi
from torchnmf_b200 import engine as _engine
from torchnmf_b200.engine import CudaNmfdEngine, CudaNmfEngine

pytestmark = pytest.mark.gpu

HALF = [torch.bfloat16, torch.float16]
NO_STOP = float("-inf")


def _name(d):
    return str(d).replace("torch.", "")


def _target(shape, dtype, seed, lo=0.05, heavy=False, device="cuda"):
    g = torch.Generator().manual_seed(seed)
    V = torch.exp(2.0 * torch.randn(shape, generator=g)) if heavy else torch.rand(shape, generator=g) + lo
    return V.to(dtype).to(device)


def _factors(shapes, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.rand(s, generator=g) + 0.1 for s in shapes]


def _same_fit(make, V16, fit):
    """fit(make(), V) for the half target and for V16.float(); both models must agree bit for bit.  Returns the half one."""
    out = []
    for V in (V16, V16.float()):
        m = make()
        n = fit(m, V)
        out.append((m, n))
    (a, na), (b, nb) = out
    assert na == nb, (na, nb)
    assert getattr(a, "last_fit_precision", None) == getattr(b, "last_fit_precision", None)
    for name in ("W", "H"):
        x, y = getattr(a, name).data, getattr(b, name).data
        if not torch.equal(x, y):
            bad = x != y
            raise AssertionError(f"{name}: {int(bad.sum())} of {x.numel()} entries differ")
    return a


def _nmf_case(dtype, N, C, R, beta, precision, max_iter=12, tol=NO_STOP, V=None, seed=0, module_kw=None, fit_kw=None):
    V16 = _target((N, C), dtype, seed) if V is None else V
    W0, H0 = _factors([(C, R), (N, R)], seed + 1)
    make = lambda: NMF(W=W0.clone(), H=H0.clone(), **(module_kw or {})).cuda()
    return _same_fit(make, V16, lambda m, V: m.fit(V, beta, tol, max_iter, precision=precision, **(fit_kw or {})))


# ---- NMF on the tensor cores -----------------------------------------------------------------------------------------------
TC_CASES = [  # (R, beta, precision): f16 at beta 1 (R 64, 128), f16_split, the two-output kernel, the Gram-based beta 2 stage
    (64, 1, "f16"), (128, 1, "f16"), (64, 1, "f16_split"), (64, 0.5, "f16"), (64, 2, "f16"), (48, 2, "f16"),
]


@pytest.mark.parametrize("dtype", HALF, ids=_name)
@pytest.mark.parametrize("R,beta,precision", TC_CASES)
def test_nmf_tensor_core(dtype, R, beta, precision):
    # 12 iterations: the loss of iteration 10 is folded into the next W update where the path has that fold (beta 1)
    m = _nmf_case(dtype, 640, 384, R, beta, precision)
    if beta != 2:
        assert m.last_fit_precision != "f32"


@pytest.mark.parametrize("dtype", HALF, ids=_name)
def test_nmf_tensor_core_stop_rule(dtype):
    # a finite tol: the stop rule runs on the prefetched losses
    _nmf_case(dtype, 640, 384, 64, 1, "f16", max_iter=60, tol=1e-3)


# ---- NMF on the fp32 CUDA cores ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", HALF, ids=_name)
@pytest.mark.parametrize("R", [16, 200, 300])
@pytest.mark.parametrize("beta", [0, 0.5, 1, 1.5, 2])
def test_nmf_f32(dtype, R, beta):
    m = _nmf_case(dtype, 320, 272, R, beta, "f32", max_iter=11)
    assert m.last_fit_precision == "f32"


@pytest.mark.parametrize("dtype", HALF, ids=_name)
def test_nmf_auto_heavy_tailed_falls_back(dtype):
    V16 = _target((512, 384), dtype, 3, heavy=True)
    m = _nmf_case(dtype, 512, 384, 64, 1, "auto", V=V16)
    assert m.last_fit_precision == "f32"


@pytest.mark.parametrize("dtype", HALF, ids=_name)
@pytest.mark.parametrize("R,precision", [(64, "f16"), (16, "f32")])
def test_nmf_ragged(dtype, R, precision):
    _nmf_case(dtype, 333, 257, R, 1, precision)


@pytest.mark.parametrize("dtype", HALF, ids=_name)
@pytest.mark.parametrize("R,beta,precision", [(64, 1, "f16"), (32, 2, "f32"), (300, 1, "f32")])
def test_nmf_row_strided_view(dtype, R, beta, precision):
    big = _target((400, 300), dtype, 5)
    V16 = big[:, 13:13 + 259]                       # ldv = 300 > C = 259, unit column stride, not contiguous
    assert not V16.is_contiguous() and V16.stride() == (300, 1)
    _nmf_case(dtype, 400, 259, R, beta, precision, V=V16)


@pytest.mark.parametrize("dtype", HALF, ids=_name)
@pytest.mark.parametrize("precision", ["f16", "f32"])
def test_nmf_frozen_w(dtype, precision):
    _nmf_case(dtype, 384, 320, 64, 1, precision, module_kw={"trainable_W": False})


@pytest.mark.parametrize("dtype", HALF, ids=_name)
@pytest.mark.parametrize("precision", ["f16", "f32"])
def test_nmf_regularised(dtype, precision):
    _nmf_case(dtype, 384, 320, 64, 1, precision, fit_kw={"alpha": 0.1, "l1_ratio": 0.4})


# ---- NMFD / NMF2D / NMF3D ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", HALF, ids=_name)
@pytest.mark.parametrize("R,beta,precision", [(16, 1, "f16"), (129, 1, "f16"), (16, 2, "f32"), (16, 0.5, "f32")])
def test_nmfd(dtype, R, beta, precision):
    B, C, L, T = 2, 48, 300, 7
    V16 = _target((B, C, L), dtype, 7)
    W0, H0 = _factors([(C, R, T), (B, R, L - T + 1)], 8)
    m = _same_fit(lambda: NMFD(W=W0.clone(), H=H0.clone()).cuda(), V16,
                  lambda m, V: m.fit(V, beta, NO_STOP, 12, precision=precision))
    assert (m.last_fit_precision == "f32") == (precision == "f32")


@pytest.mark.parametrize("dtype", HALF, ids=_name)
def test_nmf2d(dtype):
    V16 = _target((2, 6, 12, 40), dtype, 9)
    W0, H0 = _factors([(6, 3, 2, 5), (2, 3, 11, 36)], 10)
    _same_fit(lambda: NMF2D(W=W0.clone(), H=H0.clone()).cuda(), V16, lambda m, V: m.fit(V, 1, NO_STOP, 8))


@pytest.mark.parametrize("dtype", HALF, ids=_name)
def test_nmf3d(dtype):
    V16 = _target((1, 4, 6, 7, 30), dtype, 11)
    W0, H0 = _factors([(4, 3, 2, 3, 4), (1, 3, 5, 5, 27)], 12)
    _same_fit(lambda: NMF3D(W=W0.clone(), H=H0.clone()).cuda(), V16, lambda m, V: m.fit(V, 2, NO_STOP, 8))


# ---- sparse_fit, host staging, sharding -------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", HALF, ids=_name)
@pytest.mark.parametrize("sW,sH", [(0.5, None), (None, 0.4), (0.5, 0.4)])
def test_sparse_fit(dtype, sW, sH):
    V16 = _target((96, 80), dtype, 13)
    W0, H0 = _factors([(80, 8), (96, 8)], 14)
    _same_fit(lambda: NMF(W=W0.clone(), H=H0.clone()).cuda(), V16, lambda m, V: m.sparse_fit(V, 2, 6, False, sW, sH))


@pytest.mark.parametrize("dtype", HALF, ids=_name)
def test_host_target_host_module(dtype):
    V16 = _target((256, 192), dtype, 15, device="cpu")
    W0, H0 = _factors([(192, 32), (256, 32)], 16)
    m = _same_fit(lambda: NMF(W=W0.clone(), H=H0.clone()), V16, lambda m, V: m.fit(V, 1, NO_STOP, 12))
    assert m.W.device.type == "cpu"


@pytest.mark.parametrize("dtype", HALF, ids=_name)
def test_sharded_one_rank(dtype):
    import torch.distributed as dist
    dist.init_process_group("gloo", store=dist.HashStore(), rank=0, world_size=1)
    try:
        m = _nmf_case(dtype, 512, 256, 64, 1, "f16", fit_kw={"group": dist.group.WORLD})
        assert m.last_w_update_path == "nccl"          # the all-reduce path (peer memory needs two ranks or more)
    finally:
        dist.destroy_process_group()


# ---- engine calls, validation errors, memory, the C ABI ---------------------------------------------------------------------
@pytest.mark.parametrize("dtype", HALF, ids=_name)
@pytest.mark.parametrize("precision,betas", [("f16", (1, 0.5, 2)), ("f32", (0, 0.5, 1, 1.5, 2, 3))])
def test_engine_minmax_and_loss(dtype, precision, betas):
    V16 = _target((448, 320), dtype, 17)
    W0, H0 = _factors([(320, 64), (448, 64)], 18)
    engs = [CudaNmfEngine(V, W0.cuda(), H0.cuda(), precision) for V in (V16, V16.float())]
    try:
        assert engs[0].minmax() == engs[1].minmax()
        assert engs[0].minmax() == (float(V16.min()), float(V16.max()))
        for beta in betas:
            assert engs[0].loss(beta) == engs[1].loss(beta), beta
    finally:
        for e in engs:
            e.close()
    V16 = _target((2, 40, 200), dtype, 19)
    W0, H0 = _factors([(40, 16, 5), (2, 16, 196)], 20)
    engs = [CudaNmfdEngine(V, W0.cuda(), H0.cuda(), precision) for V in (V16, V16.float())]
    try:
        assert engs[0].minmax() == engs[1].minmax()
        for beta in (1,) if precision == "f16" else (1, 2, 0.5):
            assert engs[0].loss(beta) == engs[1].loss(beta), beta
    finally:
        for e in engs:
            e.close()


def _error_of(fn):
    try:
        fn()
    except Exception as e:       # noqa: BLE001 -- the type and message are what is compared
        return type(e), str(e)
    return None


@pytest.mark.parametrize("dtype", HALF, ids=_name)
def test_validation_errors(dtype):
    W0, H0 = _factors([(96, 8), (128, 8)], 21)
    neg = _target((128, 96), dtype, 22)
    neg[3, 5] = -1
    zero = _target((128, 96), dtype, 23)
    zero[7, 2] = 0
    for V, beta in ((neg, 1), (zero, 0), (zero, -0.5)):
        got = [_error_of(lambda: NMF(W=W0.clone(), H=H0.clone()).cuda().fit(X, beta, NO_STOP, 3)) for X in (V, V.float())]
        assert got[0] is not None and got[0] == got[1], got


def test_no_fp32_copy():
    from torchnmf_b200.engine import release_workspaces
    N, C, R = 8192, 4096, 64                          # 64 MiB of bf16
    V16 = _target((N, C), torch.bfloat16, 24)
    W0, H0 = _factors([(C, R), (N, R)], 25)
    m = NMF(W=W0, H=H0).cuda()
    for precision in ("auto", "f32"):
        release_workspaces()
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        m.fit(V16, 1, NO_STOP, 2, precision=precision)
        torch.cuda.synchronize()
        grown = torch.cuda.max_memory_allocated() - base
        assert grown < 2 * V16.numel(), (precision, grown)
    release_workspaces()


def test_set_target_rejects_bad_dtypes_and_alignment():
    lib = _capi.load()
    V16 = _target((64, 48), torch.bfloat16, 26)
    W0, H0 = _factors([(48, 8), (64, 8)], 27)
    eng = CudaNmfEngine(V16, W0.cuda(), H0.cuda(), "f32")
    st = _engine._stream(V16.device)
    p = V16.data_ptr()
    try:
        assert lib.nmfb200_nmf_set_target(eng._ctx, ctypes.c_void_p(p), 48, 3, st) == 1      # NMFB200_ERR_INVALID
        assert b"unknown target dtype 3" in lib.nmfb200_last_error()
        assert lib.nmfb200_nmf_set_target(eng._ctx, ctypes.c_void_p(p + 1), 48, _capi.DTYPE_BF16, st) == 1
        assert b"not aligned to its element size (2 bytes)" in lib.nmfb200_last_error()
        assert lib.nmfb200_nmf_set_target(eng._ctx, ctypes.c_void_p(p + 2), 48, _capi.DTYPE_F32, st) == 1
        assert b"not aligned to its element size (4 bytes)" in lib.nmfb200_last_error()
        assert eng.minmax() == (float(V16.min()), float(V16.max()))     # the registered target is unchanged
    finally:
        eng.close()
    Vd = _target((1, 8, 40), torch.float16, 28)
    Wd, Hd = _factors([(8, 4, 5), (1, 4, 36)], 29)
    eng = CudaNmfdEngine(Vd, Wd.cuda(), Hd.cuda(), "f32")
    try:
        assert lib.nmfb200_nmfd_set_target(eng._ctx, ctypes.c_void_p(Vd.data_ptr()), 3, st) == 1
        assert b"unknown target dtype 3" in lib.nmfb200_last_error()
        assert lib.nmfb200_nmfd_set_target(eng._ctx, ctypes.c_void_p(Vd.data_ptr() + 1), _capi.DTYPE_F16, st) == 1
        assert b"not aligned to its element size (2 bytes)" in lib.nmfb200_last_error()
    finally:
        eng.close()
