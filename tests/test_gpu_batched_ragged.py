"""BatchedNMF.fit(V, ..., lengths=L) on the H100: problem b of a ragged batch is, bit for bit, the single fp32 fit of its
real rows -- `NMF(W=W0[b], H=H0[b, :L]).fit(V[b, :L], ..., precision="f32")` -- with its n_iter, for every beta, rank
branch and target dtype, while rows L: of V (NaN here) are never read and rows L: of H (a sentinel) never written.  Also the
C ABI of the ragged context (include/nmf_b200.h: nmfb200_nmf_batched_create_ragged)."""
import ctypes
import os

import pytest
import torch

from torchnmf_b200 import NMF, BatchedNMF, _capi

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SENTINEL = 3.25
ERR_INVALID = 1                       # include/nmf_b200.h: NMFB200_ERR_INVALID
N, C = 300, 96
LENGTHS = [1, 63, 64, 65, N]          # chunk counts of the W update 1, 1, 1, 2, 5 (test_lengths_change_the_plans)


def _inputs(lengths, N=N, C=C, R=16, seed=0, dtype=torch.float32):
    B = len(lengths)
    g = torch.Generator().manual_seed(seed)
    V = (torch.rand(B, N, C, generator=g) * torch.linspace(0.3, 2.0, B).view(B, 1, 1) + 0.05).to(dtype)
    W0 = torch.rand(B, C, R, generator=g) + 0.1
    H0 = torch.rand(B, N, R, generator=g) + 0.1
    for b, L in enumerate(lengths):
        V[b, L:] = float("nan")
        H0[b, L:] = SENTINEL
    return V, W0, H0


def _batched(V, W0, H0, lengths, trainable_W=True, trainable_H=True, **kw):
    m = BatchedNMF(W=W0, H=H0, trainable_W=trainable_W, trainable_H=trainable_H).cuda()
    n = m.fit(V, lengths=lengths, **kw)
    assert m.last_fit_precision == "f32"
    return n, m.W.data.cpu(), m.H.data.cpu()


def _check_against_loop(V, W0, H0, lengths, n, W, H, trainable_W=True, trainable_H=True, **kw):
    """Problem by problem against the single fp32 fit of its rows; returns the single fits' iteration counts."""
    counts = []
    for b, L in enumerate(lengths):
        s = NMF(W=W0[b], H=H0[b, :L], trainable_W=trainable_W, trainable_H=trainable_H).cuda()
        counts.append(s.fit(V[b, :L], precision="f32", **kw))
        assert int(n[b]) == counts[-1], (b, L, int(n[b]), counts[-1])
        assert torch.equal(W[b], s.W.data.cpu()), (b, L, (W[b] - s.W.data.cpu()).abs().max())
        assert torch.equal(H[b, :L], s.H.data.cpu()), (b, L, (H[b, :L] - s.H.data.cpu()).abs().max())
        assert bool((H[b, L:] == SENTINEL).all()), (b, L)
    return counts


def test_lengths_change_the_plans():
    plans = [_capi.nmf_plan(L, C, 16) for L in LENGTHS]
    assert len({p["nch_w"] for p in plans}) >= 3
    big = [_capi.nmf_plan(L, 1024, 16) for L in (65, 4200)]
    assert big[0]["nch_h"] != big[1]["nch_h"] and big[0]["loss_chunks"] != big[1]["loss_chunks"]


@pytest.mark.parametrize("R", [1, 16, 17, 64, 256])
@pytest.mark.parametrize("beta", [0, 0.5, 1, 1.5, 2, 3])
def test_bit_exact_against_the_loop(beta, R):
    V, W0, H0 = _inputs(LENGTHS, R=R, seed=R)
    kw = dict(beta=beta, tol=1e-3, max_iter=40)
    n, W, H = _batched(V.cuda(), W0, H0, LENGTHS, **kw)
    _check_against_loop(V.cuda(), W0, H0, LENGTHS, n, W, H, **kw)


def test_problems_stop_at_different_iterations():
    lengths = [1, 63, 64, 65, N, 200, 130]
    V, W0, H0 = _inputs(lengths, seed=5)
    kw = dict(beta=1, tol=2e-3, max_iter=200)
    n, W, H = _batched(V.cuda(), W0, H0, lengths, **kw)
    counts = _check_against_loop(V.cuda(), W0, H0, lengths, n, W, H, **kw)
    assert len(set(counts)) >= 3 and max(counts) < 200, counts


def test_different_h_chunk_counts():
    lengths = [65, 4200, 1, 2000]
    V, W0, H0 = _inputs(lengths, N=4200, C=1024, seed=6)
    for beta in (1, 2):
        kw = dict(beta=beta, tol=1e-4, max_iter=20)
        n, W, H = _batched(V.cuda(), W0, H0, lengths, **kw)
        _check_against_loop(V.cuda(), W0, H0, lengths, n, W, H, **kw)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_half_targets_in_place_strided(dtype):
    V, W0, H0 = _inputs(LENGTHS, seed=7, dtype=dtype)
    big = torch.full((len(LENGTHS), N + 3, C + 5), float("nan"), dtype=dtype, device="cuda")
    big[:, :N, :C] = V.cuda()
    Vs = big[:, :N, :C]                                     # rows C + 5 apart, problems (N + 3) (C + 5) apart
    for beta in (0.5, 1, 2):
        kw = dict(beta=beta, tol=1e-3, max_iter=30)
        n, W, H = _batched(Vs, W0, H0, LENGTHS, **kw)
        _check_against_loop(Vs, W0, H0, LENGTHS, n, W, H, **kw)


@pytest.mark.parametrize("frozen", ["W", "H"])
def test_frozen_factor(frozen):
    V, W0, H0 = _inputs(LENGTHS, seed=8)
    tk = dict(trainable_W=frozen != "W", trainable_H=frozen != "H")
    for beta in (1, 2):
        kw = dict(beta=beta, tol=1e-3, max_iter=30)
        n, W, H = _batched(V.cuda(), W0, H0, LENGTHS, **tk, **kw)
        _check_against_loop(V.cuda(), W0, H0, LENGTHS, n, W, H, **tk, **kw)
        if frozen == "W":
            assert torch.equal(W, W0)


@pytest.mark.parametrize("beta", [0.5, 1, 2])
def test_alpha_l1_ratio(beta):
    V, W0, H0 = _inputs(LENGTHS, seed=9)
    kw = dict(beta=beta, tol=1e-3, max_iter=30, alpha=0.05, l1_ratio=0.4)
    n, W, H = _batched(V.cuda(), W0, H0, LENGTHS, **kw)
    _check_against_loop(V.cuda(), W0, H0, LENGTHS, n, W, H, **kw)


def test_host_and_float64_modules_keep_their_padding():
    V, W0, H0 = _inputs(LENGTHS, seed=10)
    ref_n, ref_W, ref_H = _batched(V.cuda(), W0, H0, LENGTHS, beta=1, tol=1e-3, max_iter=30)
    m = BatchedNMF(W=W0, H=H0).double()                                  # a float64 module on the host
    m.H.data[:, :, 0] += torch.where(m.H.data[:, :, 0] == SENTINEL, 1 / 3, 0.0)   # padding values fp32 cannot hold
    H64 = m.H.data.clone()
    n = m.fit(V.double(), beta=1, tol=1e-3, max_iter=30, lengths=torch.tensor(LENGTHS))
    assert torch.equal(n, ref_n) and torch.equal(m.W.data, ref_W.double())
    for b, L in enumerate(LENGTHS):
        assert torch.equal(m.H.data[b, :L], ref_H[b, :L].double())
        assert torch.equal(m.H.data[b, L:], H64[b, L:])


def test_all_lengths_n_equal_the_uniform_batch():
    V, W0, H0 = _inputs([N] * 4, seed=11)
    for beta in (0.5, 1, 2):
        kw = dict(beta=beta, tol=1e-3, max_iter=40)
        n, W, H = _batched(V.cuda(), W0, H0, [N] * 4, **kw)
        m = BatchedNMF(W=W0, H=H0).cuda()
        n0 = m.fit(V.cuda(), **kw)
        assert torch.equal(n, n0) and torch.equal(W, m.W.data.cpu()) and torch.equal(H, m.H.data.cpu())


def test_lengths_on_the_device():
    V, W0, H0 = _inputs(LENGTHS, seed=12)
    n1, W1, H1 = _batched(V.cuda(), W0, H0, LENGTHS, beta=2, max_iter=20)
    n2, W2, H2 = _batched(V.cuda(), W0, H0, torch.tensor(LENGTHS, device="cuda"), beta=2, max_iter=20)
    assert torch.equal(n1, n2) and torch.equal(W1, W2) and torch.equal(H1, H2)


# ---- C ABI ----------------------------------------------------------------------------------------------------------------

def _create(B, N, C, R, lengths):
    lib = _capi.load()
    ctx = ctypes.c_void_p()
    lens = (ctypes.c_int64 * len(lengths))(*lengths)
    rc = lib.nmfb200_nmf_batched_create_ragged(ctypes.byref(ctx), 0, B, N, C, R, lens)
    return rc, ctx


def test_grid_x_refusal_from_shapes():
    # 2048 problems of one row over 2^26 columns: each W update takes 2^20 row blocks, 2^31 together -- past grid x
    lib = _capi.load()
    before = lib.nmfb200_launch_count()
    rc, ctx = _create(2048, 1, 1 << 26, 1, [1] * 2048)
    assert rc == ERR_INVALID and not ctx and "grid x" in lib.nmfb200_last_error().decode()
    assert lib.nmfb200_launch_count() == before


def test_abi_symbols_refusals_and_header():
    lib = _capi.load()
    assert hasattr(lib, "nmfb200_nmf_batched_create_ragged")
    assert lib.nmfb200_abi_version() == 2
    lens = (ctypes.c_int64 * 2)(3, 4)
    assert lib.nmfb200_nmf_batched_create_ragged(None, 0, 2, 4, 5, 2, lens) == ERR_INVALID
    ctx = ctypes.c_void_p()
    assert lib.nmfb200_nmf_batched_create_ragged(ctypes.byref(ctx), 0, 2, 4, 5, 2, None) == ERR_INVALID
    for bad in ((0, 4), (3, 5), (-1, 2)):
        assert _create(2, 4, 5, 2, bad)[0] == ERR_INVALID
    assert _create(1, 4, 5, 257, [4])[0] == ERR_INVALID
    assert lib.nmfb200_nmf_batched_set_target(None, None, 5, 20, 0, None) == ERR_INVALID
    rc, ctx = _create(2, 4, 5, 2, [3, 4])
    assert rc == 0 and ctx
    try:
        V = torch.rand(2, 4, 5, device="cuda")
        W = torch.rand(2, 5, 2, device="cuda")
        H = torch.rand(2, 4, 2, device="cuda")
        s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        assert lib.nmfb200_nmf_batched_set_target(ctx, ctypes.c_void_p(V.data_ptr()), 5, 20, 0, s) == 0
        for call in (lambda: lib.nmfb200_nmf_batched_cd_update(ctx, ctypes.c_void_p(W.data_ptr()),
                                                               ctypes.c_void_p(H.data_ptr()), 0, 0.0, 0.0, s),
                     lambda: lib.nmfb200_nmf_batched_cd_iterate(ctx, ctypes.c_void_p(W.data_ptr()),
                                                                ctypes.c_void_p(H.data_ptr()), 0.0, 0.0, 1, s)):
            assert call() == ERR_INVALID
        torch.cuda.synchronize()
    finally:
        lib.nmfb200_destroy(ctx)
    with open(os.path.join(ROOT, "include", "nmf_b200.h")) as f:
        header = f.read()
    assert "int nmfb200_nmf_batched_create_ragged(nmfb200_ctx** out, int device, int64_t B, int64_t N, int64_t C, " \
           "int64_t R,\n                                      const int64_t* lengths);" in header
