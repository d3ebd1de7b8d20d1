"""BatchedNMFD / BatchedNMF2D / BatchedNMF3D .fit(V, ..., lengths=L) on the H100: problem p of a ragged batch is, bit for
bit, the single fp32 fit of its real positions along the last convolved axis -- `NMFD(W=W0[p], H=H0[p, ..., :L - T + 1])
.fit(V[p, ..., :L], ..., precision="f32")` -- with its n_iter, for every beta, rank tile, kernel length and target dtype,
while positions L: of V (NaN here) are never read and positions L - T + 1: of H (a sentinel) never written.  Also the C
ABI of the ragged context (include/nmf_b200.h: nmfb200_nmfnd_batched_create_ragged)."""
import ctypes
import os

import pytest
import torch

from torchnmf_b200 import NMFD, NMF2D, NMF3D, BatchedNMFD, BatchedNMF2D, BatchedNMF3D, _capi

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SENTINEL = 3.25
ERR_INVALID = 1                       # include/nmf_b200.h: NMFB200_ERR_INVALID
SINGLE = {BatchedNMFD: NMFD, BatchedNMF2D: NMF2D, BatchedNMF3D: NMF3D}


def _inputs(lengths, outer, C, R, K, B=1, seed=0, dtype=torch.float32):
    """V (P, B, C, *outer, X) padded to X = max(lengths) with NaN, W0 (P, C, R, *K), H0 (P, B, R, *J) padded with the
    sentinel; problem p's noise level grows with p, so that the problems stop at different counts."""
    P, X = len(lengths), max(lengths)
    g = torch.Generator().manual_seed(seed)
    shape = (P, B, C) + tuple(outer) + (X,)
    J = tuple(x - k + 1 for x, k in zip(tuple(outer) + (X,), K))
    level = torch.linspace(0.05, 1.5, P).view(P, *([1] * (len(shape) - 1)))
    V = (torch.rand(shape, generator=g) * level + torch.rand(shape, generator=g).pow(4) + 0.05).to(dtype)
    W0 = torch.rand((P, C, R) + tuple(K), generator=g) + 0.1
    H0 = torch.rand((P, B, R) + J, generator=g) + 0.1
    for p, L in enumerate(lengths):
        V[p, ..., L:] = float("nan")
        H0[p, ..., L - K[-1] + 1:] = SENTINEL
    return V, W0, H0


def _batched(cls, V, W0, H0, lengths, trainable_W=True, trainable_H=True, cuda=True, **kw):
    m = cls(W=W0, H=H0, trainable_W=trainable_W, trainable_H=trainable_H)
    if cuda:
        m = m.cuda()
    n = m.fit(V, lengths=lengths, **kw)
    assert m.last_fit_precision == "f32"
    return n, m.W.data.cpu(), m.H.data.cpu()


def _check_against_loop(cls, V, W0, H0, lengths, n, W, H, trainable_W=True, trainable_H=True, **kw):
    """Problem by problem against the single fp32 fit of its real positions; returns the single fits' counts."""
    T = W0.shape[-1]
    counts = []
    for p, L in enumerate(lengths):
        lin = L - T + 1
        s = SINGLE[cls](W=W0[p], H=H0[p, ..., :lin].contiguous(), trainable_W=trainable_W, trainable_H=trainable_H).cuda()
        counts.append(s.fit(V[p, ..., :L].contiguous(), precision="f32", **kw))
        assert int(n[p]) == counts[-1], (p, L, int(n[p]), counts[-1])
        assert torch.equal(W[p].float(), s.W.data.cpu()), (p, L, (W[p].float() - s.W.data.cpu()).abs().max())
        assert torch.equal(H[p, ..., :lin].float(), s.H.data.cpu()), (p, L, (H[p, ..., :lin].float() - s.H.data.cpu()).abs().max())
        assert bool((H[p, ..., lin:] == SENTINEL).all()), (p, L)
    return counts


# 1-D: C = 48, T = 16, padded to 300; recon grid x 1, 2, 2, 4, 5, dgrad grid x 1, 1, 2, 3, 5 (T = L: one H position)
LENGTHS = [16, 79, 80, 200, 300]


@pytest.mark.parametrize("beta", [0, 0.5, 1, 1.5, 2, 3])
def test_nmfd_each_problem_is_its_own_fit(beta):
    V, W0, H0 = _inputs(LENGTHS, (), 48, 8, (16,), seed=1)
    kw = dict(beta=beta, tol=2e-3, max_iter=120)
    n, W, H = _batched(BatchedNMFD, V, W0, H0, LENGTHS, **kw)
    counts = _check_against_loop(BatchedNMFD, V, W0, H0, LENGTHS, n, W, H, **kw)
    if beta in (0.5, 1, 1.5):              # the problems stop at their own counts (the others all run to max_iter here)
        assert len(set(counts)) >= 3, counts


# T = 16: the W update's ratio stage reads each problem's partial slabs as float4 (vec4_w), at per-problem offsets that
# odd ranks and R = 6 would leave unaligned if the slabs were packed without rounding
@pytest.mark.parametrize("T", [5, 16])
@pytest.mark.parametrize("R", [1, 6, 8, 16, 17, 64, 256])
def test_dgrad_row_tiles(R, T):
    lengths = [129, 20, 64, 65]
    V, W0, H0 = _inputs(lengths, (), 24, R, (T,), B=2, seed=R)
    assert _capi.nmfd_plan(2, 24, [129], R, [T])["vec4_w"] == (T % 4 == 0)
    kw = dict(beta=1, tol=1e-3, max_iter=40)
    n, W, H = _batched(BatchedNMFD, V, W0, H0, lengths, **kw)
    _check_against_loop(BatchedNMFD, V, W0, H0, lengths, n, W, H, **kw)


@pytest.mark.parametrize("R", [5, 6])
def test_long_problem_ahead_of_a_short_one_with_float4_slabs(R):
    """B = 1, C = 513, T = 16: the first problem's dgrad slabs (17 splits x R x 2001 floats) are no multiple of 4 floats,
    so the second problem's partials start 16-byte aligned only because every problem's slabs are rounded up."""
    lengths = [2016, 300]
    assert 17 * R * 2001 % 4 != 0 and _capi.nmfd_plan(1, 513, [2016], R, [16])["dgrad_nsplit"] == 17
    V, W0, H0 = _inputs(lengths, (), 513, R, (16,), seed=20 + R)
    for beta in (1, 2):
        kw = dict(beta=beta, tol=1e-3, max_iter=30)
        n, W, H = _batched(BatchedNMFD, V, W0, H0, lengths, **kw)
        _check_against_loop(BatchedNMFD, V, W0, H0, lengths, n, W, H, **kw)


@pytest.mark.parametrize("T, lengths", [(1, [1, 64, 65, 150]), (70, [70, 133, 134, 200])])
def test_kernel_lengths(T, lengths):
    V, W0, H0 = _inputs(lengths, (), 20, 6, (T,), seed=T)
    for beta in (1, 2):
        kw = dict(beta=beta, tol=1e-3, max_iter=40)
        n, W, H = _batched(BatchedNMFD, V, W0, H0, lengths, **kw)
        _check_against_loop(BatchedNMFD, V, W0, H0, lengths, n, W, H, **kw)


def test_plans_differ_across_lengths():
    """The dgrad splits and the recon grid follow each problem's length: the bit tests below run distinct plans."""
    plans = [_capi.nmfd_plan(1, 513, [L], 8, [16]) for L in (115, 715, 2015)]
    assert len({p["dgrad_nsplit"] for p in plans}) == 3, [p["dgrad_nsplit"] for p in plans]
    assert len({p["recon_grid"][0] for p in plans}) == 3
    assert len({p["dgrad_grid"][0] for p in plans}) == 3


def test_spectrogram_shape_with_distinct_plans():
    lengths = [115, 715, 2015]
    V, W0, H0 = _inputs(lengths, (), 513, 8, (16,), seed=7)
    for beta in (1, 0.5):
        kw = dict(beta=beta, tol=1e-3, max_iter=30)
        n, W, H = _batched(BatchedNMFD, V, W0, H0, lengths, **kw)
        _check_against_loop(BatchedNMFD, V, W0, H0, lengths, n, W, H, **kw)


@pytest.mark.parametrize("cls, outer, K, lengths", [
    (BatchedNMF2D, (6,), (2, 5), [5, 40, 68, 90]),
    (BatchedNMF3D, (3, 4), (2, 1, 3), [3, 30, 66, 80]),
])
def test_nmf2d_nmf3d(cls, outer, K, lengths):
    V, W0, H0 = _inputs(lengths, outer, 7, 5, K, B=2, seed=3)
    for beta in (1, 1.5):
        kw = dict(beta=beta, tol=1e-3, max_iter=40)
        n, W, H = _batched(cls, V, W0, H0, lengths, **kw)
        _check_against_loop(cls, V, W0, H0, lengths, n, W, H, **kw)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_half_targets_read_in_place(dtype):
    V, W0, H0 = _inputs(LENGTHS, (), 32, 8, (16,), seed=5, dtype=dtype)
    for beta in (1, 2):
        kw = dict(beta=beta, tol=1e-3, max_iter=40)
        n, W, H = _batched(BatchedNMFD, V.cuda(), W0, H0, LENGTHS, **kw)
        _check_against_loop(BatchedNMFD, V.cuda(), W0, H0, LENGTHS, n, W, H, **kw)


@pytest.mark.parametrize("frozen", ["W", "H"])
def test_frozen_factor_and_regularisation(frozen):
    V, W0, H0 = _inputs(LENGTHS, (), 32, 8, (16,), seed=9)
    kw = dict(beta=1.5, tol=1e-3, max_iter=40, alpha=0.05, l1_ratio=0.3,
              trainable_W=frozen != "W", trainable_H=frozen != "H")
    n, W, H = _batched(BatchedNMFD, V, W0, H0, LENGTHS, **kw)
    _check_against_loop(BatchedNMFD, V, W0, H0, LENGTHS, n, W, H, **kw)


@pytest.mark.parametrize("module", ["host", "float64"])
def test_staged_modules_keep_their_padding(module):
    V, W0, H0 = _inputs(LENGTHS, (), 32, 8, (16,), seed=11)
    kw = dict(beta=1, tol=1e-3, max_iter=40)
    if module == "host":
        n, W, H = _batched(BatchedNMFD, V, W0, H0, LENGTHS, cuda=False, **kw)
    else:
        m = BatchedNMFD(W=W0, H=H0).double().cuda()
        n = m.fit(V.double().cuda(), lengths=LENGTHS, **kw)
        W, H = m.W.data.cpu(), m.H.data.cpu()
        assert W.dtype == torch.float64
    _check_against_loop(BatchedNMFD, V, W0, H0, LENGTHS, n, W, H, **kw)


def test_lengths_on_the_device_and_full_lengths():
    V, W0, H0 = _inputs(LENGTHS, (), 32, 8, (16,), seed=13)
    kw = dict(beta=1, tol=1e-3, max_iter=40)
    ref = _batched(BatchedNMFD, V, W0, H0, LENGTHS, **kw)
    got = _batched(BatchedNMFD, V, W0, H0, torch.tensor(LENGTHS, device="cuda"), **kw)
    assert all(torch.equal(a, b) for a, b in zip(ref, got))
    full = [300] * 4
    Vf, Wf, Hf = _inputs(full, (), 32, 8, (16,), seed=13)
    m = BatchedNMFD(W=Wf, H=Hf).cuda()
    n_uni = m.fit(Vf.cuda(), **kw)
    n, W, H = _batched(BatchedNMFD, Vf, Wf, Hf, full, **kw)
    assert torch.equal(n, n_uni) and torch.equal(W, m.W.data.cpu()) and torch.equal(H, m.H.data.cpu())


def test_checks_look_at_the_real_positions_only():
    V, W0, H0 = _inputs(LENGTHS, (), 16, 4, (16,), seed=2)
    for p, L in enumerate(LENGTHS):
        V[p, ..., L:] = -1.0                                    # negative padding: not part of any problem
    _batched(BatchedNMFD, V, W0, H0, LENGTHS, beta=1, max_iter=10)
    Vn = V.clone()
    Vn[1, 0, 3, 5] = -0.5
    with pytest.raises(AssertionError):
        _batched(BatchedNMFD, Vn, W0, H0, LENGTHS, beta=1, max_iter=10)
    for p, L in enumerate(LENGTHS):
        V[p, ..., L:] = 0.0                                     # zero padding: beta <= 0 is still fine
    _batched(BatchedNMFD, V, W0, H0, LENGTHS, beta=0, max_iter=10)
    V[2, 0, 1, 10] = 0.0
    with pytest.raises(ValueError):
        _batched(BatchedNMFD, V, W0, H0, LENGTHS, beta=0, max_iter=10)


# ---- C ABI -----------------------------------------------------------------------------------------------------------

def _create(lib, P, B, C, X, R, K, lengths):
    ctx = ctypes.c_void_p()
    nd = len(X)
    lens = None if lengths is None else (ctypes.c_int64 * len(lengths))(*lengths)
    rc = lib.nmfb200_nmfnd_batched_create_ragged(ctypes.byref(ctx), 0, P, B, C, nd, (ctypes.c_int64 * nd)(*X), R,
                                                 (ctypes.c_int64 * nd)(*K), lens)
    return rc, ctx


def test_capi_refusals_and_plca():
    lib = _capi.load()
    assert hasattr(lib, "nmfb200_nmfnd_batched_create_ragged")
    for lengths in (None, [3, 40], [4, 41], [0, 40]):         # T = 4, L = 40
        rc, ctx = _create(lib, 2, 1, 6, [40], 3, [4], lengths)
        assert rc == ERR_INVALID and not ctx.value, lengths
    rc, ctx = _create(lib, 0, 1, 6, [40], 3, [4], [])
    assert rc == ERR_INVALID
    rc, ctx = _create(lib, 2, 1, 6, [40], 3, [4], [4, 40])
    assert rc == 0 and ctx.value
    try:
        V = torch.rand(2, 1, 6, 40, device="cuda")
        W = torch.rand(2, 6, 3, 4, device="cuda")
        H = torch.rand(2, 1, 3, 37, device="cuda")
        Z = torch.rand(2, 3, device="cuda")
        stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        assert lib.nmfb200_nmfd_batched_set_target(ctx, ctypes.c_void_p(V.data_ptr()), V[0].numel(), 0, stream) == 0
        n = int(lib.nmfb200_plca_work_numel(ctx))
        work = torch.empty(max(n, 1), device="cuda")
        assert lib.nmfb200_plca_iterate(ctx, W.data_ptr(), H.data_ptr(), Z.data_ptr(), H.data_ptr(), work.data_ptr(), 7,
                                        None, None, None, 1, stream) == ERR_INVALID
        loss = torch.zeros(2, dtype=torch.float64, device="cuda")
        assert lib.nmfb200_plca_loss(ctx, W.data_ptr(), H.data_ptr(), Z.data_ptr(), loss.data_ptr(),
                                     stream) == ERR_INVALID
    finally:
        lib.nmfb200_destroy(ctx)


def test_header_declares_the_ragged_create():
    with open(os.path.join(ROOT, "include", "nmf_b200.h")) as f:
        text = f.read()
    assert "int nmfb200_nmfnd_batched_create_ragged(nmfb200_ctx** out, int device, int64_t P, int64_t B, int64_t C," in text
