"""Batched NMFD / NMF2D / NMF3D on the GPU: every problem's raw terms and loss against float64 at the tile edges, then whole
fits bit for bit against single `.fit(precision="f32")` fits, at the line, split and element-count limits, and next to
cached single-problem workspaces."""
import math

import pytest
import torch
import torch.nn.functional as F

from torchnmf_b200 import NMFD, NMF2D, NMF3D, BatchedNMFD, BatchedNMF2D, BatchedNMF3D, _capi
from torchnmf_b200 import engine as E

pytestmark = pytest.mark.gpu

EPS = float(torch.finfo(torch.float32).eps)
SENTINEL = -12345.0
CONV = {1: F.conv1d, 2: F.conv2d, 3: F.conv3d}
SINGLE = {1: NMFD, 2: NMF2D, 3: NMF3D}
BATCHED = {1: BatchedNMFD, 2: BatchedNMF2D, 3: BatchedNMF3D}


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda", 0)


def _recon64(H, W):
    K = W.shape[2:]
    return CONV[len(K)](H, W.flip(tuple(range(2, W.dim()))), padding=tuple(k - 1 for k in K))


def _phi64(V, S, beta):
    if beta == 1:
        return V / (S + EPS), None
    if beta == 2:
        return V, S
    x = S + EPS
    return V * x ** (beta - 2), x ** (beta - 1)


def _beta_div64(S, V, beta):
    if beta == 1:
        return float((V * ((V + EPS).log() - (S + EPS).log()) - V + S).sum())
    if beta == 2:
        return float(((S - V) ** 2).sum() * 0.5)
    if beta == 0:
        te, xe = V + EPS, S + EPS
        return float((te / xe - te.log() + xe.log() - 1).sum())
    x = S + EPS
    return float(((V ** beta) + (beta - 1) * x ** beta - beta * V * x ** (beta - 1)).sum() / (beta * (beta - 1)))


def _grads64(H, W, G):
    """(d<recon, G>/dW, d<recon, G>/dH) in float64."""
    W, H = W.clone().requires_grad_(True), H.clone().requires_grad_(True)
    (_recon64(H, W) * G).sum().backward()
    return W.grad, H.grad


def _problem(P, B, C, X, R, K, seed, dev):
    g = torch.Generator().manual_seed(seed)
    J = tuple(x - k + 1 for x, k in zip(X, K))
    nk = math.prod(K)
    V = (torch.rand(P, B, C, *X, generator=g) + 0.05).to(dev)
    W = (torch.rand(P, C, R, *K, generator=g) / math.sqrt(R * nk) + 0.01).to(dev)
    H = (torch.rand(P, B, R, *J, generator=g) / math.sqrt(R * nk) + 0.01).to(dev)
    return V, W, H


# (C, X, K): channels and kernels across the row tiles (4 ... 64) and wgrad's TP = roundup(min(T, 64), 4)
SHAPES = [(3, (9,), (1,)), (17, (40,), (5,)), (65, (100,), (64,)), (3, (90,), (65,)),
          (5, (7, 30), (2, 5)), (17, (6, 9), (3, 1)), (3, (4, 5, 20), (2, 3, 5)), (4, (3, 4, 12), (1, 2, 1))]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: f"C{s[0]}_X{'x'.join(map(str, s[1]))}_K{'x'.join(map(str, s[2]))}")
@pytest.mark.parametrize("R", [1, 16, 17, 64, 256])
@pytest.mark.parametrize("beta", [0, 0.5, 1, 2, 3])
def test_raw_terms_and_loss_per_problem(beta, R, shape):
    dev = _dev()
    C, X, K = shape
    P, B = 4, 2
    V, W, H = _problem(P, B, C, X, R, K, R * 10 + int(beta * 2) + C, dev)
    active = torch.tensor([1, 0, 1, 1], dtype=torch.bool)
    eng = E.CudaBatchedNmfdEngine(V, W, H)
    try:
        eng.set_active(active)
        for which in (0, 1):
            n = int(eng._lib.nmfb200_raw_terms_numel(eng._ctx, which, float(beta)))
            buf = torch.full((n,), SENTINEL, dtype=torch.float32, device=dev)
            eng._raw_terms_into(which, beta, buf)
            f = W if which == 0 else H
            num = buf[:f.numel()].view(f.shape)
            den = buf[f.numel():].view(P, R) if beta == 1 else buf[f.numel():].view(f.shape)
            for p in range(P):
                if not active[p]:
                    assert bool((num[p] == SENTINEL).all()) and bool((den[p] == SENTINEL).all())
                    continue
                V64, W64, H64 = V[p].double().cpu(), W[p].double().cpu(), H[p].double().cpu()
                Pn, Pp = _phi64(V64, _recon64(H64, W64), beta)
                want_n = _grads64(H64, W64, Pn)[which]
                assert torch.allclose(num[p].double().cpu(), want_n, rtol=2e-5, atol=1e-6 * float(want_n.abs().max())), \
                    (p, which)
                if beta == 1:
                    other = H64 if which == 0 else W64
                    want_d = other.sum([d for d in range(other.dim()) if d != 1])
                else:
                    want_d = _grads64(H64, W64, Pp)[which]
                assert torch.allclose(den[p].double().cpu(), want_d, rtol=2e-5, atol=1e-6 * float(want_d.abs().max())), \
                    (p, which)
        eng._loss.fill_(SENTINEL)
        d = eng.losses(beta)
        for p in range(P):
            if not active[p]:
                assert d[p] == SENTINEL
                continue
            want = _beta_div64(_recon64(H[p].double().cpu(), W[p].double().cpu()), V[p].double().cpu(), beta)
            assert math.isclose(float(d[p]), want, rel_tol=1e-4, abs_tol=1e-6 * V[p].numel()), (p, float(d[p]), want)
        # bit for bit what a single-problem fp32 context computes
        for p in (0, 3):
            single = E.CudaNmfdEngine(V[p], W[p].clone(), H[p].clone(), "f32")
            try:
                for which in (0, 1):
                    sn, sd = single.raw_terms(which, beta)
                    bn, bd = eng.raw_terms(which, beta)
                    assert torch.equal(sn, bn[p]) and torch.equal(sd.reshape(bd[p].shape), bd[p]), (p, which)
                assert float(single.loss(beta)) == float(eng.losses(beta)[p])
            finally:
                single.close()
    finally:
        eng.close()


def _single_fits(nd, V, W0, H0, problems=None, trainable_W=True, trainable_H=True, **kw):
    out = []
    for p in (range(W0.shape[0]) if problems is None else problems):
        Vp = V if V.dim() == nd + 2 else V[p]
        m = SINGLE[nd](W=W0[p], H=H0[p], trainable_W=trainable_W, trainable_H=trainable_H).to(W0.device)
        n = m.fit(Vp, precision="f32", **kw)
        assert m.last_fit_precision == "f32"
        out.append((n, m.W.data, m.H.data))
    return out


def _check_batched(nd, V, W0, H0, problems=None, trainable_W=True, trainable_H=True, **kw):
    m = BATCHED[nd](W=W0, H=H0, trainable_W=trainable_W, trainable_H=trainable_H).to(W0.device)
    n = m.fit(V, **kw)
    assert n.dtype == torch.int64 and m.last_fit_precision == "f32"
    singles = _single_fits(nd, V, W0, H0, problems, trainable_W, trainable_H, **kw)
    for p, (npb, Wp, Hp) in zip(range(W0.shape[0]) if problems is None else problems, singles):
        assert int(n[p]) == npb, (p, int(n[p]), npb)
        assert torch.equal(m.W.data[p], Wp), p
        assert torch.equal(m.H.data[p], Hp), p
    return n


FIT_SHAPES = {1: (12, (60,), (7,)), 2: (5, (9, 24), (2, 5)), 3: (4, (4, 5, 16), (2, 2, 3))}


@pytest.mark.parametrize("nd", [1, 2, 3])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
@pytest.mark.parametrize("beta", [0.5, 1, 2])
def test_fits_bit_equal_to_single_fits(beta, dtype, nd):
    dev = _dev()
    C, X, K = FIT_SHAPES[nd]
    V, W0, H0 = _problem(5, 2, C, X, 6, K, 7 + nd, dev)
    V = (V * torch.linspace(0.3, 3, 5, device=dev).view(5, *([1] * (nd + 2)))).to(dtype)
    n = _check_batched(nd, V, W0, H0, beta=beta, tol=2e-3, max_iter=120)
    assert int(n.max()) <= 120


@pytest.mark.parametrize("nd", [1, 2])
def test_shared_target_penalties_and_frozen_factors(nd):
    dev = _dev()
    C, X, K = FIT_SHAPES[nd]
    V, W0, H0 = _problem(4, 2, C, X, 5, K, 11, dev)
    _check_batched(nd, V[2], W0, H0, beta=1, tol=1e-3, max_iter=60)                        # one shared target
    _check_batched(nd, V[1].expand(4, *V[1].shape), W0, H0, beta=2, tol=1e-3, max_iter=40)   # expanded: stride 0
    _check_batched(nd, V, W0, H0, beta=0.5, tol=1e-3, max_iter=50, alpha=0.1, l1_ratio=0.4)
    _check_batched(nd, V, W0, H0, beta=1, tol=1e-3, max_iter=40, trainable_W=False)
    _check_batched(nd, V, W0, H0, beta=2, tol=1e-3, max_iter=40, trainable_H=False)
    # a strided problem axis (every problem's block contiguous) is read in place
    Vs = torch.zeros(4, 2 * V[0].numel(), device=dev)
    Vs[:, :V[0].numel()] = V.reshape(4, -1)
    Vv = Vs[:, :V[0].numel()].view(V.shape)
    assert Vv.stride(0) == 2 * V[0].numel()
    _check_batched(nd, Vv, W0, H0, beta=1, tol=1e-3, max_iter=40)


def test_host_module_and_p1_equal_single_fit():
    dev = _dev()
    C, X, K = FIT_SHAPES[1]
    V, W0, H0 = _problem(3, 2, C, X, 4, K, 5, dev)
    m = BatchedNMFD(W=W0.cpu(), H=H0.cpu())                                     # host module: staged and written back
    n = m.fit(V.cpu(), beta=1, tol=1e-3, max_iter=50)
    for p, (npb, Wp, Hp) in enumerate(_single_fits(1, V, W0, H0, beta=1, tol=1e-3, max_iter=50)):
        assert int(n[p]) == npb and torch.equal(m.W.data[p], Wp.cpu()) and torch.equal(m.H.data[p], Hp.cpu())
    _check_batched(1, V[:1], W0[:1], H0[:1], beta=0.5, tol=1e-3, max_iter=70)       # P = 1
    _check_batched(3, *_problem(1, 1, 3, (3, 4, 10), 3, (1, 2, 4), 6, dev), beta=2, tol=1e-3, max_iter=30)


def test_single_fit_around_batched_fit_on_cached_workspaces():
    dev = _dev()
    C, X, K = FIT_SHAPES[1]
    V, W0, H0 = _problem(3, 2, C, X, 4, K, 9, dev)
    before = _single_fits(1, V, W0, H0, problems=[1], beta=1, tol=1e-3, max_iter=40)
    _check_batched(1, V, W0, H0, beta=1, tol=1e-3, max_iter=40)
    assert any(k[0] == "nmfd_batched" for k in E._WORKSPACES) and any(k[0] == "nmfd" for k in E._WORKSPACES)
    after = _single_fits(1, V, W0, H0, problems=[1], beta=1, tol=1e-3, max_iter=40)
    assert before[0][0] == after[0][0] and torch.equal(before[0][1], after[0][1]) and torch.equal(before[0][2], after[0][2])
    key = next(k for k in E._WORKSPACES if k[0] == "nmfd_batched")
    assert E._workspace_bytes(key) >= 3 * 4 * V[0].numel()


def _terms_equal_single(eng, V, W, H, problems, betas):
    for beta in betas:
        for p in problems:
            single = E.CudaNmfdEngine(V[p], W[p].clone(), H[p].clone(), "f32")
            try:
                for which in (0, 1):
                    sn, sd = single.raw_terms(which, beta)
                    bn, bd = eng.raw_terms(which, beta)
                    assert torch.equal(sn, bn[p]) and torch.equal(sd.reshape(bd[p].shape), bd[p]), (beta, p, which)
                assert float(single.loss(beta)) == float(eng.losses(beta)[p]), (beta, p)
            finally:
                single.close()


def test_lines_and_wgrad_splits_past_grid_z():
    """P x B = 70400 lines (two grid-z slices of the sliding kernels) and P x 64 wgrad splits = 70400 (two wgrad slices)."""
    dev = _dev()
    P, B = 1100, 64
    V, W, H = _problem(P, B, 2, (8,), 2, (3,), 1, dev)
    assert _capi.nmfd_plan(B, 2, (8,), 2, (3,))["wgrad_nsplit"] * P > 65535 and P * B > 65535
    eng = E.CudaBatchedNmfdEngine(V, W, H)
    try:
        eng.set_active(torch.arange(P) != 1050)
        _terms_equal_single(eng, V, W, H, [0, 1023, 1099], [1, 0.5])
        n = int(eng._lib.nmfb200_raw_terms_numel(eng._ctx, 0, 2.0))
        buf = torch.full((n,), SENTINEL, dtype=torch.float32, device=dev)
        eng._raw_terms_into(0, 2.0, buf)
        assert bool((buf[:W.numel()].view(W.shape)[1050] == SENTINEL).all())
    finally:
        eng.close()
    _check_batched(1, V[:1030], W[:1030].clone(), H[:1030].clone(), problems=[0, 1029], beta=1, tol=1e-3, max_iter=30)


def test_bf16_target_past_2_31_elements():
    dev = _dev()
    P, B, C, L, R, T = 4, 1, 1024, 600_000, 4, 4
    assert P * B * C * L > 2 ** 31
    g = torch.Generator(device=dev).manual_seed(0)
    V = (torch.rand(P, B, C, L, generator=g, device=dev) + 0.05).bfloat16()
    W = torch.rand(P, C, R, T, generator=g, device=dev) / 4 + 0.01
    H = torch.rand(P, B, R, L - T + 1, generator=g, device=dev) / 4 + 0.01
    eng = E.CudaBatchedNmfdEngine(V, W, H)
    try:
        _terms_equal_single(eng, V, W, H, [3], [1])
        vmin, vmax = eng.minmax()
        assert vmin == float(V.min()) and vmax == float(V.max())
    finally:
        eng.close()
        E.release_workspaces()


def test_refusals_on_device():
    dev = _dev()
    lib = _capi.load()
    V, W, H = _problem(2, 1, 3, (10,), 2, (3,), 0, dev)
    eng = E.CudaBatchedNmfdEngine(V, W, H)
    try:
        ctx = eng._ctx
        M = torch.ones(V.shape, dtype=torch.uint8, device=dev)
        assert lib.nmfb200_set_mask(ctx, E._ptr(M), None) != 0
        assert lib.nmfb200_set_weight(ctx, E._ptr(M.float()), None) != 0
        assert lib.nmfb200_w_apply(ctx, E._ptr(W), E._ptr(W), 1.0, 1.0, 0.0, 0.0, None) != 0
        assert lib.nmfb200_nmfd_set_target(ctx, E._ptr(V), 0, None) != 0
        assert lib.nmfb200_nmf_contract_only(ctx, E._ptr(W), E._ptr(H), 0, 1.0, None) != 0
        assert lib.nmfb200_nmf_iterate(ctx, E._ptr(W), E._ptr(H), 1.0, 1.0, 0.0, 0.0, 1, None) != 0
        assert lib.nmfb200_nmf_batched_set_active(ctx, None, None) != 0
        assert lib.nmfb200_nmfd_batched_set_target(ctx, E._ptr(V), 5, 0, None) != 0              # stride too small
        assert lib.nmfb200_precision_for_beta(ctx, 1.0) == _capi.PREC_F32
    finally:
        eng.close()
    import ctypes
    out = ctypes.c_void_p()
    vd, kd = (ctypes.c_int64 * 1)(10), (ctypes.c_int64 * 1)(3)
    assert lib.nmfb200_nmfnd_batched_create(ctypes.byref(out), 0, 70000, 40000, 3, 1, vd, 2, kd) != 0
    assert b"2^31" in lib.nmfb200_last_error()
    assert lib.nmfb200_nmfnd_batched_create(ctypes.byref(out), 0, 0, 1, 3, 1, vd, 2, kd) != 0
