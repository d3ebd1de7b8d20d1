"""Batched NMF on the GPU: every problem's raw terms and loss against float64, then whole fits bit for bit against single
`NMF.fit(precision="f32")` fits, at the batch and size limits, and next to cached single-problem workspaces."""
import math

import pytest
import torch

from torchnmf_b200 import NMF, BatchedNMF, _capi
from torchnmf_b200 import engine as E

pytestmark = pytest.mark.gpu

EPS = float(torch.finfo(torch.float32).eps)
SENTINEL = -12345.0


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda", 0)


def _phi64(V, S, beta):
    """Pn, Pp of nmf.py:61-74 in float64 (S: the reconstruction)."""
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


@pytest.mark.parametrize("R", [1, 16, 17, 64, 200, 256])
@pytest.mark.parametrize("beta", [0, 0.5, 1, 2, 3])
def test_raw_terms_and_loss_per_problem(beta, R):
    dev = _dev()
    g = torch.Generator(device="cpu").manual_seed(R * 10 + int(beta * 2))
    B, N, C = 4, 70, 97
    V = (torch.rand(B, N, C, generator=g) + 0.05).to(dev)
    W = (torch.rand(B, C, R, generator=g) / math.sqrt(R) + 0.01).to(dev)
    H = (torch.rand(B, N, R, generator=g) / math.sqrt(R) + 0.01).to(dev)
    active = torch.tensor([1, 0, 1, 1], dtype=torch.bool)
    eng = E.CudaBatchedNmfEngine(V, W, H)
    try:
        eng.set_active(active)
        for which in (0, 1):
            n = int(eng._lib.nmfb200_raw_terms_numel(eng._ctx, which, float(beta)))
            buf = torch.full((n,), SENTINEL, dtype=torch.float32, device=dev)
            eng._raw_terms_into(which, beta, buf)
            f = W if which == 0 else H
            num = buf[:f.numel()].view(f.shape)
            den = buf[f.numel():].view(B, R) if beta == 1 else buf[f.numel():].view(f.shape)
            for b in range(B):
                if not active[b]:
                    assert bool((num[b] == SENTINEL).all()) and bool((den[b] == SENTINEL).all())
                    continue
                V64, W64, H64 = V[b].double(), W[b].double(), H[b].double()
                Pn, Pp = _phi64(V64, H64 @ W64.T, beta)
                G = H64 if which == 0 else W64
                want_n = Pn.T @ G if which == 0 else Pn @ G
                scale = float(want_n.abs().max())
                assert torch.allclose(num[b].double(), want_n, rtol=2e-5, atol=1e-6 * scale), (b, which)
                if beta == 1:
                    want_d = (W64 if which == 1 else H64).sum(0)
                else:
                    want_d = Pp.T @ G if which == 0 else Pp @ G
                assert torch.allclose(den[b].double(), want_d, rtol=2e-5, atol=1e-6 * float(want_d.abs().max()))
        eng._loss.fill_(SENTINEL)
        d = eng.losses(beta)
        for b in range(B):
            if not active[b]:
                assert d[b] == SENTINEL
                continue
            want = _beta_div64(H[b].double() @ W[b].double().T, V[b].double(), beta)
            assert math.isclose(float(d[b]), want, rel_tol=1e-4, abs_tol=1e-6 * N * C), (b, float(d[b]), want)
        # bit for bit what a single-problem fp32 context computes
        for b in (0, 3):
            single = E.CudaNmfEngine(V[b], W[b].clone(), H[b].clone(), "f32")
            try:
                for which in (0, 1):
                    sn, sd = single.raw_terms(which, beta)
                    bn, bd = eng.raw_terms(which, beta)
                    assert torch.equal(sn, bn[b]) and torch.equal(sd, bd[b]), (b, which)
                assert float(single.loss(beta)) == float(eng.losses(beta)[b])
            finally:
                single.close()
    finally:
        eng.close()


def _single_fits(V, W0, H0, problems=None, trainable_W=True, trainable_H=True, **kw):
    out = []
    for b in (range(W0.shape[0]) if problems is None else problems):
        Vb = V if V.dim() == 2 else V[b]
        m = NMF(W=W0[b], H=H0[b], trainable_W=trainable_W, trainable_H=trainable_H).to(W0.device)
        n = m.fit(Vb, precision="f32", **kw)
        out.append((n, m.W.data, m.H.data))
    return out


def _check_batched(V, W0, H0, problems=None, trainable_W=True, trainable_H=True, **kw):
    m = BatchedNMF(W=W0, H=H0, trainable_W=trainable_W, trainable_H=trainable_H).to(W0.device)
    n = m.fit(V, **kw)
    assert n.dtype == torch.int64 and m.last_fit_precision == "f32"
    singles = _single_fits(V, W0, H0, problems, trainable_W, trainable_H, **kw)
    for b, (nb, Wb, Hb) in zip(range(W0.shape[0]) if problems is None else problems, singles):
        assert int(n[b]) == nb, (b, int(n[b]), nb)
        assert torch.equal(m.W.data[b], Wb), b
        assert torch.equal(m.H.data[b], Hb), b
    return n


def _stop_inputs(dev, dtype=torch.float32, B=4, N=100, C=90, R=8, seed=3):
    """Problems that stop at different iterations at beta 2, tol 1e-2 (rank-4 targets with growing noise)."""
    g = torch.Generator().manual_seed(seed)
    Ht, Wt = torch.rand(B, N, 4, generator=g), torch.rand(B, C, 4, generator=g)
    lev = torch.tensor([0.0, 0.05, 0.4, 3.0])[:B].view(B, 1, 1)
    V = (Ht @ Wt.transpose(1, 2) + lev * torch.rand(B, N, C, generator=g) + 0.01).to(dtype)
    W0, H0 = torch.rand(B, C, R, generator=g) + 0.05, torch.rand(B, N, R, generator=g) + 0.05
    return V.to(dev), W0.to(dev), H0.to(dev)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_fit_matches_single_fits_bit_for_bit(dtype):
    dev = _dev()
    V, W0, H0 = _stop_inputs(dev, dtype)
    n = _check_batched(V, W0, H0, beta=2, tol=1e-2, max_iter=60)
    assert len(set(n.tolist())) >= 2, n
    # beta 1 and 0.5 too, at other stop counts
    _check_batched(V, W0, H0, beta=1, tol=1e-2, max_iter=60)
    _check_batched(V, W0, H0, beta=0.5, tol=1e-2, max_iter=50)


def test_fit_shared_target_strided_and_penalties():
    dev = _dev()
    V, W0, H0 = _stop_inputs(dev)
    big = torch.zeros(100, 128, device=dev)
    big[:, :90] = V[2]
    shared = big[:, :90]                                  # row-strided, read in place
    _check_batched(shared, W0, H0, beta=1.5, tol=1e-3, max_iter=40, alpha=0.1, l1_ratio=0.4)
    _check_batched(shared.expand(4, 100, 90), W0, H0, beta=3, tol=1e-3, max_iter=30)
    _check_batched(V, W0, H0, beta=0, tol=-math.inf, max_iter=25, alpha=0.05, l1_ratio=1.0)


@pytest.mark.parametrize("frozen", ["W", "H"])
def test_fit_frozen_factor(frozen):
    dev = _dev()
    V, W0, H0 = _stop_inputs(dev)
    kw = dict(trainable_W=frozen != "W", trainable_H=frozen != "H")
    _check_batched(V, W0, H0, beta=2, tol=1e-2, max_iter=60, **kw)


def test_host_module_and_float64_target():
    dev = _dev()
    V, W0, H0 = _stop_inputs(dev)
    m = BatchedNMF(W=W0.cpu(), H=H0.cpu())
    n = m.fit(V.double().cpu(), beta=1, tol=1e-2, max_iter=40)
    assert m.W.device.type == "cpu"
    for b, (nb, Wb, Hb) in enumerate(_single_fits(V, W0, H0, beta=1, tol=1e-2, max_iter=40)):
        assert int(n[b]) == nb and torch.equal(m.W.data[b], Wb.cpu()) and torch.equal(m.H.data[b], Hb.cpu())


def test_batch_beyond_grid_y_limit():
    dev = _dev()
    B, N, C, R = 70000, 3, 5, 2
    g = torch.Generator().manual_seed(7)
    V = (torch.rand(B, N, C, generator=g) * torch.rand(B, 1, 1, generator=g) * 4 + 0.01).to(dev)
    W0 = (torch.rand(B, C, R, generator=g) + 0.05).to(dev)
    H0 = (torch.rand(B, N, R, generator=g) + 0.05).to(dev)
    picks = [0, 1, 65534, 65535, 65536, 69999] + torch.randint(0, B, (4,), generator=g).tolist()
    _check_batched(V, W0, H0, problems=picks, beta=1, tol=1e-3, max_iter=40)


def test_target_beyond_2_31_elements():
    dev = _dev()
    B, N, C, R = 1100, 1024, 2048, 4
    if torch.cuda.get_device_properties(dev).total_memory < 24 << 30:
        pytest.skip("needs a large device")
    g = torch.Generator(device=dev).manual_seed(5)
    V = torch.rand(B, N, C, generator=g, device=dev, dtype=torch.bfloat16)          # 2.3e9 elements, 4.6 GB
    W0 = torch.rand(B, C, R, generator=g, device=dev) + 0.05
    H0 = torch.rand(B, N, R, generator=g, device=dev) + 0.05
    try:
        _check_batched(V, W0, H0, problems=[0, 1023, 1024, 1099], beta=2, tol=-math.inf, max_iter=10)
    finally:
        del V
        E.release_workspaces()
        torch.cuda.empty_cache()


def test_b1_equals_nmf_and_caches_keep_their_bits():
    dev = _dev()
    V, W0, H0 = _stop_inputs(dev, B=1)
    single = _single_fits(V, W0, H0, beta=1, tol=1e-3, max_iter=50)[0]
    _check_batched(V, W0, H0, beta=1, tol=1e-3, max_iter=50)
    again = _single_fits(V, W0, H0, beta=1, tol=1e-3, max_iter=50)[0]      # after a batched fit on the same cache
    assert again[0] == single[0] and torch.equal(again[1], single[1]) and torch.equal(again[2], single[2])
    V4, W4, H4 = _stop_inputs(dev)
    a = _check_batched(V4, W4, H4, beta=2, tol=1e-2, max_iter=60)
    b = _check_batched(V4, W4, H4, beta=2, tol=1e-2, max_iter=60)         # the cached batched context: flags reset
    assert torch.equal(a, b)


def test_abi_refusals():
    dev = _dev()
    lib = _capi.load()
    import ctypes
    ctx = ctypes.c_void_p()
    assert lib.nmfb200_nmf_batched_create(ctypes.byref(ctx), 0, 2, 8, 8, 257) == 1
    assert lib.nmfb200_nmf_batched_create(ctypes.byref(ctx), 0, 0, 8, 8, 4) == 1
    V = torch.rand(2, 8, 8, device=dev)
    W, H = torch.rand(2, 8, 4, device=dev), torch.rand(2, 8, 4, device=dev)
    eng = E.CudaBatchedNmfEngine(V, W, H)
    single = E.CudaNmfEngine(V[0], W[0].clone(), H[0].clone(), "f32")
    try:
        p = E._ptr
        st = E._stream(dev)
        assert lib.nmfb200_set_mask(eng._ctx, p(V), st) == 1
        assert lib.nmfb200_set_weight(eng._ctx, p(V), st) == 1
        assert lib.nmfb200_w_apply(eng._ctx, p(W), p(V), 1.0, 1.0, 0.0, 0.0, st) == 1
        assert lib.nmfb200_nmf_set_target(eng._ctx, p(V), 8, 0, st) == 1
        assert lib.nmfb200_nmf_contract_only(eng._ctx, p(W), p(H), 0, 1.0, st) == 1
        assert lib.nmfb200_nmf_peer_alloc(eng._ctx, p(V)) == 1
        assert lib.nmfb200_nmf_batched_set_target(eng._ctx, p(V), 8, 7 * 8, 0, st) == 1        # stride below N ldv
        assert lib.nmfb200_nmf_batched_set_target(single._ctx, p(V), 8, 0, 0, st) == 1
        assert lib.nmfb200_nmf_batched_set_active(single._ctx, None, st) == 1
        assert lib.nmfb200_precision_for_beta(eng._ctx, 1.0) == _capi.PREC_F32
        assert lib.nmfb200_raw_terms_numel(eng._ctx, 0, 1.0) == 2 * 8 * 4 + 2 * 4
        assert lib.nmfb200_raw_terms_numel(eng._ctx, 1, 2.0) == 2 * (2 * 8 * 4)
    finally:
        single.close()
        eng.close()
