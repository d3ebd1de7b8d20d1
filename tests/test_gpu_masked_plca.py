"""Masked PLCA / SIPLCA / SIPLCA2 / SIPLCA3 fits on the H100: `fit(V, ..., mask=M)` against the reference's fixtures
(tests/golden/reference_masked_plca.npz), and the kernel terms of `nmfb200_plca_masked_terms` against float64 at every plan
branch of the fp32 contraction and the sliding kernels.
"""
import math

import pytest
import torch

from test_masked_plca import CLS, NAMES, case
from torchnmf_b200 import PLCA, SIPLCA, SIPLCA2, SIPLCA3
from torchnmf_b200 import engine as _engine
from torchnmf_b200.constants import eps as EPS

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
U = 2.0 ** -24


def _module(c, device=DEV):
    kw = {k: bool(int(c[k])) for k in ("trainable_W", "trainable_H", "trainable_Z")}
    m = CLS[int(c["cls"])](W=c["W0"], H=c["H0"], Z=c["Z0"], **kw)
    return m.to(device)


def _alphas(c):
    a = tuple(float(c[k]) for k in ("W_alpha", "H_alpha", "Z_alpha"))
    return tuple(torch.tensor(x) for x in a) if int(c["tensor_alpha"]) else a


def _close(got, want, rtol):
    return torch.allclose(got, want, rtol=rtol, atol=1e-5 * float(want.abs().max()))


def _worst(got, want):
    return float(((got - want).abs() / (want.abs() + 1e-5 * want.abs().max())).max())


# ---- whole fits against the reference's fixtures ------------------------------------------------------------------------------
@pytest.mark.parametrize("name", NAMES)
def test_fit_matches_reference(name):
    c = case(name)
    m = _module(c)
    n_iter, norm = m.fit(c["V"].to(DEV), float(c["tol"]), int(c["iters"]), False, *_alphas(c), mask=c["M"].to(DEV))
    assert n_iter == int(c["n_iter"])
    assert norm.dim() == 0 and abs(float(norm) - float(c["norm"])) <= 1e-3 * float(c["norm"])
    assert m.last_fit_precision == "f32"
    for nm in ("W", "H", "Z"):
        got, want = getattr(m, nm).detach().double().cpu(), c[nm]
        assert _close(got, want, 1e-3), (name, nm, _worst(got, want))


def test_imputation_uses_the_returned_norm():
    c = case("plca_gap")
    m = _module(c)
    M = c["M"].to(DEV)
    _, norm = m.fit(c["V"].to(DEV), float("-inf"), 30, mask=M)
    V = c["V"].to(DEV)
    with torch.no_grad():
        X = m(norm=norm)
    assert abs(float(X[M].sum()) - float(V[M].sum())) <= 1e-4 * float(V[M].sum())
    assert float(X[~M].min()) > 0                                      # the gap is filled by the model


# ---- the kernel terms against float64 ----------------------------------------------------------------------------------------
def _problem(vshape, wshape, hshape, missing, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    V = torch.rand(vshape, generator=g, device=DEV) * 3
    M = torch.rand(vshape, generator=g, device=DEV) >= missing
    W = torch.rand(wshape, generator=g, device=DEV) + 0.05
    Hz = torch.rand(hshape, generator=g, device=DEV) + 0.05
    W /= W.sum()                                           # keeps q a distribution's size, as in a fit
    Hz /= Hz.sum()
    Vn = torch.where(M, V, torch.zeros((), device=DEV))
    Vn = (Vn / Vn.sum()).contiguous()
    return Vn, M.contiguous(), W.contiguous(), Hz.contiguous()


def _conv(Hz, W):
    nd = W.dim() - 2
    conv = (None, torch.nn.functional.conv1d, torch.nn.functional.conv2d, torch.nn.functional.conv3d)[nd]
    return conv(Hz, W.flip(tuple(range(2, 2 + nd))), padding=tuple(k - 1 for k in W.shape[2:]))


def _terms64(Vn, M, W, Hz):
    """(A_W, B_W, A_H, B_H, q_O, and the same contractions of |P| for the bounds) in float64 from the fp32 inputs."""
    W64 = W.double().requires_grad_(True)
    H64 = Hz.double().requires_grad_(True)
    q = (H64 @ W64.t()) if W.dim() == 2 else _conv(H64, W64)
    q0 = q.detach()
    Mf = M.double()
    PA = Mf * Vn.double() / (q0 + EPS)
    PB = (1 - Mf) * q0 / (q0 + EPS)
    out = []
    for P in (PA, PB):
        out.append(torch.autograd.grad(q, (W64, H64), P, retain_graph=True))
    qo = float((q0 * Mf).sum())
    return out[0][0], out[1][0], out[0][1], out[1][1], qo


def _check_terms(eng, Vn, M, W, Hz, K_w, K_h):
    R = W.shape[1]
    aw64, bw64, ah64, bh64, qo64 = _terms64(Vn, M, W, Hz)
    qobs = torch.zeros(1, dtype=torch.float64, device=DEV)
    aw, bw = eng.plca_masked_terms(0, qobs)
    ah, bh = eng.plca_masked_terms(1)
    torch.cuda.synchronize()
    assert abs(float(qobs) - qo64) <= 1e-6 * qo64, (float(qobs), qo64)
    # every term is a sum of non-negative products: K fp32 accumulations of ratios whose S carries R roundings
    for got, want, K in ((aw, aw64, K_w), (bw, bw64, K_w), (ah, ah64, K_h), (bh, bh64, K_h)):
        bound = 1.01 * (K + R + 8) * U * want + 1e-30
        err = (got.double() - want).abs()
        assert bool((err <= bound).all()), float((err / bound).max())
        assert torch.isfinite(got).all()


NMF_CASES = [                 # (N, C, R): rows and columns at residues {0, 1, 63} mod 64, every register block, rank blocks
    (64, 65, 1), (65, 127, 16), (127, 128, 17), (128, 191, 256), (129, 64, 257), (63, 129, 300),
    (65, 2049, 16),           # several chunks for both updates (W: 2 chunks, H: 32)
    (2049, 65, 17),
    (1, 64, 1), (191, 1, 300),
]


@pytest.mark.parametrize("N,C,R", NMF_CASES)
def test_nmf_masked_terms(N, C, R):
    Vn, M, W, Hz = _problem((N, C), (C, R), (N, R), 0.3, N * 7 + C + R)
    eng = _engine.CudaNmfEngine(Vn, W, Hz, "f32")
    try:
        eng.set_mask(M)
        _check_terms(eng, Vn, M, W, Hz, N, C)
    finally:
        eng.close()


ND_CASES = [                  # (V shape, kernel, R): wgrad / dgrad splits from one to many, row tiles 4 ... 64
    ((2, 21, 61), (5,), 4),
    ((1, 3, 700), (16,), 7),
    ((8, 70, 129), (3,), 33),
    ((1, 257, 300), (32,), 16),
    ((3, 2, 130), (1,), 256),
    ((2, 5, 12, 20), (2, 3), 3),
    ((1, 9, 17, 66), (4, 5), 20),
    ((1, 3, 6, 7, 16), (2, 2, 3), 3),
    ((2, 2, 5, 9, 70), (3, 2, 4), 5),
]


@pytest.mark.parametrize("vs,ks,R", ND_CASES)
def test_nmfd_masked_terms(vs, ks, R):
    B, C, *X = vs
    hs = (B, R, *(x - k + 1 for x, k in zip(X, ks)))
    Vn, M, W, Hz = _problem(vs, (C, R, *ks), hs, 0.3, sum(vs) + R)
    eng = _engine.CudaNmfdEngine(Vn, W, Hz, "f32")
    try:
        eng.set_mask(M)
        kvol = math.prod(ks)
        _check_terms(eng, Vn, M, W, Hz, Vn.numel() // C, C * kvol)
    finally:
        eng.close()


def test_masked_terms_refusals():
    Vn, M, W, Hz = _problem((65, 70), (70, 4), (65, 4), 0.3, 1)
    from torchnmf_b200 import _capi
    eng = _engine.CudaNmfEngine(Vn, W, Hz, "f32")
    try:
        with pytest.raises(_capi.NmfB200Error, match="error 3"):      # no mask yet: NMFB200_ERR_STATE
            eng.plca_masked_terms(0)
        eng.set_weight(torch.ones_like(Vn))
        with pytest.raises(_capi.NmfB200Error, match="error 1"):      # a weight: NMFB200_ERR_INVALID
            eng.plca_masked_terms(0)
        eng.set_mask(M)
        eng.plca_masked_terms(1)
    finally:
        eng.close()
    lib = _capi.load()
    assert lib.nmfb200_plca_masked_terms(None, None, None, 0, None, None, None) != 0


# ---- fit properties -----------------------------------------------------------------------------------------------------------
def _fit(cls_args, V, M, iters=20, device=DEV, **kw):
    cls, args, ckw = cls_args
    torch.manual_seed(4)
    m = cls(*args, **ckw)
    m = m.to(device)
    out = m.fit(V, float("-inf"), iters, mask=M, **kw)
    return m, out


MODELS = [(PLCA, ((300, 200), 12), {}), (SIPLCA, ((2, 30, 150), 6, 9), {}), (SIPLCA2, ((1, 4, 20, 33), 5, (3, 4)), {}),
          (SIPLCA3, ((1, 3, 8, 9, 20), 4, (2, 3, 4)), {}), (PLCA, ((200, 150), 270), {})]


@pytest.mark.parametrize("model", MODELS, ids=lambda m: f"{m[0].__name__}_r{m[1][1]}")
def test_missing_cells_are_never_read(model):
    shape = model[1][0]
    g = torch.Generator(device=DEV).manual_seed(9)
    V = torch.rand(shape, generator=g, device=DEV)
    M = torch.rand(shape, generator=g, device=DEV) >= 0.3
    a, (na, norm_a) = _fit(model, V.masked_fill(~M, 0.0), M)
    b, (nb, norm_b) = _fit(model, V.masked_fill(~M, float("nan")), M)
    c, _ = _fit(model, V.masked_fill(~M, -7.0), M)
    assert na == nb and torch.equal(norm_a, norm_b)
    for x in (b, c):
        for nm in ("W", "H", "Z"):
            assert torch.equal(getattr(a, nm), getattr(x, nm)), nm


@pytest.mark.parametrize("model", MODELS[:4], ids=lambda m: m[0].__name__)
def test_all_true_mask_is_the_unmasked_fit(model):
    shape = model[1][0]
    V = torch.rand(shape, generator=torch.Generator(device=DEV).manual_seed(3), device=DEV)
    a, (na, norm_a) = _fit(model, V, torch.ones(shape, dtype=torch.bool, device=DEV), iters=30)
    cls, args, ckw = model
    torch.manual_seed(4)
    b = cls(*args, **ckw).to(DEV)
    nb, norm_b = b.fit(V, float("-inf"), 30, precision="f32")
    assert na == nb and abs(float(norm_a) - float(norm_b)) <= 1e-5 * float(norm_b)
    for nm in ("W", "H", "Z"):
        got, want = getattr(a, nm).detach(), getattr(b, nm).detach()
        assert _close(got, want, 1e-3), (nm, _worst(got, want))


@pytest.mark.parametrize("frozen", ["W", "H", "Z", "WZ"])
def test_frozen_factors_stay_bit_identical(frozen):
    c = case("plca_rand30")
    kw = {f"trainable_{k}": k not in frozen for k in "WHZ"}
    m = PLCA(W=c["W0"], H=c["H0"], Z=c["Z0"], **kw).to(DEV)
    before = {k: getattr(m, k).detach().clone() for k in "WHZ"}
    m.fit(c["V"].to(DEV), float("-inf"), 15, mask=c["M"].to(DEV))
    for k in "WHZ":
        same = torch.equal(getattr(m, k), before[k])
        assert same == (k in frozen), k


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_host_resident_modules_are_staged_and_written_back(dtype):
    c = case("siplca_rand30")
    dev_mod = _module(c)
    host = _module(c, "cpu").to(dtype)
    for nm in "WHZ":
        getattr(host, nm).data.copy_(getattr(dev_mod, nm).data.to(dtype))
    n1, norm1 = dev_mod.fit(c["V"].to(DEV), float("-inf"), 12, mask=c["M"].to(DEV))
    n2, norm2 = host.fit(c["V"].to(dtype), float("-inf"), 12, mask=c["M"])
    assert n1 == n2 and host.W.device.type == "cpu" and host.W.dtype == dtype
    assert abs(float(norm1) - float(norm2)) <= 1e-5 * float(norm1)
    for nm in "WHZ":
        got = getattr(host, nm).detach()
        want = getattr(dev_mod, nm).detach().cpu().to(dtype)
        if dtype == torch.float32:
            assert torch.equal(got, want), nm
        else:
            assert _close(got.double(), want.double(), 1e-6), nm
