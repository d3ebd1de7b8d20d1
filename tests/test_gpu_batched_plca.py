"""BatchedPLCA / BatchedSIPLCA / BatchedSIPLCA2 / BatchedSIPLCA3 on the H100 (nmfb200_plca_iterate, nmfb200_plca_loss): the EM
step term by term against a float64 model, whole fits bit for bit against P = 1 fits (under permutation, with problems
stopping early), against the single models' fp32 fits and the reference fixtures, shared and half / double targets, staged
modules, launch counts and large batches."""
import os

import numpy as np
import pytest
import torch

from batched_plca_oracle import em_step, kl_loss, raw_terms, _rank
from conftest import GOLDEN
from test_batched_plca import BATCHED, CASES, SINGLE, _worst, golden_case, golden_module
from torchnmf_b200 import BatchedPLCA, BatchedSIPLCA, BatchedSIPLCA2, BatchedSIPLCA3, _capi
from torchnmf_b200 import engine as _engine

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")

SHAPES = {   # model -> (single target shape, K) for rank R
    "plca": ((40, 24), ()),
    "nd1": ((2, 12, 40), (5,)),
    "nd2": ((1, 5, 9, 14), (2, 4)),
    "nd3": ((1, 4, 5, 6, 9), (2, 2, 3)),
}


def _factors(model, P, R, seed=0):
    g = torch.Generator().manual_seed(seed)
    vs, K = SHAPES[model]
    # multiples of 2^-8 below 2: every sum of a problem's target is exact in fp32, so its norm does not depend on the order
    # torch reduces it in (which follows the memory alignment of the problem's block)
    V = torch.randint(13, 512, (P, *vs), generator=g).float() / 256
    if model == "plca":
        N, C = vs
        W, H = torch.rand(P, C, R, generator=g) + 0.1, torch.rand(P, N, R, generator=g) + 0.1
    else:
        B, C, *X = vs
        W = torch.rand(P, C, R, *K, generator=g) + 0.1
        H = torch.rand(P, B, R, *(x - k + 1 for x, k in zip(X, K)), generator=g) + 0.1
    W = W / W.sum([d for d in range(W.dim()) if d not in (0, 2)], keepdim=True)
    H = H / H.sum([d for d in range(H.dim()) if d not in (0, 2)], keepdim=True)
    Z = torch.rand(P, R, generator=g) + 0.1
    return V, W, H, Z / Z.sum(1, keepdim=True)


def _engine_for(model, Vn, W, Hz):
    cls = _engine.CudaBatchedNmfEngine if model == "plca" else _engine.CudaBatchedNmfdEngine
    return cls(Vn, W, Hz)


def _em_once(model, R, flags, alpha, inactive=None, P=3, seed=0):
    """One plca_iterate step on the GPU and the float64 model's step from the same state: (got, want) dicts."""
    V, W, H, Z = _factors(model, P, R, seed)
    Vn = V / V.sum([d for d in range(1, V.dim())], keepdim=True)
    norm = V.sum([d for d in range(1, V.dim())]).float()
    g = torch.Generator().manual_seed(seed + 1)
    alphas = []
    for t in (W, H, Z):
        if alpha == "none":
            alphas.append(None)
        elif alpha == "scalar":
            alphas.append(torch.full(t.shape, 1.3))
        else:
            alphas.append(0.8 + 0.6 * torch.rand(t.shape, generator=g))
    Wd, Hd, Zd = (t.to(DEV).contiguous() for t in (W, H, Z))
    Hz = (Hd * _rank(Zd, Hd)).contiguous()
    eng = _engine_for(model, Vn.to(DEV).contiguous(), Wd, Hz)
    try:
        if inactive is not None:
            act = torch.ones(P, dtype=torch.bool); act[inactive] = False
            eng.set_active(act)
        before = {k: t.clone() for k, t in (("W", Wd), ("H", Hd), ("Z", Zd), ("Hz", Hz))}
        eng.plca_iterate(1, Hd, Zd, bool(flags & 1), bool(flags & 2), bool(flags & 4),
                         *[a.to(DEV).contiguous() if a is not None else None for a in alphas])
        loss = eng.plca_losses(norm.to(DEV))
        torch.cuda.synchronize()
        got = {"W": Wd.cpu(), "H": Hd.cpu(), "Z": Zd.cpu(), "Hz": Hz.cpu(), "loss": loss}
    finally:
        eng.close()
    W64, H64, Z64 = W.double(), H.double(), Z.double()
    dW, dHz = raw_terms(Vn.double(), W64, (H64 * _rank(Z64, H64)))
    Wn, Hn, Zn = em_step(W64, H64, Z64, dW, dHz, bool(flags & 1), bool(flags & 2), bool(flags & 4),
                         *[a.double() if a is not None else None for a in alphas])
    want = {"W": Wn, "H": Hn, "Z": Zn, "Hz": Hn * _rank(Zn, Hn),
            "loss": kl_loss(Vn.double(), Wn, Hn * _rank(Zn, Hn), norm.double())}
    if inactive is not None:
        for k in ("W", "H", "Z", "Hz"):
            want[k][inactive] = before[k][inactive].cpu().double()
    return got, want


def _check(got, want, rtol=2e-4):
    for k in ("W", "H", "Z", "Hz"):
        g, w = got[k].double(), want[k]
        assert torch.allclose(g, w, rtol=rtol, atol=1e-6 * float(w.abs().max())), (k, _worst(g, w))


@pytest.mark.parametrize("flags", range(8))
@pytest.mark.parametrize("alpha", ["none", "scalar", "tensor"])
def test_em_step_flags_and_alphas(flags, alpha):
    got, want = _em_once("plca", 7, flags, alpha, inactive=1)
    _check(got, want)


@pytest.mark.parametrize("model", list(SHAPES))
@pytest.mark.parametrize("R", [1, 7, 16, 256])
def test_em_step_models_and_ranks(model, R):
    got, want = _em_once(model, R, 7, "tensor" if R == 7 else "none", inactive=0)
    _check(got, want)
    # the loss of the de-normalised reconstruction, every active problem
    act = torch.tensor([False, True, True])
    assert torch.allclose(got["loss"][act], want["loss"][act], rtol=1e-4, atol=1e-6)


def _module(cls, W, H, Z, device=DEV):
    """A module holding exactly these (already normalised) factors: the constructor's normalisation is a torch reduction
    whose bits depend on P, so it is undone by copying the factors back."""
    m = cls(W=W, H=H, Z=Z)
    for k, t in (("W", W), ("H", H), ("Z", Z)):
        getattr(m, k).data.copy_(t)
    return m.to(device)


def _fit(cls, V, W, H, Z, **kw):
    m = _module(cls, W, H, Z)
    n, norm = m.fit(V, **kw)
    return m, n, norm


@pytest.mark.parametrize("model", ["plca", "nd1", "nd2", "nd3"])
def test_batch_independence_bit_for_bit(model):
    cls = {"plca": BatchedPLCA, "nd1": BatchedSIPLCA, "nd2": BatchedSIPLCA2, "nd3": BatchedSIPLCA3}[model]
    V, W, H, Z = _factors(model, 5, 4, seed=3)
    Vd = V.to(DEV)
    for tol in torch.logspace(-4, -0.5, 22).tolist():   # the first tolerance at which the problems stop at different counts
        m, n, norm = _fit(cls, Vd, W, H, Z, tol=tol, max_iter=60)
        if len(set(n.tolist())) > 1:
            break
    assert len(set(n.tolist())) > 1 and int(n.min()) < 59
    perm = [3, 0, 4, 2, 1]
    mp, n_p, norm_p = _fit(cls, Vd[perm].contiguous(), W[perm], H[perm], Z[perm], tol=tol, max_iter=60)
    for p in range(5):
        m1, n1, norm1 = _fit(cls, Vd[p:p + 1].contiguous(), W[p:p + 1], H[p:p + 1], Z[p:p + 1], tol=tol, max_iter=60)
        assert int(n1[0]) == int(n[p]) and torch.equal(norm1[0], norm[p])
        for k in ("W", "H", "Z"):
            assert torch.equal(getattr(m1, k).data[0], getattr(m, k).data[p]), (k, p)
    for i, p in enumerate(perm):
        assert int(n_p[i]) == int(n[p]) and torch.equal(norm_p[i], norm[p])
        for k in ("W", "H", "Z"):
            assert torch.equal(getattr(mp, k).data[i], getattr(m, k).data[p])


@pytest.mark.parametrize("name", CASES)
def test_against_single_fp32_fits(name):
    c = golden_case(name)
    m, V, kw = golden_module(c)
    m = m.to(DEV)
    n, norm = m.fit(V.to(DEV), **kw)
    worst = 0.0
    for p in range(m.W.shape[0]):
        s = SINGLE[type(m)](W=c["W0"][p], H=c["H0"][p], Z=c["Z0"][p], trainable_W=bool(c["trainable_W"]),
                            trainable_Z=bool(c["trainable_Z"])).to(DEV)
        skw = dict(kw)
        if isinstance(kw["W_alpha"], torch.Tensor):
            skw["W_alpha"] = kw["W_alpha"][p].reshape(())
        n1, norm1 = s.fit((V if c["shared"] else V[p]).to(DEV), precision="f32", **skw)
        assert int(n[p]) == n1 and float(norm[p]) == float(norm1)
        for k in ("W", "H", "Z"):
            got, want = getattr(m, k).data[p], getattr(s, k).data
            worst = max(worst, _worst(got, want))
    print(f"{name}: worst relative deviation from the single fp32 fits {worst:.2e}")
    assert worst < 5e-5                 # measured on an H100: at most 1.3e-5 over the fixture cases


@pytest.mark.parametrize("name", CASES)
def test_against_reference_fixtures(name):
    c = golden_case(name)
    m, V, kw = golden_module(c)
    m = m.to(DEV)
    n, norm = m.fit(V.to(DEV), **kw)
    assert n.tolist() == c["n_iter"].tolist()
    assert torch.allclose(norm.double().cpu(), c["norm"], rtol=1e-6)
    for k in ("W", "H", "Z"):
        got, want = getattr(m, k).data.cpu(), c[k]
        assert torch.allclose(got, want, rtol=1e-3, atol=1e-5 * float(want.abs().max())), (k, _worst(got, want))


def test_shared_target_dtypes_and_staging():
    V, W, H, Z = _factors("plca", 4, 5, seed=5)
    Vs = V[1].to(DEV)
    a, na, norma = _fit(BatchedPLCA, Vs, W, H, Z, tol=1e-4, max_iter=40)
    b, nb, normb = _fit(BatchedPLCA, Vs.expand(4, *Vs.shape).contiguous(), W, H, Z, tol=1e-4, max_iter=40)
    assert na.tolist() == nb.tolist() and torch.equal(norma, normb)
    for k in ("W", "H", "Z"):
        assert torch.equal(getattr(a, k).data, getattr(b, k).data)
    ref, nr, _ = _fit(BatchedPLCA, V.to(DEV), W, H, Z, tol=-1.0, max_iter=20)
    for dt in (torch.bfloat16, torch.float16, torch.float64):
        Vt = V.to(dt)
        m, n, norm = _fit(BatchedPLCA, Vt.to(DEV), W, H, Z, tol=-1.0, max_iter=20)
        assert norm.dtype == dt and n.tolist() == nr.tolist()
        for p in range(4):                   # the norm is taken in V's dtype, as the single fit takes it
            s = SINGLE[BatchedPLCA](W=W[p], H=H[p], Z=Z[p]).to(DEV)
            s.W.data.copy_(W[p]); s.H.data.copy_(H[p]); s.Z.data.copy_(Z[p])
            _, norm1 = s.fit(Vt[p].to(DEV), tol=-1.0, max_iter=20)
            assert torch.equal(norm[p], norm1)
            assert torch.allclose(m.W.data[p], s.W.data, rtol=1e-4, atol=1e-7), _worst(m.W.data[p], s.W.data)
    host = _module(BatchedPLCA, W, H, Z, device="cpu")
    nh, _ = host.fit(V.to(DEV), tol=-1.0, max_iter=20)
    assert host.W.device.type == "cpu" and nh.tolist() == nr.tolist()
    assert torch.equal(host.W.data, ref.W.data.cpu()) and torch.equal(host.Z.data, ref.Z.data.cpu())
    dbl = _module(BatchedPLCA, W, H, Z, device="cpu").double().to(DEV)
    dbl.fit(V.to(DEV), tol=-1.0, max_iter=20)
    assert dbl.W.dtype == torch.float64 and torch.equal(dbl.W.data.float(), ref.W.data)


def test_launch_count_independent_of_batch():
    counts = {}
    for P in (1, 64):
        V, W, H, Z = _factors("plca", P, 8, seed=7)
        Vn = (V / V.sum((1, 2), keepdim=True)).to(DEV)
        Wd, Hd, Zd = (t.to(DEV).contiguous() for t in (W, H, Z))
        Hz = (Hd * Zd.unsqueeze(1)).contiguous()
        eng = _engine.CudaBatchedNmfEngine(Vn, Wd, Hz)
        try:
            eng.plca_iterate(1, Hd, Zd, True, True, True)
            c0 = _capi.launch_count()
            eng.plca_iterate(10, Hd, Zd, True, True, True, torch.full_like(Wd, 1.2), None, None)
            c10 = _capi.launch_count() - c0
            c0 = _capi.launch_count()
            eng.raw_terms(0, 1.0); eng.raw_terms(1, 1.0)
            terms = _capi.launch_count() - c0
        finally:
            eng.close()
        counts[P] = (c10, terms)
    assert counts[1] == counts[64]
    c10, terms = counts[1]
    assert c10 % 10 == 0 and c10 // 10 <= terms + 3        # the raw terms without their column sums, plus the EM step


def test_large_batch_and_rank_256():
    P = 4096
    g = torch.Generator().manual_seed(11)
    V = (torch.rand(P, 24, 16, generator=g) + 0.05).to(DEV)
    m = BatchedPLCA((P, 24, 16), rank=6).to(DEV)
    W0, H0, Z0 = m.W.data.clone(), m.H.data.clone(), m.Z.data.clone()
    n, norm = m.fit(V, tol=1e-4, max_iter=30)
    assert bool(torch.isfinite(m.W.data).all()) and bool(torch.isfinite(m.H.data).all())
    for p in (0, 1234, P - 1):
        s = _module(BatchedPLCA, W0[p:p + 1], H0[p:p + 1], Z0[p:p + 1])
        n1, _ = s.fit(V[p:p + 1], tol=1e-4, max_iter=30)
        assert int(n1[0]) == int(n[p]) and torch.equal(s.W.data[0], m.W.data[p]) and torch.equal(s.Z.data[0], m.Z.data[p])
    V2, W2, H2, Z2 = _factors("plca", 2, 256, seed=12)
    m2, n2, _ = _fit(BatchedPLCA, V2.to(DEV), W2, H2, Z2, tol=-1.0, max_iter=10)
    assert n2.tolist() == [9, 9] and bool(torch.isfinite(m2.W.data).all())
    assert torch.allclose(m2.Z.data.sum(1), torch.ones(2, device=DEV), rtol=1e-5)
