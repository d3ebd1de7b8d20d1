"""BatchedPLCA / BatchedSIPLCA / BatchedSIPLCA2 / BatchedSIPLCA3 host logic on the CPU (no GPU): the per-problem stop rule
and its n_iter convention, freezing of stopped problems, norms, shared targets, alpha broadcasting, frozen factors, every
refusal and the module surface, through a float64 engine (tests/batched_plca_oracle.py, the `_engine_factory` hook); and
that engine against tests/golden/reference_batched_plca.npz (tools/make_golden_batched_plca.py: the unmodified reference's
PLCA / SIPLCA* `.fit`, problem by problem)."""
import os

import numpy as np
import pytest
import torch

from batched_plca_oracle import BatchedPlcaOracleEngine
from conftest import GOLDEN
from torchnmf_b200 import (PLCA, SIPLCA, SIPLCA2, SIPLCA3, BatchedPLCA, BatchedSIPLCA, BatchedSIPLCA2,
                           BatchedSIPLCA3)

Z_GOLD = np.load(os.path.join(GOLDEN, "reference_batched_plca.npz"), allow_pickle=False)
CASES = sorted({k.split("/")[0] for k in Z_GOLD.files})
BATCHED = {"plca": BatchedPLCA, "siplca": BatchedSIPLCA, "siplca2": BatchedSIPLCA2, "siplca3": BatchedSIPLCA3}
SINGLE = {BatchedPLCA: PLCA, BatchedSIPLCA: SIPLCA, BatchedSIPLCA2: SIPLCA2, BatchedSIPLCA3: SIPLCA3}


def golden_case(name):
    c = {k.split("/", 1)[1]: Z_GOLD[k] for k in Z_GOLD.files if k.startswith(name + "/")}
    model = str(c.pop("model"))
    out = {k: (torch.from_numpy(v.copy()) if v.dtype != np.float64 or v.ndim else float(v)) for k, v in c.items()}
    out["model"] = model
    return out


def golden_module(c):
    """The batched module of a fixture case and the fit arguments: (module, V, kwargs)."""
    m = BATCHED[c["model"]](W=c["W0"], H=c["H0"], Z=c["Z0"], trainable_W=bool(c["trainable_W"]),
                            trainable_Z=bool(c["trainable_Z"]))
    W_alpha = c["W_alpha"].reshape(-1, 1, *([1] * (c["W0"].dim() - 2))) if "W_alpha" in c and not isinstance(
        c["W_alpha"], float) else c["W_alpha"]
    V = c["V"][0] if c["shared"] else c["V"]
    return m, V, dict(tol=c["tol"], max_iter=int(c["max_iter"]), W_alpha=W_alpha, H_alpha=c["H_alpha"],
                      Z_alpha=c["Z_alpha"])


def oracle(m):
    engines = []

    def factory(V, W, Hz):
        engines.append(BatchedPlcaOracleEngine(V, W, Hz))
        return engines[-1]
    m._engine_factory = factory
    return engines


def _worst(got, want):
    return float(((got - want).abs() / (want.abs() + 1e-5 * want.abs().max())).max())


@pytest.mark.parametrize("name", CASES)
def test_oracle_engine_matches_reference(name):
    c = golden_case(name)
    m, V, kw = golden_module(c)
    oracle(m)
    n_iter, norm = m.fit(V, **kw)
    assert n_iter.dtype == torch.int64 and n_iter.tolist() == c["n_iter"].tolist()
    assert torch.allclose(norm.double(), c["norm"], rtol=1e-6)
    for k in ("W", "H", "Z"):
        got, want = getattr(m, k).data, c[k]
        assert torch.allclose(got, want, rtol=1e-3, atol=1e-5 * float(want.abs().max())), (k, _worst(got, want))


def test_fixture_problems_stop_at_different_counts():
    assert any(len(set(golden_case(n)["n_iter"].tolist())) > 1 for n in CASES if golden_case(n)["model"] == "plca")
    for model in BATCHED:
        assert any(golden_case(n)["model"] == model for n in CASES)


def _problems(P=3, N=12, C=9, R=3, seed=0):
    g = torch.Generator().manual_seed(seed)
    V = torch.rand(P, N, C, generator=g) + 0.05
    V[0] = V[0] * 0.0 + torch.rand(N, 1, generator=g) @ torch.rand(1, C, generator=g) + 0.01   # rank 1: stops early
    return V, torch.rand(P, C, R, generator=g) + 0.1, torch.rand(P, N, R, generator=g) + 0.1


def test_stop_rule_per_problem_and_stopped_problems_frozen():
    V, W0, H0 = _problems()
    m = BatchedPLCA(W=W0, H=H0)
    engines = oracle(m)
    n_iter, norm = m.fit(V, tol=1e-3, max_iter=200)
    eng = engines[0]
    # each problem's count is the loop index of the single fit: a multiple of 10 minus one, and the EM steps it received
    for p in range(3):
        assert n_iter[p] % 10 == 9 and eng.steps[p] == n_iter[p] + 1
    assert len(set(n_iter.tolist())) > 1
    for p in range(3):
        single = BatchedPLCA(W=W0[p:p + 1], H=H0[p:p + 1])
        oracle(single)
        n1, norm1 = single.fit(V[p:p + 1], tol=1e-3, max_iter=200)
        assert n1.tolist() == [int(n_iter[p])] and float(norm1[0]) == float(norm[p])
        for k in ("W", "H", "Z"):
            assert torch.equal(getattr(single, k).data[0], getattr(m, k).data[p])


def test_n_iter_convention():
    V, W0, H0 = _problems()
    for max_iter, want in ((0, -1), (7, 6), (25, 24)):
        m = BatchedPLCA(W=W0, H=H0)
        engines = oracle(m)
        n_iter, _ = m.fit(V, tol=float("-inf"), max_iter=max_iter)
        assert n_iter.tolist() == [want] * 3
        assert engines[0].steps == [max_iter] * 3


def test_norms_in_target_dtype():
    V, W0, H0 = _problems()
    for dt in (torch.float32, torch.float64, torch.bfloat16, torch.float16):
        m = BatchedPLCA(W=W0, H=H0)
        oracle(m)
        Vt = V.to(dt)
        _, norm = m.fit(Vt, max_iter=3)
        assert norm.dtype == dt and norm.shape == (3,)
        assert all(torch.equal(norm[p], Vt[p].sum()) for p in range(3))


def test_shared_target_equals_expanded():
    V, W0, H0 = _problems()
    a, b = BatchedPLCA(W=W0, H=H0), BatchedPLCA(W=W0, H=H0)
    oracle(a); oracle(b)
    na, norma = a.fit(V[1], tol=-1.0, max_iter=20)
    nb, normb = b.fit(V[1].expand(3, *V[1].shape).contiguous(), tol=-1.0, max_iter=20)
    assert na.tolist() == nb.tolist() and torch.equal(norma, normb)
    for k in ("W", "H", "Z"):
        assert torch.equal(getattr(a, k).data, getattr(b, k).data)


def test_alpha_broadcast_to_batched_shapes():
    V, W0, H0 = _problems()
    m = BatchedPLCA(W=W0, H=H0)
    engines = oracle(m)
    m.fit(V, max_iter=1, W_alpha=torch.full((9, 3), 1.5), H_alpha=1.2, Z_alpha=torch.tensor([[1.1], [1.2], [1.3]]))
    aW, aH, aZ = engines[0].alphas
    assert aW.shape == (3, 9, 3) and bool((aW == 1.5).all())
    assert aH.shape == (3, 12, 3) and bool((aH == 1.2).all()) and aH.dtype == torch.float32
    assert aZ.shape == (3, 3) and torch.equal(aZ[:, 0], torch.tensor([1.1, 1.2, 1.3]))
    m2 = BatchedPLCA(W=W0, H=H0)
    engines = oracle(m2)
    m2.fit(V, max_iter=1)
    assert engines[0].alphas == (None, None, None)
    m3 = BatchedPLCA(W=W0, H=H0)
    oracle(m3)
    with pytest.raises(ValueError):
        m3.fit(V, max_iter=1, W_alpha=torch.ones(4, 3))


@pytest.mark.parametrize("frozen", ["Z", "W", "WZ", "H"])
def test_frozen_factors_take_the_reference_branches(frozen):
    V, W0, H0 = _problems()
    Z0 = torch.rand(3, 3) + 0.1
    m = BatchedPLCA(W=W0, H=H0, Z=Z0, trainable_W="W" not in frozen, trainable_H="H" not in frozen,
                    trainable_Z="Z" not in frozen)
    oracle(m)
    before = {k: getattr(m, k).data.clone() for k in "WHZ"}
    m.fit(V, tol=float("-inf"), max_iter=5)
    for k in "WHZ":
        assert torch.equal(getattr(m, k).data, before[k]) == (k in frozen)
    # each problem follows plca_oracle.fit, the reference's branches in float32
    from oracle import plca_oracle
    for p in range(3):
        single = SINGLE[BatchedPLCA](W=W0[p], H=H0[p], Z=Z0[p])
        W, H, Z, _, _ = plca_oracle.fit(V[p], single.W.data, single.H.data, single.Z.data, float("-inf"), 5,
                                        trainable_W="W" not in frozen, trainable_H="H" not in frozen,
                                        trainable_Z="Z" not in frozen)
        for got, want in ((m.W.data[p], W), (m.H.data[p], H), (m.Z.data[p], Z)):
            assert torch.allclose(got, want, rtol=1e-4, atol=1e-7)


def test_refusals():
    V, W0, H0 = _problems()
    m = BatchedPLCA(W=W0, H=H0)
    oracle(m)
    for prec in ("f16", "f16_split", "auto", "bogus"):
        with pytest.raises(ValueError):
            m.fit(V, precision=prec)
    with pytest.raises(NotImplementedError):
        m.fit(V.to_sparse())
    with pytest.raises(ValueError):
        m.fit(V[:, :5])
    with pytest.raises(AssertionError, match="Target should be non-negative."):
        m.fit(-V)
    for kw in ("mask", "weight", "group"):
        with pytest.raises(TypeError):
            m.fit(V, **{kw: None})
    big = BatchedPLCA((2, 4, 3), rank=257)
    oracle(big)
    with pytest.raises(ValueError):
        big.fit(torch.rand(2, 4, 3))


def test_constructor_shapes_and_normalisation():
    m = BatchedPLCA((5, 12, 9), rank=3)
    assert m.W.shape == (5, 9, 3) and m.H.shape == (5, 12, 3) and m.Z.shape == (5, 3)
    assert torch.allclose(m.W.data.sum(1), torch.ones(5, 3)) and torch.allclose(m.H.data.sum(1), torch.ones(5, 3))
    assert torch.equal(m.Z.data, torch.full((5, 3), 1 / 3))
    s = BatchedSIPLCA((4, 2, 6, 20), rank=3, T=5)
    assert s.W.shape == (4, 6, 3, 5) and s.H.shape == (4, 2, 3, 16) and s.Z.shape == (4, 3)
    assert torch.allclose(s.W.data.sum((1, 3)), torch.ones(4, 3)) and torch.allclose(s.H.data.sum((1, 3)), torch.ones(4, 3))
    s2 = BatchedSIPLCA2((2, 1, 3, 7, 8), rank=2, kernel_size=(2, 3))
    assert s2.W.shape == (2, 3, 2, 2, 3) and s2.H.shape == (2, 1, 2, 6, 6)
    s3 = BatchedSIPLCA3((2, 1, 3, 5, 6, 7), rank=2, kernel_size=2)
    assert s3.W.shape == (2, 3, 2, 2, 2, 2) and s3.H.shape == (2, 1, 2, 4, 5, 6)
    assert s3.kernel_size == (2, 2, 2) and s3.out_channels == 3
    Z = torch.rand(5, 3)
    mz = BatchedPLCA((5, 12, 9), rank=3, Z=Z)
    assert torch.allclose(mz.Z.data, Z / Z.sum(1, keepdim=True))
    with pytest.raises(ValueError):
        BatchedPLCA(W=torch.rand(2, 9, 3), H=torch.rand(3, 12, 3))           # P disagrees
    with pytest.raises(ValueError):
        BatchedPLCA(W=torch.rand(2, 9, 3), H=torch.rand(2, 12, 4))           # R disagrees
    with pytest.raises(ValueError):
        BatchedPLCA(W=torch.rand(2, 9, 3), H=torch.rand(2, 12, 3), Z=torch.rand(3, 3))
    with pytest.raises(ValueError):
        BatchedPLCA(W=torch.rand(2, 9, 3), H=torch.rand(2, 12, 3), Z=torch.rand(2, 4))
    with pytest.raises(ValueError):
        BatchedPLCA(W=torch.rand(9, 3), H=torch.rand(12, 3))


@pytest.mark.parametrize("cls, shape, kw", [
    (BatchedPLCA, (3, 12, 9), {}), (BatchedSIPLCA, (3, 2, 6, 20), {"T": 4}),
    (BatchedSIPLCA2, (3, 2, 3, 7, 8), {"kernel_size": (2, 3)}), (BatchedSIPLCA3, (3, 1, 3, 5, 6, 7), {"kernel_size": 2})])
def test_reconstruct_matches_single_models(cls, shape, kw):
    torch.manual_seed(0)
    m = cls(shape, rank=3, **kw)
    m.Z.data.copy_(torch.rand(3, 3))
    norm = torch.tensor([1.0, 2.0, 3.0])
    out = m(norm=norm)
    assert out.shape == shape
    for p in range(3):
        want = SINGLE[cls].reconstruct(m.H.data[p], m.W.data[p], m.Z.data[p])
        assert torch.allclose(out[p], want * norm[p], rtol=1e-5, atol=1e-7)
