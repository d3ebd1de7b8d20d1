"""BatchedNMF's host logic on the CPU (no GPU): the per-problem stop rule, freezing of stopped problems, shared targets,
frozen factors and every refusal, through an engine that fits each problem with the CPU oracle (the `_engine_factory` hook),
and the fits against tests/golden/reference_batched.npz (tools/make_golden_batched.py: the unmodified reference's
`NMF.fit`, problem by problem)."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from batched_oracle import BatchedOracleEngine
from oracle_engine import OracleNmfEngine
from torchnmf_b200 import NMF, BatchedNMF


def _single_oracle(V, W0, H0, **kw):
    m = NMF(W=W0, H=H0, trainable_W=kw.pop("trainable_W", True), trainable_H=kw.pop("trainable_H", True))
    m._engine_factory = OracleNmfEngine
    n = m.fit(V, **kw)
    return n, m.W.data.clone(), m.H.data.clone()


def _batched(V, W0, H0, trainable_W=True, trainable_H=True, log=None, **kw):
    m = BatchedNMF(W=W0, H=H0, trainable_W=trainable_W, trainable_H=trainable_H)
    m._engine_factory = BatchedOracleEngine.factory(OracleNmfEngine, [] if log is None else log)
    n = m.fit(V, **kw)
    return n, m.W.data.clone(), m.H.data.clone(), m


def _inputs(B=3, N=20, C=14, R=4, seed=0):
    g = torch.Generator().manual_seed(seed)
    V = (torch.rand(B, N, C, generator=g) * torch.linspace(0.2, 2.0, B).view(B, 1, 1) + 0.01)
    return V, torch.rand(B, C, R, generator=g) + 0.1, torch.rand(B, N, R, generator=g) + 0.1


def load_batched():
    z = np.load(os.path.join(GOLDEN, "reference_batched.npz"), allow_pickle=False)
    cases = {}
    for key in z.files:
        name, field = key.split("/", 1)
        v = z[key]
        if field in ("V", "W0", "H0", "W", "H"):
            v = torch.from_numpy(v.copy())
        elif field == "n_iter":
            v = [int(x) for x in v]
        else:
            v = float(v)
            if field == "max_iter":
                v = int(v)
        cases.setdefault(name, {})[field] = v
    return cases


GOLD = load_batched()


@pytest.mark.parametrize("name", sorted(GOLD))
def test_batched_fit_matches_reference_problem_by_problem(name):
    c = GOLD[name]
    log = []
    n, W, H, m = _batched(c["V"], c["W0"], c["H0"], log=log, beta=c["beta"], tol=c["tol"], max_iter=c["max_iter"])
    assert n.dtype == torch.int64 and n.shape == (4,)
    assert n.tolist() == c["n_iter"]
    assert torch.allclose(W, c["W"], rtol=2e-5, atol=1e-7), (W - c["W"]).abs().max()
    assert torch.allclose(H, c["H"], rtol=2e-5, atol=1e-7), (H - c["H"]).abs().max()
    eng, = log
    assert eng.updates_w == c["n_iter"] and eng.updates_h == c["n_iter"]


def test_golden_problems_stop_at_different_counts():
    for c in GOLD.values():
        assert len(set(c["n_iter"])) >= 3 and max(c["n_iter"]) < c["max_iter"]
    assert sorted(c["beta"] for c in GOLD.values()) == [0.5, 1, 2]


@pytest.mark.parametrize("beta", [0.5, 1, 2])
def test_each_problem_is_its_own_fit_and_stopped_problems_stay_frozen(beta):
    V, W0, H0 = _inputs()
    log = []
    n, W, H, _ = _batched(V, W0, H0, log=log, beta=beta, tol=3e-3, max_iter=120, alpha=0.05, l1_ratio=0.3)
    counts = []
    for b in range(V.shape[0]):
        nb, Wb, Hb = _single_oracle(V[b], W0[b], H0[b], beta=beta, tol=3e-3, max_iter=120, alpha=0.05, l1_ratio=0.3)
        counts.append(nb)
        assert int(n[b]) == nb
        assert torch.equal(W[b], Wb) and torch.equal(H[b], Hb)
    assert len(set(counts)) > 1, counts
    eng, = log
    assert eng.updates_w == counts and eng.updates_h == counts     # no update after a problem's stop


def test_max_iter_and_tol_minus_inf():
    V, W0, H0 = _inputs()
    n, *_ = _batched(V, W0, H0, beta=1, tol=float("-inf"), max_iter=23)
    assert n.tolist() == [23, 23, 23]
    n, W, H, _ = _batched(V, W0, H0, beta=1, max_iter=0)
    assert n.tolist() == [0, 0, 0] and torch.equal(W, W0) and torch.equal(H, H0)


def test_shared_target_equals_expanded():
    V, W0, H0 = _inputs()
    shared = V[1]
    n1, W1, H1, _ = _batched(shared, W0, H0, beta=2, tol=1e-3, max_iter=60)
    n2, W2, H2, _ = _batched(shared.expand(3, *shared.shape).contiguous(), W0, H0, beta=2, tol=1e-3, max_iter=60)
    assert torch.equal(n1, n2) and torch.equal(W1, W2) and torch.equal(H1, H2)


@pytest.mark.parametrize("frozen", ["W", "H"])
def test_frozen_factor(frozen):
    V, W0, H0 = _inputs()
    kw = dict(trainable_W=frozen != "W", trainable_H=frozen != "H")
    n, W, H, _ = _batched(V, W0, H0, beta=1, tol=1e-3, max_iter=50, **kw)
    assert torch.equal(W if frozen == "W" else H, W0 if frozen == "W" else H0)
    for b in range(3):
        nb, Wb, Hb = _single_oracle(V[b], W0[b], H0[b], beta=1, tol=1e-3, max_iter=50, **kw)
        assert int(n[b]) == nb and torch.equal(W[b], Wb) and torch.equal(H[b], Hb)


def test_constructor_shapes():
    m = BatchedNMF((5, 20, 14), 3)
    assert m.W.shape == (5, 14, 3) and m.H.shape == (5, 20, 3) and m.rank == 3
    assert bool((m.W >= 0).all()) and bool((m.H >= 0).all())
    assert BatchedNMF((2, 6, 4)).rank == 4
    m = BatchedNMF(W=torch.rand(2, 7, 3), H=torch.rand(2, 9, 3))
    assert m.rank == 3
    assert m().shape == (2, 9, 7)
    assert torch.allclose(m(), m.H @ m.W.transpose(1, 2))
    with pytest.raises(ValueError):
        BatchedNMF(W=torch.rand(2, 7, 3), H=torch.rand(2, 9, 4))
    with pytest.raises(ValueError):
        BatchedNMF(W=torch.rand(2, 7, 3), H=torch.rand(3, 9, 3))


def test_refusals():
    V, W0, H0 = _inputs()
    m = BatchedNMF(W=W0, H=H0)
    m._engine_factory = BatchedOracleEngine.factory(OracleNmfEngine, [])
    for prec in ("f16", "f16_split", "bogus"):
        with pytest.raises(ValueError):
            m.fit(V, precision=prec)
    for kw in ({"mask": torch.ones_like(V, dtype=torch.bool)}, {"weight": torch.ones_like(V)}, {"group": object()}):
        with pytest.raises(TypeError):
            m.fit(V, **kw)
    with pytest.raises(NotImplementedError):
        m.fit(V.to_sparse())
    with pytest.raises(NotImplementedError):
        m.sparse_fit(V)
    for bad in (V[:, :, :-1], V[:2], V[0, :-1], V.unsqueeze(0)):
        with pytest.raises(ValueError):
            m.fit(bad)
    with pytest.raises(AssertionError):
        m.fit(V - 0.5)
    with pytest.raises(ValueError):
        m.fit(torch.cat([V[:, :1] * 0, V[:, 1:]], 1), beta=0)
    big = BatchedNMF(W=torch.rand(1, 4, 257), H=torch.rand(1, 3, 257))
    big._engine_factory = BatchedOracleEngine.factory(OracleNmfEngine, [])
    with pytest.raises(ValueError):
        big.fit(torch.rand(1, 3, 4))


def test_last_fit_precision():
    V, W0, H0 = _inputs()
    _, _, _, m = _batched(V, W0, H0, beta=1, max_iter=10, precision="f32")
    assert m.last_fit_precision == "f32"
