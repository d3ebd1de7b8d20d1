"""BatchedNMFD / BatchedNMF2D / BatchedNMF3D host logic on the CPU (no GPU): the per-problem stop rule, freezing of stopped
problems, shared targets, frozen factors, constructor shapes and every refusal, through an engine that fits each problem with
the CPU oracle (the `_engine_factory` hook), and the fits against tests/golden/reference_batched_nd.npz
(tools/make_golden_batched_nd.py: the unmodified reference's NMFD / NMF2D / NMF3D `.fit`, problem by problem)."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from batched_oracle import BatchedOracleEngine
from oracle_engine import OracleNmfdEngine, OracleNmfndEngine
from torchnmf_b200 import NMFD, NMF2D, NMF3D, BatchedNMF, BatchedNMFD, BatchedNMF2D, BatchedNMF3D


SINGLE = {BatchedNMFD: (NMFD, OracleNmfdEngine), BatchedNMF2D: (NMF2D, OracleNmfndEngine),
          BatchedNMF3D: (NMF3D, OracleNmfndEngine)}
CLASSES = {"nmfd": BatchedNMFD, "nmf2d": BatchedNMF2D, "nmf3d": BatchedNMF3D}


def _single_oracle(cls, V, W0, H0, **kw):
    model, engine = SINGLE[cls]
    m = model(W=W0, H=H0, trainable_W=kw.pop("trainable_W", True), trainable_H=kw.pop("trainable_H", True))
    m._engine_factory = engine
    n = m.fit(V, **kw)
    return n, m.W.data.clone(), m.H.data.clone()


def _batched(cls, V, W0, H0, trainable_W=True, trainable_H=True, log=None, **kw):
    m = cls(W=W0, H=H0, trainable_W=trainable_W, trainable_H=trainable_H)
    m._engine_factory = BatchedOracleEngine.factory(SINGLE[cls][1], [] if log is None else log)
    n = m.fit(V, **kw)
    return n, m.W.data.clone(), m.H.data.clone(), m


SHAPES = {BatchedNMFD: ((16,), (4,)), BatchedNMF2D: ((7, 9), (2, 3)), BatchedNMF3D: ((4, 5, 6), (2, 2, 3))}


def _inputs(cls, P=3, B=2, C=5, R=3, seed=0):
    X, K = SHAPES[cls]
    g = torch.Generator().manual_seed(seed)
    J = tuple(x - k + 1 for x, k in zip(X, K))
    scale = torch.linspace(0.2, 2.0, P).view(P, *([1] * (len(X) + 2)))
    V = torch.rand(P, B, C, *X, generator=g) * scale + 0.01
    return V, torch.rand(P, C, R, *K, generator=g) + 0.1, torch.rand(P, B, R, *J, generator=g) + 0.1


def load_batched_nd():
    z = np.load(os.path.join(GOLDEN, "reference_batched_nd.npz"), allow_pickle=False)
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


GOLD = load_batched_nd()


@pytest.mark.parametrize("name", sorted(GOLD))
def test_batched_nd_fit_matches_reference_problem_by_problem(name):
    c = GOLD[name]
    cls = CLASSES[name.split("_")[0]]
    log = []
    n, W, H, m = _batched(cls, c["V"], c["W0"], c["H0"], log=log, beta=c["beta"], tol=c["tol"], max_iter=c["max_iter"])
    assert n.dtype == torch.int64 and n.shape == (4,)
    assert n.tolist() == c["n_iter"]
    for p in range(4):
        assert torch.allclose(W[p], c["W"][p], rtol=1e-4, atol=1e-6), (p, (W[p] - c["W"][p]).abs().max())
        assert torch.allclose(H[p], c["H"][p], rtol=1e-4, atol=1e-6), (p, (H[p] - c["H"][p]).abs().max())
    eng, = log
    assert eng.updates_w == c["n_iter"] and eng.updates_h == c["n_iter"]


def test_golden_problems_stop_at_different_counts():
    for c in GOLD.values():
        assert len(set(c["n_iter"])) >= 3 and max(c["n_iter"]) < c["max_iter"]
    assert sorted(c["beta"] for n, c in GOLD.items() if n.startswith("nmfd")) == [0.5, 1, 2]
    assert {n.split("_")[0] for n in GOLD} == {"nmfd", "nmf2d", "nmf3d"}


@pytest.mark.parametrize("cls", [BatchedNMFD, BatchedNMF2D, BatchedNMF3D])
@pytest.mark.parametrize("beta", [0.5, 1, 2])
def test_each_problem_is_its_own_fit_and_stopped_problems_stay_frozen(cls, beta):
    V, W0, H0 = _inputs(cls)
    log = []
    kw = dict(beta=beta, tol=3e-3, max_iter=90, alpha=0.05, l1_ratio=0.3)
    n, W, H, _ = _batched(cls, V, W0, H0, log=log, **kw)
    counts = []
    for p in range(V.shape[0]):
        npb, Wp, Hp = _single_oracle(cls, V[p], W0[p], H0[p], **kw)
        counts.append(npb)
        assert int(n[p]) == npb
        assert torch.equal(W[p], Wp) and torch.equal(H[p], Hp)
    eng, = log
    assert eng.updates_w == counts and eng.updates_h == counts     # no update after a problem's stop


def test_problems_stop_at_different_counts_and_stay_frozen():
    V, W0, H0 = _inputs(BatchedNMFD)
    log = []
    n, W, H, _ = _batched(BatchedNMFD, V, W0, H0, log=log, beta=1, tol=2e-3, max_iter=150)
    assert len(set(n.tolist())) > 1, n
    eng, = log
    assert eng.updates_w == n.tolist()


def test_max_iter_and_tol_minus_inf():
    V, W0, H0 = _inputs(BatchedNMFD)
    n, *_ = _batched(BatchedNMFD, V, W0, H0, beta=1, tol=float("-inf"), max_iter=23)
    assert n.tolist() == [23, 23, 23]
    n, W, H, _ = _batched(BatchedNMFD, V, W0, H0, beta=1, max_iter=0)
    assert n.tolist() == [0, 0, 0] and torch.equal(W, W0) and torch.equal(H, H0)


@pytest.mark.parametrize("cls", [BatchedNMFD, BatchedNMF2D])
def test_shared_target_equals_expanded(cls):
    V, W0, H0 = _inputs(cls)
    shared = V[1]
    n1, W1, H1, _ = _batched(cls, shared, W0, H0, beta=2, tol=1e-3, max_iter=60)
    n2, W2, H2, _ = _batched(cls, shared.expand(3, *shared.shape).contiguous(), W0, H0, beta=2, tol=1e-3, max_iter=60)
    assert torch.equal(n1, n2) and torch.equal(W1, W2) and torch.equal(H1, H2)


@pytest.mark.parametrize("frozen", ["W", "H"])
@pytest.mark.parametrize("cls", [BatchedNMFD, BatchedNMF3D])
def test_frozen_factor(cls, frozen):
    V, W0, H0 = _inputs(cls)
    kw = dict(trainable_W=frozen != "W", trainable_H=frozen != "H")
    n, W, H, _ = _batched(cls, V, W0, H0, beta=1, tol=1e-3, max_iter=40, **kw)
    assert torch.equal(W if frozen == "W" else H, W0 if frozen == "W" else H0)
    for p in range(3):
        npb, Wp, Hp = _single_oracle(cls, V[p], W0[p], H0[p], beta=1, tol=1e-3, max_iter=40, **kw)
        assert int(n[p]) == npb and torch.equal(W[p], Wp) and torch.equal(H[p], Hp)


def test_constructor_shapes():
    m = BatchedNMFD((5, 2, 14, 30), 3, T=7)
    assert m.W.shape == (5, 14, 3, 7) and m.H.shape == (5, 2, 3, 24) and m.rank == 3
    assert bool((m.W >= 0).all()) and bool((m.H >= 0).all())
    assert BatchedNMFD((2, 1, 6, 9), T=(2,)).rank == 6
    m = BatchedNMF2D((3, 2, 4, 10, 12), 5, kernel_size=(3, 4))
    assert m.W.shape == (3, 4, 5, 3, 4) and m.H.shape == (3, 2, 5, 8, 9)
    assert BatchedNMF2D((3, 2, 4, 10, 12), kernel_size=2).rank == 10       # NMF2D's default rank
    m = BatchedNMF3D((2, 1, 3, 6, 7, 8), 4, kernel_size=2)
    assert m.W.shape == (2, 3, 4, 2, 2, 2) and m.H.shape == (2, 1, 4, 5, 6, 7)
    assert BatchedNMF3D((2, 1, 3, 6, 7, 8), kernel_size=2).rank == 7       # NMF3D's default rank
    for cls in (BatchedNMFD, BatchedNMF2D, BatchedNMF3D):
        V, W0, H0 = _inputs(cls)
        m = cls(W=W0, H=H0)
        assert m.rank == 3 and tuple(m.kernel_size) == SHAPES[cls][1]
        single = SINGLE[cls][0]
        out = m()
        assert out.shape == V.shape
        for p in range(3):
            assert torch.allclose(out[p], single(W=W0[p], H=H0[p])(), rtol=1e-5, atol=1e-5)
        with pytest.raises(ValueError):
            cls(W=W0, H=H0[:, :, :2])                                          # rank mismatch
        with pytest.raises(ValueError):
            cls(W=W0, H=H0[:2])                                                # problem count mismatch
        with pytest.raises(ValueError):
            cls(W=W0[0], H=H0)                                                 # axes


@pytest.mark.parametrize("cls", [BatchedNMFD, BatchedNMF2D, BatchedNMF3D])
def test_refusals(cls):
    V, W0, H0 = _inputs(cls)
    m = cls(W=W0, H=H0)
    m._engine_factory = BatchedOracleEngine.factory(SINGLE[cls][1], [])
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
    for bad in (V[..., :-1], V[:2], V[:, :1], V[:, :, :-1], V[0, :, :-1], V.unsqueeze(0)):
        with pytest.raises(ValueError):
            m.fit(bad)
    with pytest.raises(AssertionError):
        m.fit(V - 0.5)
    zero = V.clone()
    zero[1, 0, 0] = 0
    with pytest.raises(ValueError):
        m.fit(zero, beta=0)
    X, K = SHAPES[cls]
    big = cls(W=torch.rand(1, 2, 257, *K), H=torch.rand(1, 1, 257, *(x - k + 1 for x, k in zip(X, K))))
    big._engine_factory = BatchedOracleEngine.factory(SINGLE[cls][1], [])
    with pytest.raises(ValueError):
        big.fit(torch.rand(1, 1, 2, *X))


def test_last_fit_precision():
    V, W0, H0 = _inputs(BatchedNMFD)
    _, _, _, m = _batched(BatchedNMFD, V, W0, H0, beta=1, max_iter=10, precision="f32")
    assert m.last_fit_precision == "f32"


def test_batched_nmf_keeps_its_iterate_path():
    """The shared loop takes `iterate` where the engine has it: BatchedNMF's engine gets one call per 10 iterations."""
    from oracle_engine import OracleNmfEngine
    g = torch.Generator().manual_seed(3)
    V, W0, H0 = torch.rand(2, 9, 7, generator=g) + 0.1, torch.rand(2, 7, 3, generator=g), torch.rand(2, 9, 3, generator=g)
    m = BatchedNMF(W=W0, H=H0)
    log = []
    m._engine_factory = BatchedOracleEngine.factory(OracleNmfEngine, log)
    n = m.fit(V, beta=2, tol=float("-inf"), max_iter=25)
    eng, = log
    assert n.tolist() == [25, 25] and [c[:2] for c in eng.calls] == [("iterate", 10), ("iterate", 10), ("iterate", 5)]


def test_public_classes_document_themselves_and_import_without_docstrings():
    """The batched classes carry their own docstrings (Args, in-place layout, workspace), and the package imports under
    `python -OO`, where every docstring is stripped."""
    import subprocess
    import sys

    for cls in (BatchedNMFD, BatchedNMF2D, BatchedNMF3D):
        doc = cls.__doc__
        assert doc and "Args:" in doc and "in place" in doc and "Workspace" in doc, cls.__name__
    pkg = os.path.join(os.path.dirname(GOLDEN), "..", "pytorch-nmf_b200")
    r = subprocess.run([sys.executable, "-OO", "-B", "-c", "import torchnmf_b200; print(torchnmf_b200.BatchedNMFD.__doc__)"],
                       capture_output=True, text=True, env={**os.environ, "PYTHONPATH": os.path.abspath(pkg)}, timeout=300)
    assert r.returncode == 0, r.stderr
    assert r.stdout.strip() == "None"
