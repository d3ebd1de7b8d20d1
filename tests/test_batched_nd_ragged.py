"""BatchedNMFD / BatchedNMF2D / BatchedNMF3D .fit(V, ..., lengths=L) -- a ragged batch along the last convolved axis,
problem p being the fit of V[p, ..., :L[p]] -- on the CPU (no GPU): the host logic through an engine that fits each
problem's real positions with the CPU oracle (the `_engine_factory` hook), every refusal, and the fits against
tests/golden/reference_batched_nd_ragged.npz (tools/make_golden_batched_nd_ragged.py: the unmodified reference's
NMFD / NMF2D / NMF3D `.fit` on each problem's real positions)."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from batched_oracle import BatchedOracleEngine
from oracle_engine import OracleNmfdEngine, OracleNmfndEngine
from torchnmf_b200 import NMFD, NMF2D, NMF3D, BatchedNMFD, BatchedNMF2D, BatchedNMF3D

SENTINEL = 5.0


SINGLE = {BatchedNMFD: (NMFD, OracleNmfdEngine), BatchedNMF2D: (NMF2D, OracleNmfndEngine),
          BatchedNMF3D: (NMF3D, OracleNmfndEngine)}
CLASSES = {"nmfd": BatchedNMFD, "nmf2d": BatchedNMF2D, "nmf3d": BatchedNMF3D}


def _factory(cls, log):
    def make(V, W, H, **kw):
        log.append(kw)
        if "lengths" not in kw:
            raise AssertionError("a fit without lengths reached the ragged factory")
        eng = BatchedOracleEngine(V, W, H, SINGLE[cls][1], kw["lengths"])
        log.append(eng)
        return eng
    return make


def _ragged(cls, V, W0, H0, lengths, log=None, trainable_W=True, trainable_H=True, **kw):
    m = cls(W=W0, H=H0, trainable_W=trainable_W, trainable_H=trainable_H)
    m._engine_factory = _factory(cls, [] if log is None else log)
    n = m.fit(V, lengths=lengths, **kw)
    return n, m.W.data.clone(), m.H.data.clone(), m


def _single_oracle(cls, V, W0, H0, **kw):
    model, engine = SINGLE[cls]
    m = model(W=W0, H=H0, trainable_W=kw.pop("trainable_W", True), trainable_H=kw.pop("trainable_H", True))
    m._engine_factory = engine
    n = m.fit(V, **kw)
    return n, m.W.data.clone(), m.H.data.clone()


SHAPES = {BatchedNMFD: ((), (4,)), BatchedNMF2D: ((5,), (2, 3)), BatchedNMF3D: ((3, 4), (2, 1, 3))}
LENGTHS = [16, 4, 11, 7]


def _inputs(cls, lengths=LENGTHS, B=2, C=5, R=3, seed=0, pad=float("nan")):
    outer, K = SHAPES[cls]
    P, X = len(lengths), max(lengths)
    g = torch.Generator().manual_seed(seed)
    shape = (P, B, C) + outer + (X,)
    J = tuple(x - k + 1 for x, k in zip(outer + (X,), K))
    V = torch.rand(shape, generator=g) * torch.linspace(0.2, 2.0, P).view(P, *([1] * (len(shape) - 1))) + 0.01
    W0 = torch.rand((P, C, R) + K, generator=g) + 0.1
    H0 = torch.rand((P, B, R) + J, generator=g) + 0.1
    for p, L in enumerate(lengths):
        V[p, ..., L:] = pad
        H0[p, ..., L - K[-1] + 1:] = SENTINEL
    return V, W0, H0


def _check(cls, V, W0, H0, lengths, n, W, H, **kw):
    T = W0.shape[-1]
    counts = []
    for p, L in enumerate(lengths):
        lin = L - T + 1
        nb, Wb, Hb = _single_oracle(cls, V[p, ..., :L].contiguous(), W0[p], H0[p, ..., :lin].contiguous(), **kw)
        counts.append(nb)
        assert int(n[p]) == nb
        assert torch.equal(W[p], Wb) and torch.equal(H[p, ..., :lin], Hb)
        assert torch.equal(H[p, ..., lin:], H0[p, ..., lin:])       # the sentinel padding, untouched
    return counts


def load_ragged():
    z = np.load(os.path.join(GOLDEN, "reference_batched_nd_ragged.npz"), allow_pickle=False)
    cases = {}
    for key in z.files:
        name, field = key.split("/", 1)
        v = z[key]
        if field in ("V", "W0", "H0", "W", "H"):
            v = torch.from_numpy(v.copy())
        elif field in ("n_iter", "lengths"):
            v = [int(x) for x in v]
        else:
            v = float(v)
            if field == "max_iter":
                v = int(v)
        cases.setdefault(name, {})[field] = v
    return cases


GOLD = load_ragged()


@pytest.mark.parametrize("name", sorted(GOLD))
def test_ragged_fit_matches_reference_problem_by_problem(name):
    c = GOLD[name]
    cls = CLASSES[name.split("_")[0]]
    T = c["W0"].shape[-1]
    log = []
    n, W, H, _ = _ragged(cls, c["V"], c["W0"], c["H0"], c["lengths"], log=log, beta=c["beta"], tol=c["tol"],
                         max_iter=c["max_iter"])
    assert n.dtype == torch.int64 and n.tolist() == c["n_iter"]
    assert torch.allclose(W, c["W"], rtol=2e-5, atol=1e-7), (W - c["W"]).abs().max()
    for p, L in enumerate(c["lengths"]):
        lin = L - T + 1
        assert torch.allclose(H[p, ..., :lin], c["H"][p, ..., :lin], rtol=2e-5, atol=1e-7), p
        assert torch.equal(H[p, ..., lin:], c["H0"][p, ..., lin:])
    kw, eng = log
    assert kw == {"lengths": c["lengths"]} and eng.updates_h == c["n_iter"]


def test_golden_ragged_problems_differ():
    for c in GOLD.values():
        assert len(set(c["n_iter"])) >= 3 and max(c["n_iter"]) < c["max_iter"]
        assert len(set(c["lengths"])) == len(c["lengths"]) and max(c["lengths"]) == c["V"].shape[-1]
        assert bool(torch.isnan(c["V"]).any())                     # NaN padding the oracle engines never see
    assert sorted(n.split("_")[0] for n in GOLD) == ["nmf2d", "nmf3d", "nmfd", "nmfd", "nmfd"]


@pytest.mark.parametrize("cls", [BatchedNMFD, BatchedNMF2D, BatchedNMF3D])
@pytest.mark.parametrize("beta", [0, 1, 2])
def test_each_problem_is_its_own_fit(cls, beta):
    V, W0, H0 = _inputs(cls)
    kw = dict(beta=beta, tol=3e-3, max_iter=60, alpha=0.05, l1_ratio=0.3)
    log = []
    n, W, H, _ = _ragged(cls, V, W0, H0, LENGTHS, log=log, **kw)
    counts = _check(cls, V, W0, H0, LENGTHS, n, W, H, **kw)
    assert log[1].updates_h == counts                               # no update after a problem's stop


@pytest.mark.parametrize("as_tensor", [False, True])
def test_lengths_as_list_or_tensor(as_tensor):
    V, W0, H0 = _inputs(BatchedNMFD)
    ref = _ragged(BatchedNMFD, V, W0, H0, LENGTHS, beta=1, tol=1e-3, max_iter=40)
    arg = torch.tensor(LENGTHS, dtype=torch.int32) if as_tensor else tuple(np.int64(L) for L in LENGTHS)
    log = []
    got = _ragged(BatchedNMFD, V, W0, H0, arg, log=log, beta=1, tol=1e-3, max_iter=40)
    assert log[0] == {"lengths": LENGTHS} and all(type(L) is int for L in log[0]["lengths"])
    assert torch.equal(ref[0], got[0]) and torch.equal(ref[1], got[1]) and torch.equal(ref[2], got[2])


@pytest.mark.parametrize("frozen", ["W", "H"])
def test_frozen_factor(frozen):
    V, W0, H0 = _inputs(BatchedNMFD)
    kw = dict(beta=1, tol=1e-3, max_iter=40, trainable_W=frozen != "W", trainable_H=frozen != "H")
    n, W, H, _ = _ragged(BatchedNMFD, V, W0, H0, LENGTHS, **kw)
    _check(BatchedNMFD, V, W0, H0, LENGTHS, n, W, H, **kw)


def test_staged_write_back_keeps_the_padding():
    """The fit's write-back mask of H: the real positions only, for every class."""
    for cls in (BatchedNMFD, BatchedNMF2D, BatchedNMF3D):
        V, W0, H0 = _inputs(cls)
        m = cls(W=W0, H=H0)
        real = m._real_cells(LENGTHS)
        assert real.shape == H0.shape
        T = W0.shape[-1]
        for p, L in enumerate(LENGTHS):
            assert bool(real[p, ..., :L - T + 1].all()) and not bool(real[p, ..., L - T + 1:].any())
        staged = torch.full_like(H0, -1.0)
        H = H0.clone()
        H[real] = staged[real]
        for p, L in enumerate(LENGTHS):
            assert bool((H[p, ..., :L - T + 1] == -1).all()) and bool((H[p, ..., L - T + 1:] == SENTINEL).all())


def test_checks_look_at_the_real_positions_only():
    V, W0, H0 = _inputs(BatchedNMFD, pad=-1.0)                     # negative padding: not part of any problem
    _ragged(BatchedNMFD, V, W0, H0, LENGTHS, beta=1, max_iter=10)
    V0, _, _ = _inputs(BatchedNMFD, pad=0.0)                        # zero padding: beta <= 0 is still fine
    _ragged(BatchedNMFD, V0, W0, H0, LENGTHS, beta=0, max_iter=10)
    Vneg = V.clone()
    Vneg[1, 0, 2, 3] = -0.5
    with pytest.raises(AssertionError):
        _ragged(BatchedNMFD, Vneg, W0, H0, LENGTHS, beta=1, max_iter=10)
    Vz = V.clone()
    Vz[2, 1, 0, 10] = 0.0
    with pytest.raises(ValueError):
        _ragged(BatchedNMFD, Vz, W0, H0, LENGTHS, beta=0, max_iter=10)


def test_full_lengths_equal_the_uniform_fit():
    V, W0, H0 = _inputs(BatchedNMFD, lengths=[16, 16, 16], pad=0.0)
    ref = BatchedNMFD(W=W0, H=H0)
    ref._engine_factory = lambda V, W, H: BatchedOracleEngine(V, W, H, OracleNmfdEngine, [16] * 3)
    n_ref = ref.fit(V, beta=1.5, tol=1e-3, max_iter=40)
    n, W, H, _ = _ragged(BatchedNMFD, V, W0, H0, [16] * 3, beta=1.5, tol=1e-3, max_iter=40)
    assert torch.equal(n, n_ref) and torch.equal(W, ref.W.data) and torch.equal(H, ref.H.data)


def _refused(m, V, exc=ValueError, **kw):
    log = []
    m._engine_factory = _factory(type(m), log)
    with pytest.raises(exc):
        m.fit(V, **kw)
    assert log == []                                                # refused before an engine exists


@pytest.mark.parametrize("cls", [BatchedNMFD, BatchedNMF2D, BatchedNMF3D])
def test_refusals(cls):
    V, W0, H0 = _inputs(cls)
    m = cls(W=W0, H=H0)
    short = W0.shape[-1] - 1                                        # below the last kernel size
    for bad in ([16, 4, 11], [16, 4, 11, 7, 7], [short, 4, 11, 7], [17, 4, 11, 7], [16, -1, 11, 7], [16.0, 4, 11, 7],
                [True, 4, 11, 7], torch.tensor([16.0, 4, 11, 7]), torch.tensor([[16, 4, 11, 7]]), torch.tensor(7),
                torch.tensor([True, True, True, True]), "abcd", 7, {"a": 1}):
        _refused(m, V, lengths=bad)
    _refused(m, V[0], lengths=LENGTHS)                              # a shared target
    _refused(m, V, lengths=LENGTHS, beta=2, solver="cd")
    for kw in ({"mask": torch.ones_like(V, dtype=torch.bool)}, {"weight": torch.ones_like(V)}, {"group": object()}):
        _refused(m, V, TypeError, lengths=LENGTHS, **kw)


def test_default_keeps_the_three_argument_factory():
    V, W0, H0 = _inputs(BatchedNMFD, lengths=[16] * 4, pad=0.5)
    seen = []

    def make(V, W, H):                                              # no lengths keyword: today's factories
        seen.append(True)
        return BatchedOracleEngine(V, W, H, OracleNmfdEngine, [16] * 4)
    m = BatchedNMFD(W=W0, H=H0)
    m._engine_factory = make
    m.fit(V, beta=1, max_iter=10)
    assert seen == [True]
