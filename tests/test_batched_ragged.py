"""BatchedNMF.fit(V, ..., lengths=L) -- a ragged batch, problem b being the fit of V[b, :L[b]] -- on the CPU (no GPU): the
host logic through an engine that fits each problem's real rows with the CPU oracle (the `_engine_factory` hook), every
refusal, and the fits against tests/golden/reference_batched_ragged.npz (tools/make_golden_batched_ragged.py: the
unmodified reference's `NMF.fit` on each prefix V[b, :L[b]])."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from batched_oracle import BatchedOracleEngine
from oracle_engine import OracleNmfEngine
from torchnmf_b200 import NMF, BatchedNMF, BatchedNMFD, BatchedNMF2D, BatchedNMF3D


def _factory(log):
    def make(V, W, H, **kw):
        log.append(kw)
        if "lengths" not in kw:
            raise AssertionError("a fit without lengths reached the ragged factory")
        eng = BatchedOracleEngine(V, W, H, OracleNmfEngine, kw["lengths"])
        log.append(eng)
        return eng
    return make


def _ragged(V, W0, H0, lengths, log=None, trainable_W=True, trainable_H=True, **kw):
    m = BatchedNMF(W=W0, H=H0, trainable_W=trainable_W, trainable_H=trainable_H)
    m._engine_factory = _factory([] if log is None else log)
    n = m.fit(V, lengths=lengths, **kw)
    return n, m.W.data.clone(), m.H.data.clone(), m


def _single_oracle(V, W0, H0, **kw):
    m = NMF(W=W0, H=H0, trainable_W=kw.pop("trainable_W", True), trainable_H=kw.pop("trainable_H", True))
    m._engine_factory = OracleNmfEngine
    n = m.fit(V, **kw)
    return n, m.W.data.clone(), m.H.data.clone()


def _inputs(lengths=(20, 7, 13, 1), N=20, C=14, R=4, seed=0, pad=float("nan"), sentinel=5.0):
    B = len(lengths)
    g = torch.Generator().manual_seed(seed)
    V = torch.rand(B, N, C, generator=g) * torch.linspace(0.2, 2.0, B).view(B, 1, 1) + 0.01
    W0 = torch.rand(B, C, R, generator=g) + 0.1
    H0 = torch.rand(B, N, R, generator=g) + 0.1
    for b, L in enumerate(lengths):
        V[b, L:] = pad
        H0[b, L:] = sentinel
    return V, W0, H0


def load_ragged():
    z = np.load(os.path.join(GOLDEN, "reference_batched_ragged.npz"), allow_pickle=False)
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
def test_ragged_fit_matches_reference_prefix_by_prefix(name):
    c = GOLD[name]
    log = []
    n, W, H, _ = _ragged(c["V"], c["W0"], c["H0"], c["lengths"], log=log, beta=c["beta"], tol=c["tol"],
                         max_iter=c["max_iter"])
    assert n.dtype == torch.int64 and n.tolist() == c["n_iter"]
    assert torch.allclose(W, c["W"], rtol=2e-5, atol=1e-7), (W - c["W"]).abs().max()
    for b, L in enumerate(c["lengths"]):
        assert torch.allclose(H[b, :L], c["H"][b, :L], rtol=2e-5, atol=1e-7), (b, (H[b, :L] - c["H"][b, :L]).abs().max())
        assert torch.equal(H[b, L:], c["H0"][b, L:])              # the sentinel padding, untouched
    kw, eng = log
    assert kw == {"lengths": c["lengths"]} and eng.updates_h == c["n_iter"]


def test_golden_ragged_problems_differ():
    for c in GOLD.values():
        assert len(set(c["n_iter"])) >= 3 and max(c["n_iter"]) < c["max_iter"]
        assert len(set(c["lengths"])) == len(c["lengths"]) and max(c["lengths"]) == c["V"].shape[1]
        assert bool(torch.isnan(c["V"]).any())                     # NaN padding the oracle engines never see
    assert sorted(c["beta"] for c in GOLD.values()) == [0.5, 1, 2]


@pytest.mark.parametrize("beta", [0, 0.5, 1, 2, 3])
def test_each_problem_is_its_own_fit_on_its_rows(beta):
    lengths = [20, 7, 13, 1]
    V, W0, H0 = _inputs(lengths)
    kw = dict(beta=beta, tol=3e-3, max_iter=120, alpha=0.05, l1_ratio=0.3)
    log = []
    n, W, H, _ = _ragged(V, W0, H0, lengths, log=log, **kw)
    counts = []
    for b, L in enumerate(lengths):
        nb, Wb, Hb = _single_oracle(V[b, :L], W0[b], H0[b, :L], **kw)
        counts.append(nb)
        assert int(n[b]) == nb
        assert torch.equal(W[b], Wb) and torch.equal(H[b, :L], Hb)
        assert torch.equal(H[b, L:], H0[b, L:])
    assert log[1].updates_h == counts                               # no update after a problem's stop
    if beta == 1:
        assert len(set(counts)) > 1, counts


@pytest.mark.parametrize("as_tensor", [False, True])
def test_lengths_as_list_or_tensor(as_tensor):
    lengths = [20, 7, 13, 1]
    V, W0, H0 = _inputs(lengths)
    ref = _ragged(V, W0, H0, lengths, beta=1, tol=1e-3, max_iter=40)
    arg = torch.tensor(lengths, dtype=torch.int32) if as_tensor else tuple(np.int64(L) for L in lengths)
    log = []
    got = _ragged(V, W0, H0, arg, log=log, beta=1, tol=1e-3, max_iter=40)
    assert log[0] == {"lengths": lengths} and all(type(L) is int for L in log[0]["lengths"])
    assert torch.equal(ref[0], got[0]) and torch.equal(ref[1], got[1]) and torch.equal(ref[2], got[2])


@pytest.mark.parametrize("frozen", ["W", "H"])
def test_frozen_factor(frozen):
    lengths = [20, 7, 13, 1]
    V, W0, H0 = _inputs(lengths)
    kw = dict(trainable_W=frozen != "W", trainable_H=frozen != "H")
    n, W, H, _ = _ragged(V, W0, H0, lengths, beta=1, tol=1e-3, max_iter=50, **kw)
    for b, L in enumerate(lengths):
        nb, Wb, Hb = _single_oracle(V[b, :L], W0[b], H0[b, :L], beta=1, tol=1e-3, max_iter=50, **kw)
        assert int(n[b]) == nb and torch.equal(W[b], Wb) and torch.equal(H[b, :L], Hb)
        assert torch.equal(H[b, L:], H0[b, L:])


def test_checks_look_at_the_real_rows_only():
    lengths = [20, 7, 13, 1]
    V, W0, H0 = _inputs(lengths, pad=-1.0)                          # negative padding: not part of any problem
    _ragged(V, W0, H0, lengths, beta=1, max_iter=10)
    V0, _, _ = _inputs(lengths, pad=0.0)                            # zero padding: beta <= 0 is still fine
    _ragged(V0, W0, H0, lengths, beta=0, max_iter=10)
    Vneg = V.clone()
    Vneg[1, 3, 2] = -0.5
    with pytest.raises(AssertionError):
        _ragged(Vneg, W0, H0, lengths, beta=1, max_iter=10)
    Vz = V.clone()
    Vz[2, 12, 0] = 0.0
    with pytest.raises(ValueError):
        _ragged(Vz, W0, H0, lengths, beta=0, max_iter=10)


def test_all_lengths_n_equal_the_uniform_fit():
    V, W0, H0 = _inputs((20, 20, 20), pad=0.0)
    ref = BatchedNMF(W=W0, H=H0)
    ref._engine_factory = lambda V, W, H: BatchedOracleEngine(V, W, H, OracleNmfEngine, [20, 20, 20])
    n_ref = ref.fit(V, beta=1.5, tol=1e-3, max_iter=60)
    n, W, H, _ = _ragged(V, W0, H0, [20, 20, 20], beta=1.5, tol=1e-3, max_iter=60)
    assert torch.equal(n, n_ref) and torch.equal(W, ref.W.data) and torch.equal(H, ref.H.data)


def _refused(m, V, exc=ValueError, **kw):
    log = []
    m._engine_factory = _factory(log)
    with pytest.raises(exc):
        m.fit(V, **kw)
    assert log == []                                                # refused before an engine exists


def test_refusals():
    lengths = [20, 7, 13, 1]
    V, W0, H0 = _inputs(lengths)
    m = BatchedNMF(W=W0, H=H0)
    for bad in ([20, 7, 13], [20, 7, 13, 1, 1], [0, 7, 13, 1], [21, 7, 13, 1], [20, -1, 13, 1], [20.0, 7, 13, 1],
                [True, 7, 13, 1], torch.tensor([20.0, 7, 13, 1]), torch.tensor([[20, 7, 13, 1]]), torch.tensor(7),
                torch.tensor([True, True, True, True]), "abcd", 7, {"a": 1}):
        _refused(m, V, lengths=bad)
    _refused(m, V[0], lengths=[20, 7, 13, 1])                       # a shared 2-D target
    _refused(m, V, lengths=lengths, beta=2, solver="cd")
    for kw in ({"mask": torch.ones_like(V, dtype=torch.bool)}, {"weight": torch.ones_like(V)}, {"group": object()}):
        _refused(m, V, TypeError, lengths=lengths, **kw)
    for cls, V5, W5, H5 in ((BatchedNMFD, torch.rand(2, 1, 6, 12), torch.rand(2, 6, 3, 4), torch.rand(2, 1, 3, 9)),
                            (BatchedNMF2D, torch.rand(2, 1, 6, 5, 12), torch.rand(2, 6, 3, 2, 4),
                             torch.rand(2, 1, 3, 4, 9)),
                            (BatchedNMF3D, torch.rand(2, 1, 6, 3, 5, 12), torch.rand(2, 6, 3, 1, 2, 4),
                             torch.rand(2, 1, 3, 3, 4, 9))):
        _refused(cls(W=W5, H=H5), V5, lengths=[1, 1])


def test_default_keeps_the_three_argument_factory():
    V, W0, H0 = _inputs((20, 20, 20, 20), pad=0.5)
    seen = []

    def make(V, W, H):                                              # no lengths keyword: today's factories
        seen.append(True)
        return BatchedOracleEngine(V, W, H, OracleNmfEngine, [20] * 4)
    m = BatchedNMF(W=W0, H=H0)
    m._engine_factory = make
    m.fit(V, beta=1, max_iter=10)
    assert seen == [True]
