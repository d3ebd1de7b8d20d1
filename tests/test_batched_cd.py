"""`BatchedNMF.fit(V, beta=2, solver="cd")` without a GPU: its host logic through a batched engine whose every problem is
the float64 HALS oracle (tests/cd_oracle.py), plugged in with the `_engine_factory` hook, against single `NMF.fit(...,
solver="cd")` fits on the single oracle engine of tests/test_cd.py; the refusals; and the C ABI's new symbols."""
import ctypes
import os

import pytest
import torch

from batched_oracle import BatchedOracleEngine
from test_cd import CdOracleEngine
from torchnmf_b200 import NMF, BatchedNMF, BatchedNMF2D, BatchedNMF3D, BatchedNMFD

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _inputs(B=6, N=23, C=17, R=4, seed=0):
    """B planted problems of graded noise, so their fits stop at different checks; fp32-exact float64 values."""
    g = torch.Generator().manual_seed(seed)
    V = torch.rand(B, N, R, generator=g, dtype=torch.float64) @ torch.rand(B, R, C, generator=g, dtype=torch.float64)
    V += torch.logspace(-3, 0, B, dtype=torch.float64).view(B, 1, 1) * torch.rand(B, N, C, generator=g, dtype=torch.float64)
    W = torch.rand(B, C, R, generator=g) + 0.1
    H = torch.rand(B, N, R, generator=g) + 0.1
    return V.float().double(), W.double(), H.double()


def _batched(V, W0, H0, trainable_W=True, trainable_H=True, **kw):
    m = BatchedNMF(W=W0, H=H0, trainable_W=trainable_W, trainable_H=trainable_H).double()
    log = []
    m._engine_factory = BatchedOracleEngine.factory(CdOracleEngine, log)
    n = m.fit(V, **kw)
    eng, = log
    return n, m.W.data.clone(), m.H.data.clone(), eng, m


def _single(V, W0, H0, trainable_W=True, trainable_H=True, **kw):
    m = NMF(W=W0, H=H0, trainable_W=trainable_W, trainable_H=trainable_H).double()
    m._engine_factory = CdOracleEngine
    n = m.fit(V, **kw)
    return n, m.W.data.clone(), m.H.data.clone()


@pytest.mark.parametrize("alpha,l1_ratio", [(0, 0), (0.1, 0.0), (0.2, 0.25)])
def test_each_problem_is_its_single_cd_fit_and_stopped_problems_stay_frozen(alpha, l1_ratio):
    V, W0, H0 = _inputs()
    kw = dict(beta=2, tol=5e-4, max_iter=150, alpha=alpha, l1_ratio=l1_ratio, solver="cd")
    n, W, H, eng, _ = _batched(V, W0, H0, **kw)
    counts = []
    for b in range(V.shape[0]):
        nb, Wb, Hb = _single(V[b], W0[b], H0[b], **kw)
        counts.append(nb)
        assert int(n[b]) == nb
        assert torch.equal(W[b], Wb) and torch.equal(H[b], Hb)
    assert len(set(counts)) >= 3, counts
    assert eng.updates_w == counts and eng.updates_h == counts      # no update after a problem's stop
    assert all(c[0] == "cd_iterate" for c in eng.calls)


def test_iterations_between_checks_run_in_one_call():
    V, W0, H0 = _inputs()
    _, _, _, eng, m = _batched(V, W0, H0, beta=2, tol=float("-inf"), max_iter=25, alpha=0.4, l1_ratio=0.25, solver="cd")
    assert eng.calls == [("cd_iterate", 10, 0.1, pytest.approx(0.3)), ("cd_iterate", 10, 0.1, pytest.approx(0.3)),
                         ("cd_iterate", 5, 0.1, pytest.approx(0.3))]
    assert m.last_fit_precision == "f32"


@pytest.mark.parametrize("frozen", ["W", "H"])
def test_frozen_factor_runs_per_factor_updates_of_the_other(frozen):
    V, W0, H0 = _inputs()
    fr = dict(trainable_W=frozen != "W", trainable_H=frozen != "H")
    kw = dict(beta=2, tol=1e-5, max_iter=60, alpha=0.1, l1_ratio=0.5, solver="cd")
    n, W, H, eng, _ = _batched(V, W0, H0, **fr, **kw)
    assert torch.equal(W if frozen == "W" else H, W0 if frozen == "W" else H0)
    for b in range(V.shape[0]):
        nb, Wb, Hb = _single(V[b], W0[b], H0[b], **fr, **kw)
        assert int(n[b]) == nb and torch.equal(W[b], Wb) and torch.equal(H[b], Hb)
    assert {c[:2] for c in eng.calls} == {("cd_update", 1 if frozen == "W" else 0)}
    assert all(c[2:] == (0.05, 0.05) for c in eng.calls)


def test_shared_target_equals_expanded():
    V, W0, H0 = _inputs()
    shared = V[2]
    kw = dict(beta=2, tol=1e-4, max_iter=60, solver="cd")
    n1, W1, H1, _, _ = _batched(shared, W0, H0, **kw)
    n2, W2, H2, _, _ = _batched(shared.expand(6, *shared.shape).contiguous(), W0, H0, **kw)
    assert torch.equal(n1, n2) and torch.equal(W1, W2) and torch.equal(H1, H2)


@pytest.mark.parametrize("frozen", [None, "W"])
def test_solver_mu_is_the_default_call(frozen):
    V, W0, H0 = _inputs()
    fr = dict(trainable_W=frozen != "W", trainable_H=frozen != "H")
    runs = []
    for kw in ({}, {"solver": "mu"}):
        n, W, H, eng, _ = _batched(V, W0, H0, beta=2, tol=1e-4, max_iter=40, **fr, **kw)
        runs.append((n, W, H, eng.calls))
    assert torch.equal(runs[0][0], runs[1][0]) and runs[0][3] == runs[1][3]
    assert torch.equal(runs[0][1], runs[1][1]) and torch.equal(runs[0][2], runs[1][2])
    assert {c[0] for c in runs[0][3]} == ({"iterate"} if frozen is None else {"update_h"})


def _no_engine(*a, **k):
    raise AssertionError("an engine was built before the refusal")


@pytest.mark.parametrize("case", ["beta1", "beta0.5", "f16", "f16_split", "solver", "solver_mu_typo", "nmfd", "nmf2d",
                                  "nmf3d", "rank"])
def test_value_errors_raise_before_any_engine(case):
    V, W0, H0 = _inputs()
    m = BatchedNMF(W=W0, H=H0)
    kw, beta = {"solver": "cd"}, 2
    if case == "beta1":
        beta = 1
    elif case == "beta0.5":
        beta = 0.5
    elif case in ("f16", "f16_split"):
        kw["precision"] = case
    elif case == "solver":
        kw["solver"] = "hals"
    elif case == "solver_mu_typo":
        kw["solver"], beta = "MU", 1
    elif case == "nmfd":
        m, V = BatchedNMFD(W=torch.rand(2, 5, 3, 4), H=torch.rand(2, 2, 3, 7)), torch.rand(2, 2, 5, 10)
    elif case == "nmf2d":
        m, V = BatchedNMF2D(W=torch.rand(2, 5, 3, 2, 4), H=torch.rand(2, 1, 3, 5, 7)), torch.rand(2, 1, 5, 6, 10)
    elif case == "nmf3d":
        m = BatchedNMF3D(W=torch.rand(2, 5, 3, 2, 2, 4), H=torch.rand(2, 1, 3, 3, 5, 7))
        V = torch.rand(2, 1, 5, 4, 6, 10)
    elif case == "rank":
        m, V = BatchedNMF(W=torch.rand(1, 4, 257), H=torch.rand(1, 3, 257)), torch.rand(1, 3, 4)
    m._engine_factory = _no_engine
    with pytest.raises(ValueError) as e:
        m.fit(V, beta, **kw)
    if case.startswith("nmf"):
        assert "BatchedNMF only" in str(e.value)


def test_other_refusals_keep_their_errors():
    V, W0, H0 = _inputs()
    m = BatchedNMF(W=W0, H=H0)
    m._engine_factory = _no_engine
    for kw in ({"mask": torch.ones_like(V, dtype=torch.bool)}, {"weight": torch.ones_like(V)}, {"group": object()}):
        with pytest.raises(TypeError):
            m.fit(V, 2, solver="cd", **kw)
    with pytest.raises(NotImplementedError):
        m.fit(V.to_sparse(), 2, solver="cd")


def test_batched_cd_entry_points_are_bound_and_refuse_a_null_context():
    from torchnmf_b200 import _capi
    _vp, _dbl, _int = ctypes.c_void_p, ctypes.c_double, ctypes.c_int
    assert _capi.SIGNATURES["nmfb200_nmf_batched_cd_update"] == (_int, [_vp, _vp, _vp, _int, _dbl, _dbl, _vp])
    assert _capi.SIGNATURES["nmfb200_nmf_batched_cd_iterate"] == (_int, [_vp, _vp, _vp, _dbl, _dbl, _int, _vp])
    lib = _capi.load()
    assert lib.nmfb200_nmf_batched_cd_update(None, None, None, 0, 0.0, 0.0, None) == 1          # NMFB200_ERR_INVALID
    assert b"null context" in lib.nmfb200_last_error()
    assert lib.nmfb200_nmf_batched_cd_iterate(None, None, None, 0.0, 0.0, 1, None) == 1
    assert b"null context" in lib.nmfb200_last_error()
    header = " ".join(open(os.path.join(ROOT, "include", "nmf_b200.h")).read().split())
    assert ("int nmfb200_nmf_batched_cd_update(nmfb200_ctx* ctx, float* W, float* H, int which, double l1_reg, "
            "double l2_reg, void* stream);") in header
    assert ("int nmfb200_nmf_batched_cd_iterate(nmfb200_ctx* ctx, float* W, float* H, double l1_reg, double l2_reg, "
            "int n_iter, void* stream);") in header
    assert lib.nmfb200_abi_version() == 2
