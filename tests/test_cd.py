"""Coordinate descent at beta 2 (`NMF.fit(V, beta=2, solver="cd")`), without a GPU.

The float64 HALS oracle (tests/cd_oracle.py) is checked against the objective it descends -- never rising across a column
step, the KKT conditions at convergence, a dead component left alone -- and then the host logic of `fit(solver="cd")`
(validation, the loop, the stop rule, frozen factors, the alpha / l1_ratio mapping) runs through an oracle engine plugged in
with the `_engine_factory` hook.
"""
import ctypes
import os

import pytest
import torch

import cd_oracle as cdo
from oracle import mu_oracle as orc
from oracle_engine import OracleNmfEngine
from torchnmf_b200 import NMF, NMF2D, NMF3D, NMFD

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class CdOracleEngine(OracleNmfEngine):
    """The MU oracle engine plus the two coordinate-descent calls, from tests/cd_oracle.py; logs every call."""
    log = None

    def __init__(self, V, W, H):
        super().__init__(V, W, H)
        self.calls = CdOracleEngine.log if CdOracleEngine.log is not None else []

    def cd_update(self, which, l1, l2):
        self.calls.append(("cd_update", which, l1, l2))
        X = self.W if which == 0 else self.H
        X.copy_(cdo.update(self.V, self.W, self.H, which, l1, l2))

    def cd_iterate(self, n_iter, l1, l2):
        self.calls.append(("cd_iterate", n_iter, l1, l2))
        for _ in range(n_iter):
            self.W.copy_(cdo.update(self.V, self.W, self.H, 0, l1, l2))
            self.H.copy_(cdo.update(self.V, self.W, self.H, 1, l1, l2))

    def update_w(self, *a):
        self.calls.append(("update_w",) + a)
        super().update_w(*a)

    def update_h(self, *a):
        self.calls.append(("update_h",) + a)
        super().update_h(*a)


def _problem(seed, N=23, C=17, R=4, dtype=torch.float64):
    g = torch.Generator().manual_seed(seed)
    V = torch.rand(N, R, generator=g, dtype=dtype) @ torch.rand(R, C, generator=g, dtype=dtype)
    V += 0.05 * torch.rand(N, C, generator=g, dtype=dtype)
    W, H = torch.rand(C, R, generator=g, dtype=dtype) + 0.1, torch.rand(N, R, generator=g, dtype=dtype) + 0.1
    return V, W.float().to(dtype), H.float().to(dtype)       # fp32 values: NMF(W=..., H=...) stores them exactly


def _oracle_loss(V, W, H):
    return float(orc.beta_div(orc.nmf_reconstruct(H, W), V, 2))


# ---- the oracle against the objective ----------------------------------------------------------------------------------

@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("alpha,l1_ratio", [(0.0, 0.0), (0.3, 0.0), (0.3, 1.0), (0.5, 0.4)])
def test_objective_never_rises_across_a_column_step(seed, alpha, l1_ratio):
    l1, l2 = alpha * l1_ratio, alpha * (1 - l1_ratio)
    V, W, H = _problem(seed, R=5)
    for _ in range(3):
        for which in (0, 1):
            fac = {"W": W, "H": H}
            prev = [cdo.objective(V, W, H, l1, l2)]

            def on_step(k, X):
                cur = cdo.objective(V, X if which == 0 else fac["W"], fac["H"] if which == 0 else X, l1, l2)
                assert cur <= prev[0] * (1 + 1e-13) + 1e-13, (which, k, prev[0], cur)
                prev[0] = cur

            new = cdo.update(V, W, H, which, l1, l2, on_step=on_step)
            if which == 0:
                W = new
            else:
                H = new


@pytest.mark.parametrize("seed", range(3))
@pytest.mark.parametrize("alpha,l1_ratio", [(0.0, 0.0), (0.2, 0.5)])
def test_kkt_conditions_hold_at_convergence(seed, alpha, l1_ratio):
    # x > 0  =>  |grad| <= tol;   x = 0  =>  grad >= -tol;   tol = 1e-7 x the largest numerator entry
    l1, l2 = alpha * l1_ratio, alpha * (1 - l1_ratio)
    V, W, H = _problem(seed, N=15, C=12, R=3)
    for _ in range(3000):
        W = cdo.update(V, W, H, 0, l1, l2)
        H = cdo.update(V, W, H, 1, l1, l2)
    for which, X in ((0, W), (1, H)):
        g = cdo.gradient(V, W, H, which, l1, l2)
        tol = 1e-7 * float(cdo.terms(V, W, H, which)[0].abs().max())
        pos = X > 0
        assert float(g[pos].abs().max()) <= tol
        if (~pos).any():
            assert float(g[~pos].min()) >= -tol


def test_dead_component_is_left_unchanged_without_nan():
    V, W, H = _problem(7, R=4)
    H[:, 2] = 0.0                                   # B[2,2] = (H^T H)[2,2] = 0 for the W update, and l2 = 0
    W2 = cdo.update(V, W, H, 0, 0.0, 0.0)
    assert torch.equal(W2[:, 2], W[:, 2])
    assert torch.isfinite(W2).all()
    # with l2 > 0 the column does move (B[2,2] + l2 != 0): towards 0 from the penalty alone
    W3 = cdo.update(V, W, H, 0, 0.0, 0.5)
    assert torch.isfinite(W3).all() and not torch.equal(W3[:, 2], W[:, 2])


# ---- fit(solver="cd") through the engine hook ---------------------------------------------------------------------------

def _module(W0, H0, trainable_W=True, trainable_H=True):
    m = NMF(W=W0, H=H0, trainable_W=trainable_W, trainable_H=trainable_H).double()
    m._engine_factory = CdOracleEngine
    return m


@pytest.mark.parametrize("tol,max_iter", [(1e-4, 200), (float("-inf"), 25), (1e-2, 200)])
@pytest.mark.parametrize("alpha,l1_ratio", [(0, 0), (0.1, 0.0), (0.1, 1.0), (0.2, 0.25)])
def test_fit_equals_a_direct_oracle_loop(tol, max_iter, alpha, l1_ratio):
    V, W0, H0 = _problem(11)
    m = _module(W0, H0)
    n = m.fit(V, 2, tol, max_iter, False, alpha, l1_ratio, solver="cd")
    W, H, n_ref, _ = cdo.fit(V, W0, H0, tol, max_iter, alpha * l1_ratio, alpha * (1 - l1_ratio), loss=_oracle_loss)
    assert n == n_ref
    assert torch.equal(m.W.data, W) and torch.equal(m.H.data, H)


@pytest.mark.parametrize("frozen", ["W", "H"])
def test_fit_with_a_frozen_factor(frozen):
    V, W0, H0 = _problem(12)
    CdOracleEngine.log = log = []
    try:
        m = _module(W0, H0, trainable_W=frozen != "W", trainable_H=frozen != "H")
        n = m.fit(V, 2, 1e-5, 60, alpha=0.1, l1_ratio=0.5, solver="cd")
    finally:
        CdOracleEngine.log = None
    W, H, n_ref, _ = cdo.fit(V, W0, H0, 1e-5, 60, 0.05, 0.05, train_w=frozen != "W", train_h=frozen != "H",
                             loss=_oracle_loss)
    assert n == n_ref
    assert torch.equal(m.W.data, W) and torch.equal(m.H.data, H)
    assert torch.equal((m.W if frozen == "W" else m.H).data, W0 if frozen == "W" else H0)
    assert {c[:2] for c in log} == {("cd_update", 1 if frozen == "W" else 0)}
    assert all(c[2:] == (0.05, 0.05) for c in log)


def test_fit_runs_the_iterations_between_checks_in_one_call():
    V, W0, H0 = _problem(13)
    CdOracleEngine.log = log = []
    try:
        _module(W0, H0).fit(V, 2, float("-inf"), 25, alpha=0.4, l1_ratio=0.25, solver="cd")
    finally:
        CdOracleEngine.log = None
    assert log == [("cd_iterate", 10, 0.1, pytest.approx(0.3)), ("cd_iterate", 10, 0.1, pytest.approx(0.3)),
                   ("cd_iterate", 5, 0.1, pytest.approx(0.3))]


def test_solver_mu_is_the_default_call():
    V, W0, H0 = _problem(14)
    runs = []
    for kw in ({}, {"solver": "mu"}):
        CdOracleEngine.log = log = []
        try:
            m = _module(W0, H0, trainable_W=False)
            n = m.fit(V, 2, 1e-4, 40, **kw)
        finally:
            CdOracleEngine.log = None
        runs.append((n, m.W.data.clone(), m.H.data.clone(), log))
    assert runs[0][0] == runs[1][0] and runs[0][3] == runs[1][3]
    assert torch.equal(runs[0][1], runs[1][1]) and torch.equal(runs[0][2], runs[1][2])
    assert all(c[0] == "update_h" for c in runs[0][3])


def _no_engine(*a, **k):
    raise AssertionError("an engine was built before the refusal")


@pytest.mark.parametrize("case", ["beta1", "beta0.5", "mask", "weight", "group", "f16", "f16_split", "rank", "solver",
                                  "nmfd", "nmf2d", "nmf3d"])
def test_refusals_raise_before_any_engine(case):
    V, W0, H0 = _problem(15)
    m = NMF(W=W0, H=H0).double()
    kw, beta = {"solver": "cd"}, 2
    if case == "beta1":
        beta = 1
    elif case == "beta0.5":
        beta = 0.5
    elif case == "mask":
        kw["mask"] = torch.ones(V.shape, dtype=torch.bool)
    elif case == "weight":
        kw["weight"] = torch.ones(V.shape, dtype=torch.float64)
    elif case == "group":
        kw["group"] = object()
    elif case in ("f16", "f16_split"):
        kw["precision"] = case
    elif case == "rank":
        m = NMF(W=torch.rand(V.shape[1], 257), H=torch.rand(V.shape[0], 257))
    elif case == "solver":
        kw["solver"] = "hals"
    elif case == "nmfd":
        m, V = NMFD(W=torch.rand(5, 3, 4), H=torch.rand(2, 3, 7)), torch.rand(2, 5, 10)
    elif case == "nmf2d":
        m, V = NMF2D(W=torch.rand(5, 3, 2, 4), H=torch.rand(1, 3, 5, 7)), torch.rand(1, 5, 6, 10)
    elif case == "nmf3d":
        m, V = NMF3D(W=torch.rand(5, 3, 2, 2, 4), H=torch.rand(1, 3, 3, 5, 7)), torch.rand(1, 5, 4, 6, 10)
    m._engine_factory = _no_engine
    with pytest.raises(ValueError):
        m.fit(V, beta, **kw)


def test_cd_entry_points_are_bound_and_refuse_a_null_context():
    from torchnmf_b200 import _capi
    _vp, _dbl, _int = ctypes.c_void_p, ctypes.c_double, ctypes.c_int
    assert _capi.SIGNATURES["nmfb200_nmf_cd_update"] == (_int, [_vp, _vp, _vp, _int, _dbl, _dbl, _vp])
    assert _capi.SIGNATURES["nmfb200_nmf_cd_iterate"] == (_int, [_vp, _vp, _vp, _dbl, _dbl, _int, _vp])
    lib = _capi.load()
    assert lib.nmfb200_nmf_cd_update(None, None, None, 0, 0.0, 0.0, None) == 1            # NMFB200_ERR_INVALID
    assert b"null context" in lib.nmfb200_last_error()
    assert lib.nmfb200_nmf_cd_iterate(None, None, None, 0.0, 0.0, 1, None) == 1
    header = open(os.path.join(ROOT, "include", "nmf_b200.h")).read()
    assert ("int nmfb200_nmf_cd_update(nmfb200_ctx* ctx, float* W, float* H, int which, double l1_reg, double l2_reg, "
            "void* stream);") in header
    assert lib.nmfb200_abi_version() == 2
