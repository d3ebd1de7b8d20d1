"""Coordinate descent at beta 2 on the observed cells (`NMF.fit(V, beta=2, solver="cd", mask=M)` with a sparse mask or
weight), without a GPU.

The float64 oracle (tests/observed_cd_oracle.py) is checked against the objective it descends -- never rising across a
column step, the KKT conditions at convergence, the dense HALS update when every cell is observed, empty segments and dead
components left alone -- and then the host logic of `fit` (validation, the observed set the engine receives, the loop, the
stop rule, frozen factors) runs through the oracle's engine plugged in with the `_engine_factory` hook.
"""
import ctypes
import math
import os

import pytest
import torch

import cd_oracle as cdo
import observed_cd_oracle as ocd
from observed_cd_oracle import ObservedCdOracleEngine
from torchnmf_b200 import NMF, NMFD

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _problem(seed, N=23, C=17, R=4, density=0.4, weighted=False):
    """(V dense float64, M float64 weights (0: not observed), W0, H0 fp32-exact float64)."""
    g = torch.Generator().manual_seed(seed)
    V = torch.rand(N, R, generator=g, dtype=torch.float64) @ torch.rand(R, C, generator=g, dtype=torch.float64)
    V += 0.05 * torch.rand(N, C, generator=g, dtype=torch.float64)
    M = (torch.rand(N, C, generator=g) < density).double()
    if weighted:
        M = (M * (0.25 + 2 * torch.rand(N, C, generator=g))).double()       # fp32 weights, as the fit passes them
    W = (torch.rand(C, R, generator=g) + 0.1).double()
    H = (torch.rand(N, R, generator=g) + 0.1).double()
    return V.float().double(), M, W, H


# ---- the oracle against the objective ----------------------------------------------------------------------------------

@pytest.mark.parametrize("seed", range(3))
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("alpha,l1_ratio", [(0.0, 0.0), (0.3, 0.0), (0.3, 1.0), (0.5, 0.4)])
def test_objective_never_rises_across_a_column_step(seed, weighted, alpha, l1_ratio):
    l1, l2 = alpha * l1_ratio, alpha * (1 - l1_ratio)
    V, M, W, H = _problem(seed, R=5, weighted=weighted)
    for _ in range(3):
        for which in (0, 1):
            prev = [ocd.objective(V, M, W, H, l1, l2)]

            def on_step(k, X):
                cur = ocd.objective(V, M, X if which == 0 else W, H if which == 0 else X, l1, l2)
                assert cur <= prev[0] * (1 + 1e-13) + 1e-13, (which, k, prev[0], cur)
                prev[0] = cur

            new = ocd.update(V, M, W, H, which, l1, l2, on_step=on_step)
            if which == 0:
                W = new
            else:
                H = new


@pytest.mark.parametrize("seed", range(2))
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("alpha,l1_ratio", [(0.0, 0.0), (0.2, 0.5)])
def test_kkt_conditions_hold_at_convergence(seed, weighted, alpha, l1_ratio):
    # x > 0  =>  |grad| <= tol;   x = 0  =>  grad >= -tol;   tol = 1e-7 x the largest |M V| F entry
    l1, l2 = alpha * l1_ratio, alpha * (1 - l1_ratio)
    V, M, W, H = _problem(seed, N=15, C=12, R=2, density=0.9, weighted=weighted)
    for _ in range(3000):
        W = ocd.update(V, M, W, H, 0, l1, l2)
        H = ocd.update(V, M, W, H, 1, l1, l2)
    for which, X in ((0, W), (1, H)):
        g = ocd.gradient(V, M, W, H, which, l1, l2)
        scale = float(((M * V).t() @ H).abs().max()) if which == 0 else float(((M * V) @ W).abs().max())
        tol = 1e-7 * scale
        pos = X > 0
        assert float(g[pos].abs().max()) <= tol
        if (~pos).any():
            assert float(g[~pos].min()) >= -tol


@pytest.mark.parametrize("seed", range(3))
@pytest.mark.parametrize("which", [0, 1])
@pytest.mark.parametrize("l1,l2", [(0.0, 0.0), (0.1, 0.3)])
def test_all_cells_observed_equals_the_dense_update(seed, which, l1, l2):
    V, M, W, H = _problem(seed, R=6)
    M = torch.ones_like(M)
    got = ocd.update(V, M, W, H, which, l1, l2)
    want = cdo.update(V, W, H, which, l1, l2)
    assert (got - want).abs().max() <= 1e-12 * float(want.abs().max())


def test_empty_segments_and_dead_components_stay_unchanged():
    V, M, W, H = _problem(5, R=4)
    M[3] = 0.0                                  # row 3 of V: no observed cell -> H[3] keeps its value (l2 = 0)
    M[:, 7] = 0.0                               # column 7: W[7] keeps its value
    H[:, 2] = 0.0                               # component 2 of H is dead: hess = 0 for W's column 2 on every segment
    for l1 in (0.0, 0.4):
        W2 = ocd.update(V, M, W, H, 0, l1, 0.0)
        H2 = ocd.update(V, M, W2, H, 1, l1, 0.0)
        assert torch.isfinite(W2).all() and torch.isfinite(H2).all()
        assert torch.equal(W2[7], W[7]) and torch.equal(H2[3], H[3])
        assert torch.equal(W2[:, 2], W[:, 2])
        assert not torch.equal(W2, W) and not torch.equal(H2, H)


# ---- fit(solver="cd") with a sparse mask or weight, through the engine hook ---------------------------------------------

def _module(W0, H0, trainable_W=True, trainable_H=True):
    m = NMF(W=W0, H=H0, trainable_W=trainable_W, trainable_H=trainable_H).double()
    m._engine_factory = ObservedCdOracleEngine
    return m


def _selector(M, weighted):
    """The sparse mask (M > 0) or the sparse weight (M's values) of the observed set."""
    return {"weight": M.to_sparse()} if weighted else {"mask": (M > 0).to_sparse()}


@pytest.fixture
def log():
    ObservedCdOracleEngine.calls = calls = []
    ObservedCdOracleEngine.received = []
    yield calls
    ObservedCdOracleEngine.calls = []
    ObservedCdOracleEngine.received = []


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("tol,max_iter", [(1e-4, 200), (float("-inf"), 25), (1e-2, 200)])
@pytest.mark.parametrize("alpha,l1_ratio", [(0, 0), (0.1, 1.0), (0.2, 0.25)])
def test_fit_equals_a_direct_oracle_loop(log, weighted, tol, max_iter, alpha, l1_ratio):
    V, M, W0, H0 = _problem(11, weighted=weighted)
    m = _module(W0, H0)
    n = m.fit(V, 2, tol, max_iter, False, alpha, l1_ratio, solver="cd", **_selector(M, weighted))
    W, H, n_ref, checks = ocd.fit(V, M, W0, H0, tol, max_iter, alpha * l1_ratio, alpha * (1 - l1_ratio))
    assert n == n_ref
    assert torch.equal(m.W.data, W) and torch.equal(m.H.data, H)
    losses = [math.sqrt(2.0 * c[1]) for c in log if c[0] == "loss"]
    assert losses[1:] == checks
    assert m.last_fit_precision == "f32"


@pytest.mark.parametrize("weighted", [False, True])
def test_iterations_between_checks_run_in_one_call(log, weighted):
    V, M, W0, H0 = _problem(13, weighted=weighted)
    _module(W0, H0).fit(V, 2, float("-inf"), 25, alpha=0.4, l1_ratio=0.25, solver="cd", **_selector(M, weighted))
    assert [c for c in log if c[0] != "loss"] == [("cd_iterate", 10, 0.1, pytest.approx(0.3)),
                                                  ("cd_iterate", 10, 0.1, pytest.approx(0.3)),
                                                  ("cd_iterate", 5, 0.1, pytest.approx(0.3))]


@pytest.mark.parametrize("frozen", ["W", "H"])
def test_a_frozen_factor_takes_per_factor_updates_and_stays_bit_identical(log, frozen):
    V, M, W0, H0 = _problem(12)
    m = _module(W0, H0, trainable_W=frozen != "W", trainable_H=frozen != "H")
    n = m.fit(V, 2, 1e-5, 60, alpha=0.1, l1_ratio=0.5, solver="cd", mask=(M > 0).to_sparse())
    W, H, n_ref, _ = ocd.fit(V, M, W0, H0, 1e-5, 60, 0.05, 0.05, train_w=frozen != "W", train_h=frozen != "H")
    assert n == n_ref
    assert torch.equal(m.W.data, W) and torch.equal(m.H.data, H)
    assert torch.equal((m.W if frozen == "W" else m.H).data, W0 if frozen == "W" else H0)
    updates = [c for c in log if c[0] != "loss"]
    assert updates and {c[:2] for c in updates} == {("cd_update", 1 if frozen == "W" else 0)}
    assert all(c[2:] == (0.05, 0.05) for c in updates)


def test_weights_in_0_1_give_the_mask_fit(log):
    V, M, W0, H0 = _problem(14)
    runs = []
    every_cell = torch.sparse_coo_tensor(torch.ones_like(M).nonzero().t(), M.flatten(), M.shape)     # stored zeros too
    for sel in ({"mask": (M > 0).to_sparse()}, {"weight": M.to_sparse()}, {"weight": every_cell}):
        ObservedCdOracleEngine.received = []
        m = _module(W0, H0)
        n = m.fit(V, 2, 1e-4, 80, solver="cd", **sel)
        O, wts = ObservedCdOracleEngine.received[0]
        runs.append((n, m.W.data.clone(), m.H.data.clone(), O))
        assert wts is None or torch.equal(wts, torch.ones_like(wts))
    for n, W, H, O in runs[1:]:
        assert n == runs[0][0] and torch.equal(W, runs[0][1]) and torch.equal(H, runs[0][2])
        assert torch.equal(O.indices(), runs[0][3].indices()) and torch.equal(O.values(), runs[0][3].values())


def test_sparse_and_dense_targets_of_one_observed_set_reach_the_engine_identically(log):
    V, M, W0, H0 = _problem(15)
    Mb = M > 0
    Vs = (V * (torch.rand(V.shape, generator=torch.Generator().manual_seed(1)) < 0.8)).float()   # zeros, some observed
    fills = Vs.masked_fill(~Mb, float("nan"))                                                  # dense: NaN off the mask
    wide = torch.full((V.shape[0], V.shape[1] + 5), float("nan"))
    wide[:, :V.shape[1]] = Vs
    strided = wide[:, :V.shape[1]]
    assert not strided.is_contiguous()
    outs = []
    for target in (Vs.to_sparse(), fills, Vs.double(), strided):
        ObservedCdOracleEngine.received = []
        m = _module(W0, H0)
        n = m.fit(target, 2, 1e-4, 40, solver="cd", mask=Mb.to_sparse())
        outs.append((n, m.W.data.clone(), m.H.data.clone(), ObservedCdOracleEngine.received[0][0]))
    for n, W, H, O in outs[1:]:
        assert torch.equal(O.indices(), outs[0][3].indices()) and torch.equal(O.values(), outs[0][3].values())
        assert n == outs[0][0] and torch.equal(W, outs[0][1]) and torch.equal(H, outs[0][2])


def _no_engine(*a, **k):
    raise AssertionError("an engine was built before the refusal")


@pytest.mark.parametrize("case", ["dense_mask", "dense_weight", "nmfd_sparse_mask", "group", "beta1", "beta0.5", "f16",
                                  "f16_split", "rank"])
def test_refusals_raise_before_any_engine(case):
    V, M, W0, H0 = _problem(16)
    m = NMF(W=W0, H=H0).double()
    kw, beta = {"solver": "cd", "mask": (M > 0).to_sparse()}, 2
    if case == "dense_mask":
        kw["mask"] = M > 0
    elif case == "dense_weight":
        del kw["mask"]
        kw["weight"] = M
    elif case == "nmfd_sparse_mask":
        m, V = NMFD(W=torch.rand(5, 3, 4), H=torch.rand(2, 3, 7)), torch.rand(2, 5, 10)
        kw["mask"] = (torch.rand(2, 5, 10) < 0.5).to_sparse()
    elif case == "group":
        kw["group"] = object()
    elif case == "beta1":
        beta = 1
    elif case == "beta0.5":
        beta = 0.5
    elif case in ("f16", "f16_split"):
        kw["precision"] = case
    elif case == "rank":
        m = NMF(W=torch.rand(V.shape[1], 257), H=torch.rand(V.shape[0], 257))
    m._engine_factory = _no_engine
    with pytest.raises(ValueError) as e:
        m.fit(V, beta, **kw)
    if case.startswith("dense"):
        assert ".to_sparse()" in str(e.value)


def test_observed_cd_entry_points_are_bound_declared_and_refuse_a_null_context():
    from torchnmf_b200 import _capi
    _vp, _dbl, _int = ctypes.c_void_p, ctypes.c_double, ctypes.c_int
    assert _capi.SIGNATURES["nmfb200_nmf_observed_cd_update"] == (_int, [_vp, _vp, _vp, _int, _dbl, _dbl, _vp])
    assert _capi.SIGNATURES["nmfb200_nmf_observed_cd_iterate"] == (_int, [_vp, _vp, _vp, _dbl, _dbl, _int, _vp])
    lib = _capi.load()
    assert lib.nmfb200_nmf_observed_cd_update(None, None, None, 0, 0.0, 0.0, None) == 1        # NMFB200_ERR_INVALID
    assert b"null context" in lib.nmfb200_last_error()
    assert lib.nmfb200_nmf_observed_cd_iterate(None, None, None, 0.0, 0.0, 1, None) == 1
    assert b"null context" in lib.nmfb200_last_error()
    header = " ".join(open(os.path.join(ROOT, "include", "nmf_b200.h")).read().split())
    assert ("int nmfb200_nmf_observed_cd_update(nmfb200_ctx* ctx, float* W, float* H, int which, double l1_reg, "
            "double l2_reg, void* stream);") in header
    assert ("int nmfb200_nmf_observed_cd_iterate(nmfb200_ctx* ctx, float* W, float* H, double l1_reg, double l2_reg, "
            "int n_iter, void* stream);") in header
    assert lib.nmfb200_abi_version() == 2
