"""Ranks above 256 on the CPU: the planner accepts them and keeps every rank <= 256 plan as it was, the cases of
tests/test_gpu_high_rank.py reach every new branch (asked of the library's planner, no device needed), the float64
oracle matches the reference fixtures of tests/golden/reference_high_rank.npz, and the sparse-target and convolutive
plans keep their rank cap.
"""
import math

import numpy as np
import pytest
import torch

import f32_cases as fc
import high_rank_cases as hc
from conftest import GOLDEN
from oracle import mu_oracle as orc
from oracle import plca_oracle as porc
from torchnmf_b200 import PLCA, _capi


@pytest.mark.parametrize("R", [257, 272, 300, 511, 512, 513, 1000, 1024])
def test_nmf_plan_accepts_ranks_above_256(R):
    p = _capi.nmf_plan(400, 700, R)
    assert p["rb"] == 16
    # the rank blocks are counted in the chunk planning: a multiple of the blocks' CTAs does not grow the partial slabs
    nb = hc.rank_blocks(R)
    for nch, rows, cols in ((p["nch_w"], 700, 400), (p["nch_h"], 400, 700)):
        assert nch == max(1, min(hc.cdiv(528, hc.cdiv(rows, 64) * nb), hc.cdiv(cols, 64), 32))


@pytest.mark.parametrize("case", fc.NMF_EXACT, ids=str)
def test_nmf_plan_unchanged_up_to_rank_256(case):
    assert _capi.nmf_plan(*case) == hc.parent_plan(*case)


def high_branches(cases):
    hit = set()
    for N, C, R in cases:
        p = _capi.nmf_plan(N, C, R)
        nb = hc.rank_blocks(R)
        hit.add("one rank block" if nb == 1 else "several rank blocks")
        if nb > 2:
            hit.add("more than two rank blocks")
        if nb > 1 and R % 256:
            hit.add("short last rank block")
        if nb > 1 and R % 256 == 0:
            hit.add("full last rank block")
        if R % 16:
            hit.add("R%16!=0")
        for side, rows, cols, nch in (("W", C, N, p["nch_w"]), ("H", N, C, p["nch_h"])):
            if nb > 1:
                hit.add(f"{'one chunk' if nch == 1 else 'several chunks'} ({side} update)")
            hit.add(f"rows%64={rows % 64}" if rows % 64 in (0, 1, 63) else "rows other")
            hit.add(f"cols%64={cols % 64}" if cols % 64 in (0, 1, 63) else "cols other")
    return hit


HIGH_REQUIRED = ({"one rank block", "several rank blocks", "more than two rank blocks", "short last rank block",
                  "full last rank block", "R%16!=0"}
                 | {f"{k} ({s} update)" for k in ("one chunk", "several chunks") for s in "WH"}
                 | {f"rows%64={r}" for r in (0, 1, 63)} | {f"cols%64={r}" for r in (0, 1, 63)})


def test_high_rank_cases_cover_every_branch():
    miss = sorted(HIGH_REQUIRED - high_branches(hc.HIGH_EXACT))
    assert not miss, miss
    assert {257, 300, 512, 513, 1000} <= {R for _, _, R in hc.HIGH_EXACT}
    assert {"several chunks (W update)", "several chunks (H update)"} <= high_branches(hc.HIGH_CHUNKED)
    assert all(c in hc.HIGH_EXACT for c in hc.HIGH_RATIO)
    cut = [c for c in hc.HIGH_EXACT if c[2] % 256 == 0]
    assert {"short last rank block", "R%16!=0"} <= HIGH_REQUIRED - high_branches(cut)


@pytest.mark.parametrize("case", hc.HIGH_EXACT, ids=str)
def test_high_rank_exact_bounds(case):
    N, C, R = case
    f = fc.nmf_range(N, C, R)
    assert fc.nmf_bound(N, C, R, f, f * f) < fc.EXACT and fc.nmf_kl_bound(N, C, R) < fc.EXACT
    f = fc.nmf_range(N, C, R, loss=True)
    assert fc.loss_bound(R * f * f, f * f) < fc.EXACT_LOSS


def test_sparse_and_convolutive_plans_cap_the_rank():
    with pytest.raises(_capi.NmfB200Error, match="256"):
        _capi.sparse_plan(5, 6, 257)
    with pytest.raises(_capi.NmfB200Error, match="256"):
        _capi.nmfd_plan(1, 4, [100], 257, [4])
    with pytest.raises(_capi.NmfB200Error, match="256"):
        _capi.nmfd_plan(1, 3, [7, 70], 257, [3, 8])
    with pytest.raises(_capi.NmfB200Error, match="256"):
        _capi.nmfnd_tc_plan(1, 4, [100], 257, [4])
    _capi.nmfd_plan(1, 4, [100], 256, [4])


def load_high_rank():
    z = np.load(f"{GOLDEN}/reference_high_rank.npz", allow_pickle=False)
    cases = {}
    for key in z.files:
        name, field = key.split("/", 1)
        cases.setdefault(name, {})[field] = z[key]
    return cases


CASES = load_high_rank()


def inputs(c):
    """oracle/make_golden.py's recipe, regenerated from the seeds and checked against the stored sums."""
    N, C, R = int(c["N"]), int(c["C"]), int(c["R"])
    torch.manual_seed(0)
    V = torch.rand(N, C).bfloat16().float()
    torch.manual_seed(1)
    W0, H0 = torch.randn(C, R).abs(), torch.randn(N, R).abs()
    for t, k in ((V, "v_sum"), (W0, "w0_sum"), (H0, "h0_sum")):
        assert abs(float(t.double().sum()) - float(c[k])) <= 1e-12 * abs(float(c[k])), k
    return V, W0, H0


def plca_inputs(c):
    N, C, R = int(c["N"]), int(c["C"]), int(c["R"])
    torch.manual_seed(0)
    V = torch.rand(N, C).bfloat16().float() * 3
    torch.manual_seed(1)
    W0, H0, Z0 = torch.randn(C, R).abs(), torch.randn(N, R).abs(), torch.rand(R) + 0.1
    for t, k in ((V, "v_sum"), (W0, "w0_sum"), (H0, "h0_sum"), (Z0, "z0_sum")):
        assert abs(float(t.double().sum()) - float(c[k])) <= 1e-12 * abs(float(c[k])), k
    return V, W0, H0, Z0


NMF_NAMES = sorted(n for n in CASES if n.startswith("nmf_"))


def sample(x, c, key):
    """The fixture's sample of factor x ("w" or "h"): every `step`-th entry of the flattened factor."""
    return x.reshape(-1)[::int(c[f"{key}_step"])]


def test_fixture_samples_reach_every_component():
    for name, c in CASES.items():
        for key, rows in (("w", int(c["C"])), ("h", int(c["N"]))):
            R, step, n = int(c["R"]), int(c[f"{key}_step"]), c[f"{key.upper()}_sub"].size
            assert n == -(-(rows * R) // step) and n <= 8000, (name, key)
            # a stride coprime with R meets every component once in any R consecutive samples: each at least 4 times
            assert math.gcd(step, R) == 1 and n >= 4 * R, (name, key)


def test_fixtures_hold_the_issue_cases():
    assert {int(CASES[n]["R"]) for n in NMF_NAMES} == {300, 512, 600}
    assert {float(CASES[n]["beta"]) for n in NMF_NAMES if int(CASES[n]["R"]) == 300} == {0.5, 1.0, 2.0}
    assert int(CASES["nmf_default_rank"]["default_rank"]) == 1 and int(CASES["plca_r300"]["R"]) == 300


@pytest.mark.parametrize("name", NMF_NAMES)
def test_oracle_matches_high_rank_fixture(name):
    c = CASES[name]
    V, W0, H0 = inputs(c)
    W, H, n_iter, losses = orc.fit(V, W0, H0, beta=float(c["beta"]), tol=float("-inf"), max_iter=int(c["max_iter"]),
                                   alpha=float(c["alpha"]), l1_ratio=float(c["l1_ratio"]))
    assert n_iter == int(c["n_iter"])
    assert torch.allclose(sample(W, c, "w"), torch.from_numpy(c["W_sub"]), rtol=2e-4, atol=1e-6 * float(c["w_absmax"]))
    assert torch.allclose(sample(H, c, "h"), torch.from_numpy(c["H_sub"]), rtol=2e-4, atol=1e-6 * float(c["h_absmax"]))
    assert np.allclose(losses, c["losses"], rtol=1e-5)


def test_plca_oracle_matches_high_rank_fixture():
    c = CASES["plca_r300"]
    V, W0, H0, Z0 = plca_inputs(c)
    mod = PLCA(W=W0, H=H0, Z=Z0)                                  # the constructor normalises (plca.py:110-144)
    W, H, Z, n_iter, norm = porc.fit(V, mod.W.data, mod.H.data, mod.Z.data, tol=float("-inf"), max_iter=int(c["max_iter"]))
    assert n_iter == int(c["n_iter"])
    assert torch.allclose(sample(W, c, "w"), torch.from_numpy(c["W_sub"]), rtol=2e-4, atol=1e-6 * float(c["w_absmax"]))
    assert torch.allclose(sample(H, c, "h"), torch.from_numpy(c["H_sub"]), rtol=2e-4, atol=1e-6 * float(c["h_absmax"]))
    assert torch.allclose(Z, torch.from_numpy(c["Z"]), rtol=2e-4, atol=1e-7)
