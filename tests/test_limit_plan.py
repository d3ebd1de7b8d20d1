"""Host checks of the limit cases (tests/limit_cases.py) and of the launch plans at the CUDA grid limits; no GPU.

  * Every big case really crosses element 2^31 where it says, and every grid case sits where it says.
  * The plan queries (nmfb200_nmfd_plan, nmfb200_nmfnd_tc_plan) either reject a shape or report grids with x <= 2^31 - 1 and
    y, z <= 65535, and counts the library holds in 32 bits that fit, for every case and a sweep around each bound.
  * The float64 references taken in blocks (as the GPU tests take them) equal the one-block references, on scaled-down
    copies of the big cases with the same structure, and the GPU tests check every row, the crossing rows included.
  * The bars are not vacuous: the target as a 31-bit-masked index reads it moves at least one checked entry past its bar.
  * The exact cases are exact by their bound.
"""
import pytest
import torch

import f32_cases as fc
import limit_cases as lc
from oracle import mu_oracle as orc
from torchnmf_b200 import _capi

SCALE = 2 ** 14          # big cases scaled down by this factor keep their structure


def _fits(grid):
    x, y, z = grid
    return 1 <= x <= lc.GRID_X and 1 <= y <= lc.GRID_YZ and 1 <= z <= lc.GRID_YZ


def _nmfd_plan_ok(B, C, L, R, T):
    """None if the fp32 plan query rejects the shape, else asserts its grids fit and returns the plan."""
    try:
        p = _capi.nmfd_plan(B, C, [L], R, [T])
    except _capi.NmfB200Error:
        return None
    for k in ("recon_grid", "dgrad_grid"):
        assert _fits(p[k]), (B, C, L, R, T, k, p[k])
    w = p["wgrad"]
    assert _fits((w["ntt"] * w["nrg"] * w["nog"], lc.cdiv(C, w["mt"]), p["wgrad_nsplit"]))
    # every batch element is covered by the launches of one grid.z each
    assert p["recon_grid"][2] == min(B, lc.GRID_YZ) and p["dgrad_grid"][2] == min(B, lc.GRID_YZ)
    return p


def _tc_plan_ok(B, C, L, R, T):
    try:
        p = _capi.nmfnd_tc_plan(B, C, [L], R, [T])
    except _capi.NmfB200Error as e:
        return None, str(e)
    for k in ("prep_w", "prep_h", "recon", "wgrad", "dgrad"):
        assert _fits(p[k]), (B, C, L, R, T, k, p[k])
    assert p["bslice"] * (p["slices"] - 1) < B <= p["bslice"] * p["slices"]
    assert p["recon"][2] == p["dgrad"][2] == p["bslice"]
    assert p["prep_h"][0] == B * R * lc.cdiv(L - T + 1, 2048)
    assert p["loss_blocks"] == p["recon"][0] * p["recon"][1] * B <= lc.INT_MAX
    assert B * C + 128 <= lc.INT_MAX                              # the ratio tile's TMA row coordinate
    assert B * lc.cdiv(L, 64) <= lc.INT_MAX and C * lc.cdiv(T, 64) <= lc.INT_MAX   # global k-block indices
    assert p["ws_w"] * p["kbs_w"] >= B * lc.cdiv(L, 64) and p["ws_h"] * p["kbs_h"] >= C * lc.cdiv(T, 64)
    return p, ""


# ---- the cases cross what they name --------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(lc.NMF_BIG))
def test_nmf_big_case_crosses_2p31(name):
    case = lc.NMF_BIG[name]
    N, C, R = case["N"], case["C"], case["R"]
    cross = lc.nmf_crossings(case)
    assert cross, name
    for buf, (fac, row) in cross.items():
        n = N if fac == "H" else C
        assert 0 < row < n, (buf, fac, row)
    if "V" in cross:
        fac, row = cross["V"]
        if fac == "H":
            assert (row - 1) * C < lc.ELEM <= row * C + C - 1
        else:
            assert (N - 1) * C + row >= lc.ELEM > (N - 1) * C + row - 1
    if "H" in cross:
        assert N * R > lc.ELEM and cross["H"][1] * R <= lc.ELEM < (cross["H"][1] + 1) * R
    if "f16" in case["runs"]:
        assert N <= lc.NMF_TC_N and "Vt16" in cross
    else:
        assert N > lc.NMF_TC_N


@pytest.mark.parametrize("name", list(lc.NMFD_BIG))
def test_nmfd_big_case_crosses_2p31_in_both_plans(name):
    case = lc.NMFD_BIG[name]
    B, C, L, R, T = lc.nmfd_dims(case)
    assert B >= 2 and C == 1025 and (R, T) == (16, 16) and B * C * L > lc.ELEM
    cross = lc.nmfd_crossings(case)
    assert set(cross) == {"V", "Pn", "P16"}
    assert cross["V"] * L <= lc.ELEM < (cross["V"] + 1) * L and cross["V"] < B * C
    p, why = _tc_plan_ok(B, C, L, R, T)
    assert p is not None, why
    assert cross["P16"] < B * C


def test_grid_cases_sit_on_their_bounds():
    by = {c[0]: c for c in lc.GRID_CASES}
    assert by["nmf_tc_n_limit"][2][0] == 65535 * 64 == by["nmf_tc_n_over_f16"][2][0] - 1
    assert by["nmfd_b65535_f32"][2][0] == 65535 and by["nmfd_b65536_f32"][2][0] == 65536
    assert by["nmfd_b65535_f16"][2][0] == 65535 and by["nmfd_b65536_f16"][2][0] == 65536
    for name, br in (("nmfd_br65535_f16", 65535), ("nmfd_br65536_f16", 65536)):
        B, C, L, R, T = by[name][2]
        assert B * R == br
    assert by["nmfd_c_limit_f32"][2][1] == 65535 * 64 == by["nmfd_c_over_f32"][2][1] - 1
    for name, rt in (("nmfd_rt65535_f16", 65535), ("nmfd_rt65536_f16", 65536)):
        B, C, L, R, T = by[name][2]
        assert R * lc.cdiv(T, 128) == rt and L >= T


# ---- plan queries --------------------------------------------------------------------------------------------------------
def _sweep():
    shapes = [c[2] for c in lc.GRID_CASES if c[1] == "nmfd"] + [c[1] for c in lc.REJECT_CASES]
    shapes += [lc.nmfd_dims(c) for c in lc.NMFD_BIG.values()]
    for d in (-2, -1, 0, 1, 2):
        shapes += [(65535 + d, 3, 7, 4, 3), (2 * 65535 + d, 2, 5, 2, 2)]                     # batch slices
        shapes += [(1, 65535 * 64 + d, 3, 2, 2), (2, 65535 * 128 + d, 3, 1, 1)]            # recon grid.y
        shapes += [(256 + d, 1, 4, 256, 1), (1025 + d, 1, 3, 64, 1), (65535 + d, 1, 3, 1, 1)]   # B R
        shapes += [(1, 1, 32896 + d, 255, 32896), (1, 1, 32768 + d, 256, 32768 + d)]          # R ceil(T / 128)
        shapes += [(1, 1, 65535 * 2048 + d, 1, 1)]                                           # prep_h chunks
        shapes += [(2 ** 31 + d, 1, 1, 1, 1), (2 ** 20 + d, 2048, 1, 1, 1), (1, 2 ** 31 + d, 1, 1, 1)]   # narrowing
        shapes += [(2 ** 24 + d, 1, 2 ** 16, 1, 1)]                                          # loss partials
    shapes += PREP_H_X
    return [s for s in shapes if min(s) >= 1 and s[2] >= s[4]]


# prep_h's one-dimensional grid at its own limit: B R ceil(Lin / 2048) = 2^31 - 2^17 (the largest below 2^31 these factors
# form: 2^31 - 1 is prime, and no accepted shape has a factor of it), 2^31 and 2^32.  Every other bound holds at these shapes.
PREP_H_X = [(512, 1, 2 ** 25 - 2048, 256, 1), (512, 1, 2 ** 25, 256, 1), (1024, 1, 2 ** 25, 256, 1)]


def test_tc_prep_h_grid_at_its_limit():
    (ok, why), (over, why_over), (over2, _) = (_tc_plan_ok(*s) for s in PREP_H_X)
    assert ok is not None, why
    assert ok["prep_h"][0] == 2 ** 31 - 2 ** 17
    assert over is None and over2 is None and "grid" in why_over
    for B, C, L, R, T in PREP_H_X:
        assert _nmfd_plan_ok(B, C, L, R, T) is not None            # the fp32 kernels take them: only prep_h rejects


def test_plan_queries_report_launchable_grids_or_refuse():
    fp32_rejected = tc_rejected = 0
    for B, C, L, R, T in _sweep():
        p = _nmfd_plan_ok(B, C, L, R, T)
        fp32_rejected += p is None
        if p is not None:
            assert B <= lc.INT_MAX and C <= 65535 * 64
        tp, why = _tc_plan_ok(B, C, L, R, T)
        tc_rejected += tp is None
        if p is None:
            assert tp is None                                        # one validation for both paths
    assert fp32_rejected and tc_rejected


def test_plan_queries_name_their_limit():
    msg = {}
    for name, shape, prec, words in lc.REJECT_CASES:
        try:
            B, C, L, R, T = shape
            (_capi.nmfnd_tc_plan if prec == "f16" else _capi.nmfd_plan)(B, C, [L], R, [T])
        except _capi.NmfB200Error as e:
            msg[name] = str(e)
        assert words in msg.get(name, ""), (name, msg.get(name))
    for name, kind, shape, prec, expected in lc.GRID_CASES:
        if kind == "nmfd" and expected != "runs":
            with pytest.raises(_capi.NmfB200Error, match=expected[1].replace("(", r"\(").replace(")", r"\)")):
                B, C, L, R, T = shape
                (_capi.nmfnd_tc_plan if prec == "f16" else _capi.nmfd_plan)(B, C, [L], R, [T])


def test_tc_batch_slices_cover_the_batch():
    for B in (1, 65534, 65535, 65536, 131070, 131071, 2 ** 20 + 3):
        p = _capi.nmfnd_tc_plan(B, 1, [4], 2, [2])
        assert p["bslice"] == min(B, 65535) and p["slices"] == lc.cdiv(B, 65535)
        assert p["prep_h"] == (B * 2, 1, 1)


# ---- references ----------------------------------------------------------------------------------------------------------
def _nmf_scaled(name):
    return lc.scaled(lc.NMF_BIG[name], "nmf", SCALE)


@pytest.mark.parametrize("beta", [1, 2])
@pytest.mark.parametrize("name", list(lc.NMF_BIG))
def test_nmf_blocked_reference_equals_one_block(name, beta):
    case = _nmf_scaled(name)
    V, W, H = lc.nmf_data(case, beta, "cpu")
    blocks = 4096
    for which in case.get("which", [0, 1]):
        full = lc.nmf_terms_ref(V, W, H, beta, which, blocks=None)
        ranges = lc.row_ranges(case, which, blocks)
        n = case["C"] if which == 0 else case["N"]
        rows = sorted(r for rg in ranges for r in rg)
        assert rows == list(range(n))                                 # every row checked, the crossings included
        for rg in ranges:
            num, den = lc.nmf_terms_ref(V, W, H, beta, which, rg, blocks=blocks)
            assert torch.allclose(num, full[0][rg.start:rg.stop], rtol=1e-12, atol=0)
            if beta != 1:
                assert torch.allclose(den, full[1][rg.start:rg.stop], rtol=1e-12, atol=0)
            else:
                assert torch.allclose(den, full[1], rtol=1e-12, atol=0)


@pytest.mark.parametrize("name", list(lc.NMF_BIG))
def test_nmf_update_rows_cover_the_crossings(name):
    """The rows whose updates the GPU tests check include every row past each crossing, the first and the last, and the
    float64 terms of just those rows equal the full reference's."""
    big = lc.NMF_BIG[name]
    for which, fac in ((0, "W"), (1, "H")):
        rows = set(lc.update_rows(big, which).tolist())
        n = big["C"] if which == 0 else big["N"]
        assert {0, n - 1} <= rows
        for buf, (f, first) in lc.nmf_crossings(big).items():
            if f == fac:
                assert set(range(first, n)) <= rows, (buf, first)
    case = _nmf_scaled(name)
    beta = case["runs"].get("f32", [1])[0]
    V, W, H = lc.nmf_data(case, beta, "cpu")
    for which in (0, 1):
        rows = lc.update_rows(case, which, n_random=8)
        full = lc.nmf_terms_ref(V, W, H, beta, which, blocks=None)
        F = W if which == 0 else H
        num, den = lc.nmf_terms_ref(V, W, H, beta, which, rows, blocks=4096, F_rows=F[rows].clone())
        assert torch.allclose(num, full[0][rows], rtol=1e-12, atol=0)
        assert torch.allclose(den, full[1] if beta == 1 else full[1][rows], rtol=1e-12, atol=0)


def test_nmfd_blocked_reference_equals_one_block():
    case = lc.scaled(lc.NMFD_BIG["nmfd_long"], "nmfd", SCALE)
    V, W, H = lc.nmfd_data(case, "cpu")
    blocked = lc.nmfd_terms_ref(V, W, H, 1, blocks=4096)
    full = lc.nmfd_terms_ref(V, W, H, 1, blocks=None)
    for a, b in zip(blocked, full):
        for x, y in zip(a, b):
            assert torch.allclose(x, y, rtol=1e-12, atol=0)


def _rel(got, want):
    return float(((got - want).abs() / want.abs().clamp_min(1e-300)).max())


@pytest.mark.parametrize("name", list(lc.NMF_BIG))
def test_nmf_wrapped_index_moves_an_entry_past_its_bar(name):
    case = _nmf_scaled(name)
    N, C, R = case["N"], case["C"], case["R"]
    for prec, betas in case["runs"].items():
        for beta in betas:
            V, W, H = lc.nmf_data(case, beta, "cpu")
            Vw, Hw = lc.wrap_target(V, case["boundary"]), lc.wrap_target(H, case["boundary"])
            assert not (torch.equal(V, Vw) and torch.equal(H, Hw))
            moved = 0.0
            for which in case.get("which", [0, 1]):
                want = lc.nmf_terms_ref(V, W, H, beta, which)
                wrapped = lc.nmf_terms_ref(Vw, W, Hw, beta, which)
                if prec == "f16":
                    bar = lc.F16_BAR
                elif beta == 2:
                    bar = 0.0
                elif case.get("kl_exact"):
                    bar = lc.KL_EXACT_BAR
                else:
                    bar = fc.terms_bar(beta, R, N if which == 0 else C, 32)[0]
                moved = max(moved, _rel(wrapped[0], want[0]) / max(bar, 1e-300))
            assert moved > 1.0, (name, prec, beta, moved)


def test_nmfd_wrapped_line_moves_an_entry_past_its_bar():
    """Against the f16 bar plus the accumulation term the GPU test adds, with the full case's k-blocks per split."""
    big = lc.NMFD_BIG["nmfd_long"]
    B, C, L, R, T = lc.nmfd_dims(big)
    tcp = _capi.nmfnd_tc_plan(B, C, [L], R, [T])
    case = lc.scaled(big, "nmfd", SCALE)
    V, W, H = lc.nmfd_data(case, "cpu")
    want = lc.nmfd_terms_ref(V, W, H, 1, kappa=lc.nmfd_kappa(V, W, H))
    wrapped = lc.nmfd_terms_ref(lc.wrap_target(V, case["boundary"]), W, H, 1)
    for which, kb in ((0, tcp["kbs_w"]), (1, tcp["kbs_h"])):
        w = want[which][0]
        bar = lc.F16_BAR * w.abs() + lc.nmfd_tc_trunc(kb) * want[2][which][0]
        assert float(((wrapped[which][0] - w).abs() / bar).max()) > 1.0, which


@pytest.mark.parametrize("name", [n for n, c in lc.NMF_BIG.items() if 2 in c["runs"].get("f32", []) or c.get("kl_exact")])
def test_exact_cases_are_exact_by_their_bound(name):
    case = lc.NMF_BIG[name]
    assert lc.nmf_exact_bound(case) < fc.EXACT
    small = _nmf_scaled(name)
    if case.get("kl_exact"):
        V, W, H = lc.nmf_data(small, 1, "cpu")
        S = H @ W.t()
        P = V / (S + orc.EPS)                     # fp32, as the kernel: the ratio is an integer 0..3
        assert torch.equal(P, P.round()) and P.max() <= 3 and S[S > 0].min() >= 4 * case["R"]
        assert len(lc.nmf_hot_rows(case)) * 3 * 3 < fc.EXACT      # the W numerators: Q H over the hot rows
    else:
        V, W, H = lc.nmf_data(small, 2, "cpu")
        assert V.max() <= 4 and W.max() <= 2 and H.max() <= 2 and V.min() >= 0
    F = H if case["fac"] == "H" else W
    hot = lc.nmf_hot_rows(small, small["boundary"])
    mask = torch.ones(F.shape[0], dtype=torch.bool)
    mask[hot] = False
    assert not F[mask].any()
