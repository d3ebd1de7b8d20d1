"""CPU side of sparse targets at beta != 1, 2 (tests/sparse_beta_cases.py): the float64 restatement against the reference and
the dense oracle, the fixtures of tests/golden/reference_sparse_beta.npz, the bars against fp32 arithmetic, the cases'
reach over the launch plans, the C ABI binding and which engine a fit opens."""
import ctypes
import math
import os
import sys

import pytest
import torch

import f32_cases as fc
import sparse_beta_cases as sb
from conftest import load_golden
from oracle import mu_oracle as orc
from torchnmf_b200 import _capi
from torchnmf_b200 import engine as _engine
from torchnmf_b200.nmf import _sparse_engine_cls

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SMALL = [(9, 32, 33, "random"), (31, 33, 64, "edges"), (200, 150, 17, "lines")]


def _reference_nmf():
    """The reference's torchnmf.nmf from oracle/_ref (oracle/build_ref.py), or None where it is not installed."""
    ref = os.path.join(ROOT, "oracle", "_ref")
    if not os.path.isdir(os.path.join(ref, "torchnmf")):
        return None
    if ref not in sys.path:
        sys.path.insert(0, ref)
    import torchnmf.nmf as ref_nmf
    return ref_nmf


@pytest.mark.parametrize("beta", sb.BETAS)
@pytest.mark.parametrize("case", SMALL, ids=str)
def test_restatement_is_the_reference(case, beta):
    """The float64 terms equal the dense phi terms (and the reference's autograd gradients of `_nmf_sp_recon_beta_pos_neg`
    when the reference is installed) within 1e-12; the loss equals beta_div on the densified target."""
    N, C, R, _ = case
    rows, cols, vals, W, H = sb.sparse_bar_data(case, seed=11)
    vals[::7] = 0.0                                                  # stored zeros
    W, H = W.double(), H.double()
    V = sb.sparse_tensor(N, C, rows, cols, vals.double())
    got = sb.loss64(beta, rows, cols, vals, W, H)
    want = float(orc.beta_div(H @ W.t(), V.to_dense(), beta))
    assert abs(got - want) <= 1e-12 * abs(want), (got, want)
    Pn, Pp = orc.phi(V.to_dense(), H @ W.t(), beta)
    terms = [sb.terms64(which, beta, rows, cols, vals, W, H) for which in (0, 1)]
    for which in (0, 1):
        for g, w in zip(terms[which], fc.nmf_terms64(which, Pn, Pp, W, H)):
            assert torch.allclose(g, w, rtol=1e-12, atol=0), which
    ref = _reference_nmf()
    if ref is None:
        return
    Wg, Hg = W.clone().requires_grad_(), H.clone().requires_grad_()
    pos, neg = ref._nmf_sp_recon_beta_pos_neg(V.coalesce(), Hg, Wg, float(beta), orc.EPS)
    gpos = torch.autograd.grad(pos, (Wg, Hg), retain_graph=True)
    gneg = torch.autograd.grad(neg, (Wg, Hg))
    for which in (0, 1):
        assert torch.allclose(terms[which][0], gneg[which], rtol=1e-12, atol=0), which
        assert torch.allclose(terms[which][1], gpos[which], rtol=1e-12, atol=0), which
    vn, p, n = sb.loss_pieces64(beta, rows, cols, vals, W, H)
    assert math.isclose(p, float(pos.detach()), rel_tol=1e-12) and math.isclose(n, float(neg.detach()), rel_tol=1e-12)


SPB_CASES = load_golden("reference_sparse_beta.npz")


def test_fixtures_cover_the_issue_cases():
    assert {c["beta"] for c in SPB_CASES.values()} == set(sb.BETAS)
    for beta in sb.BETAS:
        pen = {(c["alpha"], c["l1_ratio"]) for c in SPB_CASES.values() if c["beta"] == beta}
        assert {(0.0, 0.0), (0.1, 0.5)} <= pen, beta
        assert any(c["tol"] > 0 and c["n_iter"] < c["max_iter"] for c in SPB_CASES.values() if c["beta"] == beta), beta
    ranks = {c["W0"].shape[1] for c in SPB_CASES.values()}
    assert 200 in ranks and any(r % 32 for r in ranks if r > 32)
    for c in SPB_CASES.values():
        V = c["V"]
        assert bool((V == 0).all(1).any()) and bool((V == 0).all(0).any()), "an empty row and an empty column"
        assert 0.03 < float((V != 0).double().mean()) < 0.1


@pytest.mark.parametrize("name", sorted(SPB_CASES))
def test_oracle_on_the_dense_target_matches_reference_sparse_beta_fit(name):
    """The reference's sparse path at beta 0.5 / 1.5 / 3 (nmf.py:621-636) is the dense update on V.to_dense(): the dense
    oracle reproduces every fixture."""
    c = SPB_CASES[name]
    torch.set_num_threads(1)
    W, H, n_iter, _ = orc.fit(c["V"], c["W0"], c["H0"], beta=c["beta"], tol=c["tol"], max_iter=c["max_iter"],
                              alpha=c["alpha"], l1_ratio=c["l1_ratio"])
    assert n_iter == c["n_iter"]
    assert torch.allclose(W, c["W"], rtol=1e-4, atol=1e-7), (W - c["W"]).abs().max()
    assert torch.allclose(H, c["H"], rtol=1e-4, atol=1e-7), (H - c["H"]).abs().max()


def _rel(got, want):
    assert bool((got[want == 0] == 0).all())
    return (got.double() - want).abs() / want.abs().clamp_min(1e-300)


@pytest.mark.parametrize("beta", sb.BETAS)
@pytest.mark.parametrize("case", sb.SPARSE_BETA, ids=str)
def test_bars_hold_for_fp32_and_catch_one_dropped_term(case, beta):
    """fp32 arithmetic on the CPU stays inside the numerator and loss bars; dropping the last stored entry of every segment of
    up to 64 entries exceeds the numerator bar, and dropping one stored entry exceeds the loss bar."""
    N, C, R, _ = case
    rows, cols, vals, W, H = sb.sparse_bar_data(case, seed=N + C + R)
    W64, H64 = W.double(), H.double()
    order = torch.argsort(cols * N + rows)
    for which in (0, 1):
        n = sb.seg_lengths(which, rows, cols, N, C)
        want = sb.terms64(which, beta, rows, cols, vals, W64, H64)[0]
        nbar = sb.num_bar(beta, R, n)[:, None]
        assert bool((_rel(sb.num32(which, beta, rows, cols, vals, W, H), want) <= nbar).all()), which
        if not rows.numel():
            continue
        keep = torch.ones(rows.numel(), dtype=torch.bool)
        ends = torch.cumsum(n, 0)[n > 0] - 1
        keep[(order[ends] if which == 0 else ends)] = False
        cut = sb.terms64(which, beta, rows[keep], cols[keep], vals[keep], W64, H64)[0]
        short = (n > 0) & (n <= 64)
        if bool(short.any()):
            assert bool(((cut[short] - want[short]).abs() / want[short] > nbar[short]).all()), which
    want = sb.loss64(beta, rows, cols, vals, W64, H64)
    bar = sb.loss_bar(beta, rows, cols, vals, W64, H64)
    assert abs(sb.loss32(beta, rows, cols, vals, W, H) - want) <= bar
    if rows.numel() and N * C < 10 ** 5:
        lost = sb.loss64(beta, rows[1:], cols[1:], vals[1:], W64, H64)
        assert abs(lost - want) > bar, (lost, want, bar)


def test_cases_cover_every_plan_branch():
    hit = set()
    for N, C, R, kind in sb.SPARSE_BETA:
        sp, p = _capi.sparse_plan(N, C, R), _capi.nmf_plan(N, C, R)
        hit |= {f"rpl={sp['rpl']}", f"rb={p['rb']}", f"pattern {kind}",
                f"W side nch {'1' if p['nch_w'] == 1 else '>1'}", f"H side nch {'1' if p['nch_h'] == 1 else '>1'}"}
    want = ({f"rpl={r}" for r in (1, 2, 4, 8)} | {f"rb={r}" for r in (1, 2, 4, 8, 16)}
            | {f"pattern {k}" for k in ("empty", "edges", "lines", "random")}
            | {f"{s} side nch {n}" for s in "WH" for n in ("1", ">1")})
    assert want <= hit, want - hit
    assert all(c in sb.SPARSE_BETA for c in sb.SPARSE_BETA_RATIO)


def test_any_beta_entry_point_is_bound():
    lib = _capi.load()
    res, args = _capi.SIGNATURES["nmfb200_nmf_set_target_sparse_any_beta"]
    assert (res, args) == _capi.SIGNATURES["nmfb200_nmf_set_target_sparse"]
    fn = lib.nmfb200_nmf_set_target_sparse_any_beta
    assert fn.restype is ctypes.c_int and list(fn.argtypes) == args
    # a null context is refused before any device work
    p = ctypes.c_void_p(0)
    assert fn(None, 0, p, p, p, p, p, p, 0.0, 0.0, None) != 0


@pytest.mark.parametrize("beta", [0.5, 1, 1.5, 2, 3, 0, -1])
@pytest.mark.parametrize("rank", [1, 256, 257])
@pytest.mark.parametrize("group", [None, "pg"])
@pytest.mark.parametrize("sparse_kernels", [True, False])
def test_routing_of_sparse_targets(beta, rank, group, sparse_kernels):
    got = _sparse_engine_cls(sparse_kernels, beta, rank, group)
    if not sparse_kernels or group is not None or rank > 256 or beta <= 0:
        assert got is None                                        # densified on the device
    elif beta in (1, 2):
        assert got is _engine.CudaSparseNmfEngine
    else:
        assert got is _engine.CudaSparseAnyBetaEngine
    assert issubclass(_engine.CudaSparseAnyBetaEngine, _engine.CudaSparseNmfEngine)
    assert _engine.CudaSparseNmfEngine._set_target == "nmfb200_nmf_set_target_sparse"
