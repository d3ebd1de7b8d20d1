"""The sparse-target kernels term by term (csrc/sparse_nmf.cu: the SDDMM gathers, the Gram matrix, rows x Gram and the loss)
at every launch plan (tests/test_f32_plan_cover.py proves the cases reach them, asking nmfb200_nmf_sparse_plan).

(a) Exact cases (tests/sparse_cases.py): integer data for which every fp32 sum is an integer below 2^24 and every double sum
    of the loss an integer below 2^52.  The raw terms of both factors at beta 2 and beta 1 and the beta-2 loss must equal the
    float64 restatement of nmf.py:603-638 bit for bit.  Before every measured call a poisoning pass runs the same context at
    factors of 2^12 (raw terms, losses and updates of both factors), leaving huge values in the Gram partials and matrices,
    the loss partials and the update scratch; the measured raw_terms writes into a NaN-filled buffer.  A segment, row, rank
    lane, Gram pass or block that is dropped, duplicated or not rewritten fails.
(b) Float64 bars on random non-integer data: numerators gamma_n + u (beta 2) or terms_bar(1, R, n, 1) (beta 1), n the
    segment's length; beta-2 denominators gamma_R + gamma_rpb + gamma_nb + u; both losses an absolute bar summed from their
    pieces (sparse_cases.loss_bar).  One SPTERMS JSON line per case with err / bar.
(c) One update of each factor (l1, l2 > 0, gamma 2/3) from exact raw terms against nmf.py:78-92 in float64
    (f32_cases.ratio_bar): the update and raw_terms run the same kernels.
"""
import json

import pytest
import torch

import f32_cases as fc
import sparse_cases as sc
from oracle import mu_oracle as orc
from torchnmf_b200 import _capi
from torchnmf_b200.engine import CudaSparseNmfEngine, _ptr, _stream

pytestmark = pytest.mark.gpu


def _id(c):
    return "-".join(str(x) for x in c)


def _report(**kw):
    print("SPTERMS " + json.dumps(kw))


def _engine(case, rows, cols, vals, W, H):
    N, C, R, _ = case
    V = sc.sparse_tensor(N, C, rows, cols, vals).cuda().coalesce()
    return CudaSparseNmfEngine(V, W.cuda().clone(), H.cuda().clone())


def _poison(eng):
    keep = eng.W.clone(), eng.H.clone()
    for beta in (1, 2):
        eng.W.fill_(fc.POISON)
        eng.H.fill_(fc.POISON)
        for which in (0, 1):
            eng.raw_terms(which, beta)
        eng.loss(beta)
        eng.update_w(beta, 1.0, 0.0, 0.0)
        eng.update_h(beta, 1.0, 0.0, 0.0)
    eng.W.copy_(keep[0])
    eng.H.copy_(keep[1])


def _raw_terms_into_nan(eng, which, beta):
    """raw_terms through the ABI into a NaN-filled buffer: an entry the kernels do not write stays NaN."""
    n = int(eng._lib.nmfb200_nmf_raw_terms_numel(eng._ctx, which, float(beta)))
    buf = torch.full((n,), float("nan"), dtype=torch.float32, device=eng.device)
    _capi.check(eng._lib.nmfb200_nmf_raw_terms(eng._ctx, _ptr(eng.W), _ptr(eng.H), which, float(beta), _ptr(buf),
                                               _stream(eng.device)))
    rows = eng.C if which == 0 else eng.N
    num, den = buf[:rows * eng.R].view(rows, eng.R), buf[rows * eng.R:]
    return num, (den if beta == 1 else den.view(rows, eng.R))


def _assert_equal(tag, got, want):
    got = got.double().reshape(want.shape)
    if not torch.equal(got, want):
        bad = ~(got == want)
        idx = bad.nonzero()[0].tolist()
        raise AssertionError(f"{tag}: {int(bad.sum())} of {want.numel()} entries differ, first at {idx}: "
                             f"{float(got[tuple(idx)])} vs {float(want[tuple(idx)])}")


def _exact(case, beta, seed):
    """(rows, cols, vals, W, H), and the exact fp32 ratio v / (dot + eps) = Q at beta 1 (None at beta 2)."""
    if beta == 2:
        return sc.sparse_eu_data(case, seed), None
    *data, Q = sc.sparse_kl_data(case, seed)
    return data, Q.cuda()


def _dev64(rows, cols, vals, W, H):
    return rows.cuda(), cols.cuda(), vals.cuda(), W.cuda().double(), H.cuda().double()


# ---- (a) exact ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("beta", [2, 1])
@pytest.mark.parametrize("case", sc.SPARSE_EXACT, ids=_id)
def test_sparse_raw_terms_exact(case, beta):
    data, Q = _exact(case, beta, seed=sum(case[:3]) + beta)
    eng = _engine(case, *data)
    d64 = _dev64(*data)
    for which in (0, 1):
        _poison(eng)
        num, den = _raw_terms_into_nan(eng, which, beta)
        enum, eden = sc.sp_terms64(which, beta, *d64, ratio=Q)
        _assert_equal(f"num{which}", num, enum)
        _assert_equal(f"den{which}", den, eden)
    eng.close()


@pytest.mark.parametrize("case", sc.SPARSE_EXACT, ids=_id)
def test_sparse_eu_loss_exact(case):
    data = sc.sparse_eu_data(case, seed=sum(case[:3]))
    eng = _engine(case, *data)
    _poison(eng)
    want = sc.sp_loss64(2, *_dev64(*data))
    got = eng.loss(2)
    assert got == want, (got, want)
    eng.close()


def test_sparse_raw_terms_reject_other_betas():
    case = (9, 32, 33, "random")
    eng = _engine(case, *sc.sparse_eu_data(case, seed=1))
    for beta in (0, 0.5, 1.5, 3):
        with pytest.raises(_capi.NmfB200Error, match="beta must be 1 or 2"):
            eng.raw_terms(0, beta)
    eng.close()


# ---- (b) float64 bars -----------------------------------------------------------------------------------------------------
def _check_bar(tag, got, want, bar):
    """Relative error against an entry-wise bar; an entry whose reference is 0 must be 0."""
    got = got.double().reshape(want.shape)
    zero = want == 0
    assert bool((got[zero] == 0).all()), f"{tag}: an empty segment is not 0"
    err = float(((got - want).abs() / (bar * want.abs()).clamp_min(1e-300)).max()) if want.numel() else 0.0
    _report(case=tag, err_over_bar=err)
    assert err <= 1.0, f"{tag}: {err:.3f} x the bar"


@pytest.mark.parametrize("beta", [2, 1])
@pytest.mark.parametrize("case", sc.SPARSE_BAR, ids=_id)
def test_sparse_terms_within_float64_bars(case, beta):
    N, C, R, _ = case
    data = sc.sparse_bar_data(case, seed=N + C + R)
    eng = _engine(case, *data)
    d64 = _dev64(*data)
    rows, cols = d64[0], d64[1]
    plan = _capi.sparse_plan(N, C, R)
    for which in (0, 1):
        num, den = eng.raw_terms(which, beta)
        enum, eden = sc.sp_terms64(which, beta, *d64)
        n = sc.seg_lengths(which, rows, cols, N, C)
        _check_bar(f"num-b{beta}-w{which}-{_id(case)}", num, enum, sc.num_bar(beta, R, n)[:, None])
        if beta == 2:
            rpb, nb = (plan["rpb_n"], plan["nb_n"]) if which == 0 else (plan["rpb_c"], plan["nb_c"])
            _check_bar(f"den-b2-w{which}-{_id(case)}", den, eden, sc.den_bar(R, rpb, nb))
        else:
            _check_bar(f"den-b1-w{which}-{_id(case)}", den, eden, fc.gam(N if which == 0 else C) + fc.U)
    eng.close()


@pytest.mark.parametrize("beta", [2, 1])
@pytest.mark.parametrize("case", sc.SPARSE_BAR, ids=_id)
def test_sparse_loss_within_float64_bar(case, beta):
    N, C, R, _ = case
    data = sc.sparse_bar_data(case, seed=N + C + R)
    eng = _engine(case, *data)
    d64 = _dev64(*data)
    want, bar = sc.sp_loss64(beta, *d64), sc.loss_bar(beta, *d64)
    got = eng.loss(beta)
    _report(case=f"loss-b{beta}-{_id(case)}", err_over_bar=abs(got - want) / bar, bar_rel=bar / abs(want))
    assert abs(got - want) <= bar, f"{got!r} vs {want!r}, bar {bar:.3e}"
    eng.close()


# ---- (c) the update runs the raw terms' kernels ---------------------------------------------------------------------------
@pytest.mark.parametrize("beta", [2, 1])
@pytest.mark.parametrize("case", sc.SPARSE_RATIO, ids=_id)
def test_sparse_update_from_exact_terms(case, beta):
    """One W update and one H update (each from the original factors) with l1, l2 > 0 and gamma = 2/3."""
    gamma = orc.gamma_of(0.5)
    data, Q = _exact(case, beta, seed=sum(case[:3]) + 7)
    W, H = data[3].cuda(), data[4].cuda()
    eng = _engine(case, *data)
    d64 = _dev64(*data)
    for which in (0, 1):
        eng.W.copy_(W)
        eng.H.copy_(H)
        _poison(eng)
        p = d64[3] if which == 0 else d64[4]
        enum, eden = sc.sp_terms64(which, beta, *d64, ratio=Q)
        if beta == 1:
            assert bool((eden[1:] != eden[:-1]).all()), "the KL denominators must differ per component"
        (eng.update_w if which == 0 else eng.update_h)(beta, gamma, fc.RATIO_L1, fc.RATIO_L2)
        got = (eng.W if which == 0 else eng.H).double()
        want, mult = fc.ratio64(p, enum, eden, gamma, fc.RATIO_L1, fc.RATIO_L2, beta == 1)
        bar = fc.ratio_bar(mult, gamma) * want
        err = float(((got - want).abs() / bar.clamp_min(1e-300)).max())
        _report(case=f"update-b{beta}-w{which}-{_id(case)}", err_over_bar=err)
        assert err <= 1.0, f"which {which}: {err:.2f} x the bar"
    eng.close()
