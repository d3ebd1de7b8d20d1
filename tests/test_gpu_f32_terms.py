"""The fp32 CUDA-core kernels term by term: the fused NMF contraction and loss (simt_nmf.cu), the NMFD / NMF2D / NMF3D sliding
GEMMs (nmfd.cu) and the ratio stage and reductions (update.cu), at every tile plan (tests/test_f32_plan_cover.py proves the
cases reach them, asking the library's planners).

(a) Exact cases (tests/f32_cases.py): integer data for which every partial sum is an integer below 2^24, so every fmaf, chunk
    and split sum is exact in any order.  The raw terms of both factors at beta 2 and beta 1, and the beta-2 losses, must
    equal float64 (plain shifted products, no convolution algorithm) bit for bit: one dropped, duplicated, shifted or stale
    term anywhere fails.  Before every measured call a poisoning pass runs the same engine at factors of 2^12 (beta 1 of
    both factors, then beta 2 of this one), leaving huge values in every chunk and split partial, in Pn / Pp and in the
    column-sum scratch: a chunk or split the measured call does not rewrite fails the comparison.
(b) Float64 bars for the mode arithmetic (beta 0, 0.5, 1.5, 3, -1; the loss at every beta), random non-integer data.  Raw
    terms: relative p (gamma_{K_S} + u) + 9u + gamma_n + gamma_{nch}, with p = |beta - 2| (numerator) or |beta - 1|
    (denominator), K_S the products per S, n the terms per sum, nch the chunks or splits (f32_cases.terms_bar: the
    powf bound is the CUDA Math API's 4 ulp).  Losses: the per-term absolute bound M rho summed over the terms, rho =
    g (gamma_{K_S} + 2u) + 16u, g = max(1, |beta|, |beta - 1|), plus gamma_16 of the sum of |terms| for the fp32 tile sums
    (f32_cases.loss_bar: powf 4 ulp, logf 1 ulp).  Term placement is proven by (a); these catch wrong eps, exponents, the IS
    branch and the loss formulas.
(c) The ratio stage (nmf.py:78-92) on exact raw terms with l1 > 0, l2 > 0 and gamma = 2/3 (gamma_of(0.5)), on the scalar and
    the four-elements-per-thread kernel, against float64 to (gamma (5 + |ln mult|) + 10) u relative (f32_cases.ratio_bar);
    the beta-1 denominators differ per component.  And the NaN-sticky min / max of the target.

Every case asserts that the fp32 kernels ran (`precision_for(beta) == "f32"`).  (b) and (c) print one F32TERMS JSON line
per case with err / bar.
"""
import json

import pytest
import torch

import f32_cases as fc
from oracle import mu_oracle as orc
from torchnmf_b200 import _capi
from torchnmf_b200.engine import CudaNmfdEngine, CudaNmfEngine

pytestmark = pytest.mark.gpu


def _id(c):
    return "-".join(str(x) for x in c).replace(" ", "").replace(",)", ")")


def _report(**kw):
    print("F32TERMS " + json.dumps(kw))


def _poison(eng, which):
    keep = eng.W.clone(), eng.H.clone()
    eng.W.fill_(fc.POISON)
    eng.H.fill_(fc.POISON)
    eng.sync()
    eng.raw_terms(1 - which, 1)
    eng.raw_terms(which, 1)
    eng.raw_terms(which, 2)
    eng.W.copy_(keep[0])
    eng.H.copy_(keep[1])
    eng.sync()


def _assert_equal(tag, got, want):
    got = got.double().reshape(want.shape)
    if not torch.equal(got, want):
        bad = got != want
        idx = bad.nonzero()[0].tolist()
        raise AssertionError(f"{tag}: {int(bad.sum())} of {want.numel()} entries differ, first at {idx}: "
                             f"{float(got[tuple(idx)])} vs {float(want[tuple(idx)])}")


def _nmf_engine(V, W, H, prec="f32"):
    return CudaNmfEngine(V.cuda(), W.cuda().clone(), H.cuda().clone(), prec)


def _nmfd_engine(case, V, W, H):
    return CudaNmfdEngine(V.cuda(), W.cuda().clone(), H.cuda().clone(), "f32" if len(case[2]) == 1 else "auto")


def _nmf_exact(case, beta, seed, loss=False):
    """(engine data, float64 phi outputs on the device): beta 2 Pn = V, Pp = S; beta 1 Pn = Q, Pp = None."""
    N, C, R = case
    if beta == 2:
        V, W, H = fc.nmf_eu_data(N, C, R, seed, loss)
        S = H.cuda().double() @ W.cuda().double().t()
        return (V, W, H), (V.cuda().double(), S)
    V, W, H, Q = fc.nmf_kl_data(N, C, R, seed)
    return (V, W, H), (Q.cuda().double(), None)


def _nmfd_exact(case, beta, seed, loss=False):
    if beta == 2:
        V, W, H = fc.nmfd_eu_data(case, seed, loss)
        return (V, W, H), (V.cuda().double(), fc.recon(H.cuda().double(), W.cuda().double()))
    V, W, H, Q = fc.nmfd_kl_data(case, seed)
    return (V, W, H), (Q.cuda().double(), None)


# ---- (a) exact ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("beta", [2, 1])
@pytest.mark.parametrize("case", fc.NMF_EXACT, ids=_id)
def test_nmf_raw_terms_exact(case, beta):
    (V, W, H), (Pn, Pp) = _nmf_exact(case, beta, seed=sum(case) + beta)
    eng = _nmf_engine(V, W, H)
    assert eng.precision_for(beta) == "f32"
    W64, H64 = W.cuda().double(), H.cuda().double()
    for which in (0, 1):
        _poison(eng, which)
        num, den = eng.raw_terms(which, beta)
        enum, eden = fc.nmf_terms64(which, Pn, Pp, W64, H64)
        _assert_equal(f"num{which}", num, enum)
        _assert_equal(f"den{which}", den, eden)
    eng.close()


@pytest.mark.parametrize("case", fc.NMF_LOSS, ids=_id)
def test_nmf_eu_loss_exact(case):
    (V, W, H), (V64, S) = _nmf_exact(case, 2, seed=sum(case), loss=True)
    eng = _nmf_engine(V, W, H)
    assert eng.precision_for(2) == "f32"
    keep = eng.H.clone()
    eng.H.fill_(fc.POISON)
    eng.loss(2)                                  # stale block partials
    eng.H.copy_(keep)
    want = float(0.5 * ((S - V64) ** 2).sum())
    assert eng.loss(2) == want
    eng.close()


@pytest.mark.parametrize("case", fc.NMF_F16, ids=_id)
def test_nmf_f16_context_beta2_runs_the_fp32_contraction(case):
    """beta 2 raw terms and the sharded W partial of an f16 context (no tensor-core partials for beta 2) are the fp32
    context's, bit for bit, and exact."""
    (V, W, H), (V64, S) = _nmf_exact(case, 2, seed=sum(case))
    a, b = _nmf_engine(V, W, H, "f32"), _nmf_engine(V, W, H, "f16")
    assert b.precision == "f16" and a.precision_for(2) == "f32"
    W64, H64 = W.cuda().double(), H.cuda().double()
    for which in (0, 1):
        enum, eden = fc.nmf_terms64(which, V64, S, W64, H64)
        for eng in (a, b):
            _poison(eng, which)
        ta, tb = a.raw_terms(which, 2), b.raw_terms(which, 2)
        for x, y, e in zip(ta, tb, (enum, eden)):
            assert torch.equal(x, y)
            _assert_equal(f"raw{which}", x, e)
    enum, eden = fc.nmf_terms64(0, V64, S, W64, H64)
    for eng in (a, b):
        _poison(eng, 0)
    pa, pb = a.w_partial(2).clone(), b.w_partial(2).clone()
    assert torch.equal(pa, pb)
    _assert_equal("w_partial", pa, torch.cat([enum.reshape(-1), eden.reshape(-1)]))
    a.close()
    b.close()


@pytest.mark.parametrize("beta", [2, 1])
@pytest.mark.parametrize("case", fc.NMFD_EXACT, ids=_id)
def test_nmfd_raw_terms_exact(case, beta):
    (V, W, H), (Pn, Pp) = _nmfd_exact(case, beta, seed=case[0] + case[1] + case[3] + beta)
    eng = _nmfd_engine(case, V, W, H)
    assert eng.precision_for(beta) == "f32"
    W64, H64 = W.cuda().double(), H.cuda().double()
    for which in (0, 1):
        _poison(eng, which)
        num, den = eng.raw_terms(which, beta)
        enum, eden = fc.nmfd_terms64(which, Pn, Pp, W64, H64)
        _assert_equal(f"num{which}", num, enum)
        _assert_equal(f"den{which}", den, eden)
    eng.close()


@pytest.mark.parametrize("case", fc.NMFD_LOSS, ids=_id)
def test_nmfd_eu_loss_exact(case):
    (V, W, H), (V64, S) = _nmfd_exact(case, 2, seed=case[1] + case[3], loss=True)
    eng = _nmfd_engine(case, V, W, H)
    assert eng.precision_for(2) == "f32"
    keep = eng.H.clone()
    eng.H.fill_(fc.POISON)
    eng.loss(2)
    eng.H.copy_(keep)
    assert eng.loss(2) == float(0.5 * ((S - V64) ** 2).sum())
    eng.close()


# ---- (b) float64 bars -----------------------------------------------------------------------------------------------------
def _check_bar(tag, got, want, bar):
    got = got.double().reshape(want.shape)
    err = float(((got - want).abs() / want.abs()).max())
    _report(case=tag, err_over_bar=err / bar, bar=bar)
    assert err <= bar, f"{tag}: {err:.3e} relative > bar {bar:.3e}"


@pytest.mark.parametrize("beta", fc.TWO_BETAS)
@pytest.mark.parametrize("case", fc.NMF_BAR, ids=_id)
def test_nmf_mode_terms_within_float64_bars(case, beta):
    N, C, R = case
    V, W, H = fc.bar_data((N, C), (C, R), (N, R), seed=N + C + R)
    eng = _nmf_engine(V, W, H)
    assert eng.precision_for(beta) == "f32"
    plan = _capi.nmf_plan(N, C, R)
    W64, H64 = W.cuda().double(), H.cuda().double()
    Pn, Pp = orc.phi(V.cuda().double(), H64 @ W64.t(), beta)
    for which, n, nch in ((0, N, plan["nch_w"]), (1, C, plan["nch_h"])):
        num, den = eng.raw_terms(which, beta)
        enum, eden = fc.nmf_terms64(which, Pn, Pp, W64, H64)
        bn, bd = fc.terms_bar(beta, R, n, nch)
        _check_bar(f"nmf-b{beta}-num{which}-{_id(case)}", num, enum, bn)
        _check_bar(f"nmf-b{beta}-den{which}-{_id(case)}", den, eden, bd)
    eng.close()


def _check_loss(tag, got, want, bar):
    _report(case=tag, err_over_bar=abs(got - want) / bar, bar_rel=bar / abs(want))
    assert abs(got - want) <= bar, f"{tag}: {got!r} vs {want!r}, bar {bar:.3e}"


@pytest.mark.parametrize("beta", fc.LOSS_BETAS)
@pytest.mark.parametrize("case", fc.NMF_BAR, ids=_id)
def test_nmf_loss_within_float64_bar(case, beta):
    N, C, R = case
    V, W, H = fc.bar_data((N, C), (C, R), (N, R), seed=N + C + R)
    eng = _nmf_engine(V, W, H)
    assert eng.precision_for(beta) == "f32"
    S = (H.cuda().double() @ W.cuda().double().t()).reshape(-1)
    want, bar = fc.loss_bar(beta, S, V.cuda().double().reshape(-1), R, orc.EPS)
    _check_loss(f"nmf-loss-b{beta}-{_id(case)}", eng.loss(beta), want, bar)
    eng.close()


def _nmfd_bar_data(case):
    B, C, X, R, K, J = fc.nmfd_dims(case)
    return fc.bar_data((B, C, *X), (C, R, *K), (B, R, *J), seed=B + C + R)


@pytest.mark.parametrize("beta", fc.TWO_BETAS)
@pytest.mark.parametrize("case", fc.NMFD_BAR, ids=_id)
def test_nmfd_mode_terms_within_float64_bars(case, beta):
    B, C, X, R, K, J = fc.nmfd_dims(case)
    V, W, H = _nmfd_bar_data(case)
    eng = _nmfd_engine(case, V, W, H)
    assert eng.precision_for(beta) == "f32"
    plan = _capi.nmfd_plan(B, C, list(X), R, list(K))
    ks, nw, nh = fc.nmfd_terms(case)
    W64, H64 = W.cuda().double(), H.cuda().double()
    Pn, Pp = orc.phi(V.cuda().double(), fc.recon(H64, W64), beta)
    for which, n, nch in ((0, nw, plan["wgrad_nsplit"]), (1, nh, plan["dgrad_nsplit"])):
        num, den = eng.raw_terms(which, beta)
        enum, eden = fc.nmfd_terms64(which, Pn, Pp, W64, H64)
        bn, bd = fc.terms_bar(beta, ks, n, nch)
        _check_bar(f"nmfd-b{beta}-num{which}-{_id(case)}", num, enum, bn)
        _check_bar(f"nmfd-b{beta}-den{which}-{_id(case)}", den, eden, bd)
    eng.close()


@pytest.mark.parametrize("beta", fc.LOSS_BETAS)
@pytest.mark.parametrize("case", fc.NMFD_BAR, ids=_id)
def test_nmfd_loss_within_float64_bar(case, beta):
    V, W, H = _nmfd_bar_data(case)
    eng = _nmfd_engine(case, V, W, H)
    assert eng.precision_for(beta) == "f32"
    S = fc.recon(H.cuda().double(), W.cuda().double()).reshape(-1)
    want, bar = fc.loss_bar(beta, S, V.cuda().double().reshape(-1), fc.nmfd_terms(case)[0], orc.EPS)
    _check_loss(f"nmfd-loss-b{beta}-{_id(case)}", eng.loss(beta), want, bar)
    eng.close()


# ---- (c) ratio stage and reductions --------------------------------------------------------------------------------------
@pytest.mark.parametrize("beta", [2, 1])
@pytest.mark.parametrize("kind,case", fc.RATIO_CASES, ids=lambda x: x if isinstance(x, str) else _id(x))
def test_ratio_stage_from_exact_terms(kind, case, beta):
    """One W update and one H update (each from the original factors) with l1, l2 > 0 and gamma = 2/3."""
    gamma = orc.gamma_of(0.5)
    if kind == "nmf":
        (V, W, H), (Pn, Pp) = _nmf_exact(case, beta, seed=sum(case) + 7)
        eng, terms = _nmf_engine(V, W, H), fc.nmf_terms64
    else:
        (V, W, H), (Pn, Pp) = _nmfd_exact(case, beta, seed=case[1] + case[3] + 7)
        eng, terms = _nmfd_engine(case, V, W, H), fc.nmfd_terms64
    assert eng.precision_for(beta) == "f32"
    W64, H64 = W.cuda().double(), H.cuda().double()
    for which in (0, 1):
        eng.W.copy_(W.cuda())
        eng.H.copy_(H.cuda())
        eng.sync()
        _poison(eng, which)
        p = (W64 if which == 0 else H64)
        enum, eden = terms(which, Pn, Pp, W64, H64)
        if beta == 1:
            assert bool((eden[1:] != eden[:-1]).all()), "the KL denominators must differ per component"
            eden = eden.reshape((1, -1) + (1,) * (p.dim() - 2))
        (eng.update_w if which == 0 else eng.update_h)(beta, gamma, fc.RATIO_L1, fc.RATIO_L2)
        got = (eng.W if which == 0 else eng.H).double()
        want, mult = fc.ratio64(p, enum, eden, gamma, fc.RATIO_L1, fc.RATIO_L2, beta == 1)
        bar = fc.ratio_bar(mult, gamma) * want
        err = float(((got - want).abs() / bar.clamp_min(1e-300)).max())
        _report(case=f"ratio-{kind}-b{beta}-w{which}-{_id(case)}", err_over_bar=err)
        assert err <= 1.0, f"which {which}: {err:.2f} x the bar"
    eng.close()


MINMAX_N, MINMAX_C = 2100, 2049        # 4.3M entries: 1024 blocks, two grid-stride steps


@pytest.mark.parametrize("where", ["first", "last_block", "last_step", "none"])
def test_minmax_is_nan_sticky(where):
    g = torch.Generator().manual_seed(4)
    V = torch.rand(MINMAX_N, MINMAX_C, generator=g) + 0.5
    flat = V.view(-1)
    flat[7] = -0.0
    flat[123456] = float("inf")
    at = {"first": 0, "last_block": 1023 * 256 + 17, "last_step": flat.numel() - 1, "none": None}[where]
    if at is not None:
        flat[at] = float("nan")
    eng = _nmf_engine(V, torch.rand(MINMAX_C, 2, generator=g), torch.rand(MINMAX_N, 2, generator=g))
    vmin, vmax = eng.minmax()
    if at is None:
        assert (vmin, vmax) == (0.0, float("inf")) and str(vmin) == "-0.0"
    else:
        assert vmin != vmin and vmax != vmax, (where, vmin, vmax)
    eng.close()


@pytest.mark.parametrize("nan", [False, True])
def test_nmfd_minmax_ragged_target(nan):
    g = torch.Generator().manual_seed(5)
    V = torch.rand(3, 5, 333, generator=g) + 0.25           # 4995 entries: not a multiple of 256 x 16
    if nan:
        V[2, 4, 332] = float("nan")
    eng = CudaNmfdEngine(V.cuda(), torch.rand(5, 2, 4, generator=g).cuda(), torch.rand(3, 2, 330, generator=g).cuda(), "f32")
    vmin, vmax = eng.minmax()
    if nan:
        assert vmin != vmin and vmax != vmax
    else:
        assert (vmin, vmax) == (float(V.min()), float(V.max()))
    eng.close()
