"""Sparse targets at beta != 1, 2 on the engine of nmfb200_nmf_set_target_sparse_any_beta (tests/sparse_beta_cases.py): the
numerators at the stored entries against float64 bars, the V-free denominators equal bit for bit to a dense fp32 context's,
the loss, one update of each factor, fits against the reference's sparse path, a target whose dense form would take 16 GiB,
and the refusals and context reuse of the entry point.

Before every measured raw-terms call a poisoning pass runs the context at factors of 2^12 at beta 1, 2 and the tested beta
(raw terms, losses and updates of both factors), leaving huge values in every scratch buffer; the measured call writes
into a NaN-filled buffer.  One SPBETA JSON line per bar check with err / bar.
"""
import json

import pytest
import torch

import f32_cases as fc
import sparse_beta_cases as sb
from conftest import load_golden
from oracle import mu_oracle as orc
from torchnmf_b200 import NMF, _capi
from torchnmf_b200 import engine as _engine
from torchnmf_b200.engine import CudaNmfEngine, CudaSparseAnyBetaEngine, CudaSparseNmfEngine, _ptr, _stream

pytestmark = pytest.mark.gpu


def _id(c):
    return "-".join(str(x) for x in c)


def _report(**kw):
    print("SPBETA " + json.dumps(kw))


def _sparse(case, rows, cols, vals):
    N, C, _, _ = case
    return sb.sparse_tensor(N, C, rows, cols, vals).cuda().coalesce()


def _engine_of(case, rows, cols, vals, W, H, cls=CudaSparseAnyBetaEngine):
    return cls(_sparse(case, rows, cols, vals), W.cuda().clone(), H.cuda().clone())


def _poison(eng, beta):
    keep = eng.W.clone(), eng.H.clone()
    for b in (1, 2, beta):
        eng.W.fill_(fc.POISON)
        eng.H.fill_(fc.POISON)
        for which in (0, 1):
            eng.raw_terms(which, b)
        eng.loss(b)
        eng.update_w(b, 1.0, 0.0, 0.0)
        eng.update_h(b, 1.0, 0.0, 0.0)
    eng.W.copy_(keep[0])
    eng.H.copy_(keep[1])


def _raw_terms_into_nan(eng, which, beta):
    n = int(eng._lib.nmfb200_raw_terms_numel(eng._ctx, which, float(beta)))
    buf = torch.full((n,), float("nan"), dtype=torch.float32, device=eng.device)
    _capi.check(eng._lib.nmfb200_raw_terms(eng._ctx, _ptr(eng.W), _ptr(eng.H), which, float(beta), _ptr(buf),
                                           _stream(eng.device)))
    rows = eng.C if which == 0 else eng.N
    return buf[:rows * eng.R].view(rows, eng.R), buf[rows * eng.R:].view(rows, eng.R)


def _dev64(rows, cols, vals, W, H):
    return rows.cuda(), cols.cuda(), vals.cuda(), W.cuda().double(), H.cuda().double()


def _check_bar(tag, got, want, bar):
    got = got.double().reshape(want.shape)
    zero = want == 0
    assert bool((got[zero] == 0).all()), f"{tag}: an empty segment is not 0"
    err = float(((got - want).abs() / (bar * want.abs()).clamp_min(1e-300)).max()) if want.numel() else 0.0
    _report(case=tag, err_over_bar=err)
    assert err <= 1.0, f"{tag}: {err:.3f} x the bar"


@pytest.mark.parametrize("beta", sb.BETAS)
@pytest.mark.parametrize("case", sb.SPARSE_BETA, ids=_id)
def test_sparse_raw_terms_numerators_in_bar_denominators_equal_dense(case, beta):
    N, C, R, _ = case
    data = sb.sparse_bar_data(case, seed=N + C + R)
    eng = _engine_of(case, *data)
    dense = CudaNmfEngine(_sparse(case, *data[:3]).to_dense(), data[3].cuda().clone(), data[4].cuda().clone(), "f32")
    d64 = _dev64(*data)
    for which in (0, 1):
        _poison(eng, beta)
        num, den = _raw_terms_into_nan(eng, which, beta)
        enum, _ = sb.terms64(which, beta, *d64)
        n = sb.seg_lengths(which, d64[0], d64[1], N, C)
        _check_bar(f"num-b{beta}-w{which}-{_id(case)}", num, enum, sb.num_bar(beta, R, n)[:, None])
        dnum, dden = dense.raw_terms(which, beta)
        assert torch.equal(den, dden), f"which {which}: the V-free denominator differs from the dense fp32 one"
        assert not bool(torch.isnan(num).any())
    eng.close()
    dense.close()


@pytest.mark.parametrize("beta", sb.BETAS)
@pytest.mark.parametrize("case", sb.SPARSE_BETA, ids=_id)
def test_loss_within_float64_bar(case, beta):
    N, C, R, _ = case
    data = sb.sparse_bar_data(case, seed=N + C + R)
    eng = _engine_of(case, *data)
    _poison(eng, beta)
    d64 = _dev64(*data)
    want, bar = sb.loss64(beta, *d64), sb.loss_bar(beta, *d64)
    got = eng.loss(beta)
    _report(case=f"loss-b{beta}-{_id(case)}", err_over_bar=abs(got - want) / bar, bar_rel=bar / abs(want))
    assert abs(got - want) <= bar, f"{got!r} vs {want!r}, bar {bar:.3e}"
    eng.close()


@pytest.mark.parametrize("beta", sb.BETAS)
@pytest.mark.parametrize("case", sb.SPARSE_BETA_RATIO, ids=_id)
def test_update_from_its_raw_terms(case, beta):
    """One W update and one H update (each from the original factors) with l1, l2 > 0 and gamma != 1 against nmf.py:78-92 in
    float64 on the raw terms the same kernels give (f32_cases.ratio_bar)."""
    N, C, R, _ = case
    gamma = 0.7
    data = sb.sparse_bar_data(case, seed=N + C + R + 7)
    W, H = data[3].cuda(), data[4].cuda()
    eng = _engine_of(case, *data)
    for which in (0, 1):
        eng.W.copy_(W)
        eng.H.copy_(H)
        num, den = (t.double() for t in eng.raw_terms(which, beta))
        _poison(eng, beta)
        (eng.update_w if which == 0 else eng.update_h)(beta, gamma, fc.RATIO_L1, fc.RATIO_L2)
        got = (eng.W if which == 0 else eng.H).double()
        want, mult = fc.ratio64((W if which == 0 else H).double(), num, den, gamma, fc.RATIO_L1, fc.RATIO_L2, False)
        err = float(((got - want).abs() / (fc.ratio_bar(mult, gamma) * want).clamp_min(1e-300)).max())
        _report(case=f"update-b{beta}-w{which}-{_id(case)}", err_over_bar=err)
        assert err <= 1.0, f"which {which}: {err:.2f} x the bar"
    eng.close()


def _close(a, b, rtol, atol_rel):
    atol = atol_rel * float(b.abs().max())
    return torch.allclose(a, b, rtol=rtol, atol=atol), ((a - b).abs() / (b.abs() + atol)).max().item()


SPB_CASES = load_golden("reference_sparse_beta.npz")


@pytest.mark.parametrize("name", sorted(SPB_CASES))
def test_fit_matches_reference_sparse_beta_golden(name, monkeypatch):
    """Fits the reference ran through its sparse path at beta 0.5 / 1.5 / 3, here on the any-beta sparse engine."""
    c = SPB_CASES[name]
    opened = []
    init = CudaSparseAnyBetaEngine.__init__

    def spy(self, *a, **k):
        opened.append(type(self))
        init(self, *a, **k)
    monkeypatch.setattr(CudaSparseAnyBetaEngine, "__init__", spy)
    m = NMF(W=c["W0"], H=c["H0"]).cuda()
    n_iter = m.fit(c["V"].to_sparse().cuda(), c["beta"], c["tol"], int(c["max_iter"]), False, c["alpha"], c["l1_ratio"],
                   precision="f32")
    assert opened == [CudaSparseAnyBetaEngine]
    assert n_iter == c["n_iter"]
    for got, want, nm in ((m.W.data.cpu(), c["W"], "W"), (m.H.data.cpu(), c["H"], "H")):
        ok, err = _close(got, want, 2e-4, 1e-6)
        assert ok, f"{name} {nm}: scaled err {err:.3e}"


def test_no_densification_of_a_16_gib_target():
    """65536 x 65536 (16 GiB dense in fp32), about 2^20 stored entries, R = 16, beta 0.5: a 2-iteration fit stays under
    256 MiB of torch allocations, and one H update matches float64 on sampled rows."""
    N = C = 65536
    R, beta = 16, 0.5
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(3)
    nnz = 1 << 20
    idx = torch.randint(0, N * C, (nnz,), generator=g, device=dev).unique()
    rows, cols = idx // C, idx % C
    vals = torch.rand(idx.numel(), generator=g, device=dev) + 0.5
    V = torch.sparse_coo_tensor(torch.stack([rows, cols]), vals, (N, C)).coalesce()
    W0 = torch.rand(C, R, generator=g, device=dev) + 0.5
    H0 = torch.rand(N, R, generator=g, device=dev) + 0.5
    _engine.release_workspaces()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    m = NMF(W=W0, H=H0).cuda()
    m.fit(V, beta, float("-inf"), 2)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    _report(case="no-densify-65536", peak_mib=peak / 2 ** 20)
    assert peak < 256 * 2 ** 20, f"{peak / 2 ** 20:.1f} MiB"
    assert bool(torch.isfinite(m.W).all()) and bool(torch.isfinite(m.H).all())

    eng = CudaSparseAnyBetaEngine(V, W0.clone(), H0.clone())
    gamma = orc.gamma_of(beta)
    eng.update_h(beta, gamma, 0.0, 0.0)
    sample = torch.randint(0, N, (64,), generator=g, device=dev).unique()
    W64, H64 = W0.double(), H0.double()
    crow = torch.zeros(N + 1, dtype=torch.int64, device=dev)
    crow[1:] = torch.cumsum(torch.bincount(rows, minlength=N), 0)
    num = torch.zeros(sample.numel(), R, dtype=torch.float64, device=dev)
    seg = torch.zeros(sample.numel(), dtype=torch.float64, device=dev)
    for i, n in enumerate(sample.tolist()):
        e0, e1 = int(crow[n]), int(crow[n + 1])
        c = cols[e0:e1]
        x = (W64[c] @ H64[n]) + sb.EPS
        num[i] = (vals[e0:e1].double() * x.pow(beta - 2)) @ W64[c]
        seg[i] = e1 - e0
    den = (H64[sample] @ W64.t() + sb.EPS).pow(beta - 1) @ W64
    want, mult = fc.ratio64(H64[sample], num, den, gamma, 0.0, 0.0, False)
    nch = _capi.nmf_plan(N, C, R)["nch_h"]
    rel = gamma * (sb.num_bar(beta, R, seg)[:, None] + sb.den_bar(beta, R, C, nch)) + fc.ratio_bar(mult, gamma)
    err = float(((eng.H[sample].double() - want).abs() / (rel * want)).max())
    _report(case="no-densify-65536-update", err_over_bar=err)
    assert err <= 1.0
    eng.close()


def test_refusals():
    case = (9, 32, 33, "random")
    eng = _engine_of(case, *sb.sparse_bar_data(case, seed=1))
    for beta in (0, -1):
        with pytest.raises(_capi.NmfB200Error, match="beta must be positive"):
            eng.raw_terms(0, beta)
        with pytest.raises(_capi.NmfB200Error, match="beta must be positive"):
            eng.loss(beta)
        with pytest.raises(_capi.NmfB200Error, match="beta must be positive"):
            eng.update_h(beta, 1.0, 0.0, 0.0)
    eng.close()
    big = (9, 32, 257, "random")
    with pytest.raises(_capi.NmfB200Error, match="rank > 256"):
        _engine_of(big, *sb.sparse_bar_data(big, seed=1))


def _steps(case, data, fresh):
    """any-beta sparse -> dense -> old-style sparse on one shape's context: (results, context pointers)."""
    out, ptrs = [], []

    def start():
        if fresh:
            _engine.release_workspaces()

    start()
    e = _engine_of(case, *data)
    ptrs.append(e._ctx.value)
    out += [t.clone() for t in e.raw_terms(0, 0.5)] + [e.loss(0.5)]
    e.update_h(0.5, orc.gamma_of(0.5), 0.1, 0.05)
    out.append(e.H.clone())
    e.close()
    start()
    d = CudaNmfEngine(_sparse(case, *data[:3]).to_dense(), data[3].cuda().clone(), data[4].cuda().clone(), "f32")
    ptrs.append(d._ctx.value)
    out += [t.clone() for t in d.raw_terms(1, 1.5)] + [d.loss(1.5)]
    d.close()
    start()
    s = _engine_of(case, *data, cls=CudaSparseNmfEngine)
    ptrs.append(s._ctx.value)
    for beta in (0.5, 1.5, 3):
        with pytest.raises(_capi.NmfB200Error, match="beta must be 1 or 2"):
            s.raw_terms(0, beta)
        with pytest.raises(_capi.NmfB200Error, match="beta must be 1 or 2"):
            s.loss(beta)
    out += [t.clone() for t in s.raw_terms(1, 2)] + [s.loss(1)]
    s.close()
    _engine.release_workspaces()
    return out, ptrs


def test_context_reuse_resets_the_any_beta_state():
    case = (800, 800, 64, "random")
    data = sb.sparse_bar_data(case, seed=5)
    _engine.release_workspaces()
    reused, ptrs = _steps(case, data, fresh=False)
    assert len(set(ptrs)) == 1, "the three engines must share one cached context"
    fresh, _ = _steps(case, data, fresh=True)
    for i, (a, b) in enumerate(zip(reused, fresh)):
        assert (torch.equal(a, b) if isinstance(a, torch.Tensor) else a == b), i
