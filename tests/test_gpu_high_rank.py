"""Dense NMF and PLCA above rank 256 on the rank-blocked fp32 kernels (simt_nmf.cu, update.cu), on the H100.

(a) Exact cases (tests/high_rank_cases.py, exact by the integer argument of tests/f32_cases.py): the raw terms of both factors
    at beta 2 and beta 1 and the beta-2 losses equal float64 bit for bit, after the poisoning pass of
    tests/test_gpu_f32_terms.py (huge stale values in every chunk slab and the column-sum scratch).
(b) Beta 0, 0.5, 1.5, 3 raw terms and losses within f32_cases.terms_bar / loss_bar; the ratio stage within ratio_bar.
(c) The entry points agree bit for bit: iterate(k) = k x (update_w; update_h), w_partial + w_apply = update_w,
    loss_prefetch_w = loss.
(d) NMF.fit / NMF((N, C)) / PLCA.fit against the reference fixtures of tests/golden/reference_high_rank.npz at the f32
    tolerances of tests/test_gpu_parity.py; BetaMu's fused path; sparse targets densified; the caps that stay.
(b) prints one HIGHRANK JSON line per case with err / bar.
"""
import ctypes
import json
import math

import pytest
import torch

import f32_cases as fc
import high_rank_cases as hc
from oracle import mu_oracle as orc
from test_high_rank_plan import CASES, NMF_NAMES, inputs, plca_inputs, sample
from torchnmf_b200 import NMF, PLCA, BetaMu, NMFD, _capi
from torchnmf_b200.engine import CudaNmfEngine

pytestmark = pytest.mark.gpu


def _id(c):
    return "-".join(str(x) for x in c)


def _report(**kw):
    print("HIGHRANK " + json.dumps(kw))


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


def _engine_of(V, W, H, prec="f32"):
    return CudaNmfEngine(V.cuda(), W.cuda().clone(), H.cuda().clone(), prec)


def _exact(case, beta, seed, loss=False):
    N, C, R = case
    if beta == 2:
        V, W, H = fc.nmf_eu_data(N, C, R, seed, loss)
        return (V, W, H), (V.cuda().double(), H.cuda().double() @ W.cuda().double().t())
    V, W, H, Q = fc.nmf_kl_data(N, C, R, seed)
    return (V, W, H), (Q.cuda().double(), None)


# ---- (a) exact ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("beta", [2, 1])
@pytest.mark.parametrize("case", hc.HIGH_EXACT, ids=_id)
def test_raw_terms_exact(case, beta):
    (V, W, H), (Pn, Pp) = _exact(case, beta, seed=sum(case) + beta)
    eng = _engine_of(V, W, H)
    assert eng.precision_for(beta) == "f32"
    W64, H64 = W.cuda().double(), H.cuda().double()
    for which in (0, 1):
        _poison(eng, which)
        num, den = eng.raw_terms(which, beta)
        enum, eden = fc.nmf_terms64(which, Pn, Pp, W64, H64)
        _assert_equal(f"num{which}", num, enum)
        _assert_equal(f"den{which}", den, eden)
    eng.close()


@pytest.mark.parametrize("case", hc.HIGH_LOSS, ids=_id)
def test_eu_loss_exact(case):
    (V, W, H), (V64, S) = _exact(case, 2, seed=sum(case), loss=True)
    eng = _engine_of(V, W, H)
    keep = eng.H.clone()
    eng.H.fill_(fc.POISON)
    eng.loss(2)
    eng.H.copy_(keep)
    assert eng.loss(2) == float(0.5 * ((S - V64) ** 2).sum())
    eng.close()


# ---- (b) float64 bars -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("beta", [0, 0.5, 1.5, 3])
@pytest.mark.parametrize("case", hc.HIGH_BAR, ids=_id)
def test_mode_terms_and_loss_within_float64_bars(case, beta):
    N, C, R = case
    V, W, H = fc.bar_data((N, C), (C, R), (N, R), seed=N + C + R)
    eng = _engine_of(V, W, H)
    assert eng.precision_for(beta) == "f32"
    plan = _capi.nmf_plan(N, C, R)
    W64, H64, V64 = W.cuda().double(), H.cuda().double(), V.cuda().double()
    S = H64 @ W64.t()
    Pn, Pp = orc.phi(V64, S, beta)
    for which, n, nch in ((0, N, plan["nch_w"]), (1, C, plan["nch_h"])):
        num, den = eng.raw_terms(which, beta)
        enum, eden = fc.nmf_terms64(which, Pn, Pp, W64, H64)
        for tag, got, want, bar in zip(("num", "den"), (num, den), (enum, eden), fc.terms_bar(beta, R, n, nch)):
            err = float(((got.double() - want).abs() / want.abs()).max())
            _report(case=f"terms-b{beta}-{tag}{which}-{_id(case)}", err_over_bar=err / bar)
            assert err <= bar, (tag, which, err, bar)
    want, bar = fc.loss_bar(beta, S.reshape(-1), V64.reshape(-1), R, orc.EPS)
    got = eng.loss(beta)
    _report(case=f"loss-b{beta}-{_id(case)}", err_over_bar=abs(got - want) / bar)
    assert abs(got - want) <= bar
    eng.close()


@pytest.mark.parametrize("beta", [2, 1])
@pytest.mark.parametrize("case", hc.HIGH_RATIO, ids=_id)
def test_ratio_stage_from_exact_terms(case, beta):
    gamma = orc.gamma_of(0.5)
    (V, W, H), (Pn, Pp) = _exact(case, beta, seed=sum(case) + 7)
    eng = _engine_of(V, W, H)
    W64, H64 = W.cuda().double(), H.cuda().double()
    for which in (0, 1):
        eng.W.copy_(W.cuda())
        eng.H.copy_(H.cuda())
        eng.sync()
        _poison(eng, which)
        p = W64 if which == 0 else H64
        enum, eden = fc.nmf_terms64(which, Pn, Pp, W64, H64)
        if beta == 1:
            assert bool((eden[1:] != eden[:-1]).all()), "the KL denominators must differ per component"
            eden = eden.reshape(1, -1)
        (eng.update_w if which == 0 else eng.update_h)(beta, gamma, fc.RATIO_L1, fc.RATIO_L2)
        got = (eng.W if which == 0 else eng.H).double()
        want, mult = fc.ratio64(p, enum, eden, gamma, fc.RATIO_L1, fc.RATIO_L2, beta == 1)
        err = float(((got - want).abs() / (fc.ratio_bar(mult, gamma) * want).clamp_min(1e-300)).max())
        _report(case=f"ratio-b{beta}-w{which}-{_id(case)}", err_over_bar=err)
        assert err <= 1.0, (which, err)
    eng.close()


# ---- (c) entry points ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("beta", [1, 2, 0.5])
@pytest.mark.parametrize("case", [(300, 700, 300), (1000, 2000, 1000)], ids=_id)
def test_entry_points_agree_bit_for_bit(case, beta):
    N, C, R = case
    V, W, H = fc.bar_data((N, C), (C, R), (N, R), seed=N + R)
    gamma, l1, l2 = orc.gamma_of(beta), 0.05, 0.02
    a, b = _engine_of(V, W, H), _engine_of(V, W, H)
    a.iterate(3, beta, gamma, l1, l2)
    for _ in range(3):
        b.update_w(beta, gamma, l1, l2)
        b.update_h(beta, gamma, l1, l2)
    assert torch.equal(a.W, b.W) and torch.equal(a.H, b.H)
    assert a.loss_prefetch_w(beta) == b.loss(beta)
    keep = b.W.clone()
    b.update_w(beta, gamma, l1, l2)
    want = b.W.clone()
    b.W.copy_(keep)
    b.sync()
    b.w_apply(b.w_partial(beta).clone(), beta, gamma, l1, l2)
    assert torch.equal(b.W, want)
    a.close()
    b.close()


# ---- (d) modules against the reference ------------------------------------------------------------------------------------------
def _close(a, b, rtol=2e-4, atol_rel=1e-6):
    atol = atol_rel * float(b.abs().max())
    return torch.allclose(a, b, rtol=rtol, atol=atol), float(((a - b).abs() / (b.abs() + atol)).max())


@pytest.mark.parametrize("name", NMF_NAMES)
def test_fit_matches_reference_fixture(name, monkeypatch):
    c = CASES[name]
    V, W0, H0 = inputs(c)
    if int(c["default_rank"]):
        m = NMF(tuple(V.shape)).cuda()                       # rank = the number of columns (nmf.py:684-686)
        assert m.W.shape == (V.shape[1], V.shape[1])
        m.W.data.copy_(W0)
        m.H.data.copy_(H0)
    else:
        m = NMF(W=W0, H=H0).cuda()
    trace = []

    def recording(orig):
        def call(self, beta):
            d = orig(self, beta)
            trace.append(math.sqrt(2.0 * d))
            return d
        return call
    for meth in ("loss", "loss_prefetch_w"):
        monkeypatch.setattr(CudaNmfEngine, meth, recording(getattr(CudaNmfEngine, meth)))
    n_iter = m.fit(V.cuda(), float(c["beta"]), float("-inf"), int(c["max_iter"]), False, float(c["alpha"]),
                   float(c["l1_ratio"]), precision="auto")
    assert m.last_fit_precision == "f32"
    assert n_iter == int(c["n_iter"])
    for got, want, nm in ((sample(m.W.data.cpu(), c, "w"), c["W_sub"], "W"),
                          (sample(m.H.data.cpu(), c, "h"), c["H_sub"], "H")):
        ok, err = _close(got, torch.from_numpy(want))
        _report(case=f"fit-{name}-{nm}", err_over_tol=err)
        assert ok, f"{name} {nm}: scaled err {err:.3e}"
    assert len(trace) == len(c["losses"])
    assert torch.allclose(torch.tensor(trace, dtype=torch.float64), torch.from_numpy(c["losses"]), rtol=2e-4)


def test_plca_fit_matches_reference_fixture():
    c = CASES["plca_r300"]
    V, W0, H0, Z0 = plca_inputs(c)
    m = PLCA(W=W0, H=H0, Z=Z0).cuda()
    n_iter, norm = m.fit(V.cuda(), float("-inf"), int(c["max_iter"]))
    assert n_iter == int(c["n_iter"])
    assert abs(float(norm) - float(c["norm"])) <= 1e-6 * float(c["norm"])
    for got, want, nm in ((sample(m.W.data.cpu(), c, "w"), c["W_sub"], "W"),
                          (sample(m.H.data.cpu(), c, "h"), c["H_sub"], "H"), (m.Z.data.cpu(), c["Z"], "Z")):
        ok, err = _close(got, torch.from_numpy(want))
        _report(case=f"plca-{nm}", err_over_tol=err)
        assert ok, f"{nm}: scaled err {err:.3e}"


def test_explicit_tensor_core_precision_keeps_its_limit():
    V, W0, H0 = fc.bar_data((200, 300), (300, 300), (200, 300), seed=1)
    m = NMF(W=W0, H=H0).cuda()
    with pytest.raises(_capi.NmfB200Error, match="R <= 128"):
        m.fit(V.cuda(), 1, float("-inf"), 2, precision="f16")


def test_betamu_fused_at_rank_300():
    V, W0, H0 = fc.bar_data((200, 350), (350, 300), (200, 300), seed=3)
    out = {}
    for fused in (True, False):                                # the autograd path: the same module on the host
        dev = "cuda" if fused else "cpu"
        m = NMF(W=W0, H=H0).to(dev)
        Vd = V.to(dev)
        tr = BetaMu([m.W, m.H], 1.0)

        def closure():
            tr.zero_grad()
            return Vd, (m if fused else m())
        paths = []
        for _ in range(5):
            tr.step(closure)
            paths += tr.last_step_paths
        assert paths and set(paths) == ({"fused"} if fused else {"autograd"}), paths
        out[fused] = (m.W.data.cpu(), m.H.data.cpu())
    for a, b in zip(out[True], out[False]):
        ok, err = _close(a, b)
        assert ok, err


def test_sparse_target_above_256_runs_densified():
    g = torch.Generator().manual_seed(5)
    N, C, R = 300, 400, 300
    V = torch.rand(N, C, generator=g) * (torch.rand(N, C, generator=g) < 0.2)
    W0, H0 = torch.rand(C, R, generator=g) + 0.1, torch.rand(N, R, generator=g) + 0.1
    a, b = NMF(W=W0, H=H0).cuda(), NMF(W=W0, H=H0).cuda()
    na = a.fit(V.cuda().to_sparse(), 1, float("-inf"), 20)
    nb = b.fit(V.cuda(), 1, float("-inf"), 20)
    assert na == nb and torch.equal(a.W.data, b.W.data) and torch.equal(a.H.data, b.H.data)


def test_sparse_target_rejected_by_the_c_abi_above_256():
    N, C, R = 40, 50, 300
    W, H = torch.rand(C, R, device="cuda"), torch.rand(N, R, device="cuda")
    lib = _capi.load()
    ctx = ctypes.c_void_p()
    _capi.check(lib.nmfb200_nmf_create(ctypes.byref(ctx), torch.cuda.current_device(), N, C, R, _capi.PREC_F32))
    try:
        z = torch.zeros(max(N, C) + 1, dtype=torch.int64, device="cuda")
        p = ctypes.c_void_p(z.data_ptr())
        rc = lib.nmfb200_nmf_set_target_sparse(ctx, 0, p, p, p, p, p, p, 0.0, 0.0, None)
        assert rc == 1 and b"256" in lib.nmfb200_last_error()
    finally:
        lib.nmfb200_destroy(ctx)
    del W, H


def test_nmfd_keeps_the_rank_cap():
    V = torch.rand(1, 4, 100, device="cuda")
    m = NMFD(W=torch.rand(4, 257, 4), H=torch.rand(1, 257, 97)).cuda()
    with pytest.raises(_capi.NmfB200Error, match="256"):
        m.fit(V, 1, float("-inf"), 1)
