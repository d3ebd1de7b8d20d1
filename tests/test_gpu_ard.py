"""Automatic relevance determination on the GPU (`fit(V, ..., ard=ARD(...))`, include/nmf_b200.h: nmfb200_set_ard).

Every ratio stage that takes the penalties is checked bit for bit against the scalar l1 update it generalises: with every
pen_k equal to p (registered with b = 2^60, c = 1, phi = p 2^60, so lambda_k = 2^60 and pen_k = fp32(p) exactly), one W and
one H update equal the update with l1_reg = p; with distinct penalties, column k equals the update with l1_reg = pen_k.  The
lambda update is checked against float64, whole fits against the float64 ARD oracle (tests/ard_oracle.py), and the
plumbing for determinism and for a registration that is cleared again.
"""
import math

import pytest
import torch

import ard_oracle as ao
from ard_cases import PLANTED_ITERS, planted_nmf, planted_nmfd, relevant
from torchnmf_b200 import NMF, NMF2D, NMF3D, NMFD
from torchnmf_b200 import _capi, engine as E
from torchnmf_b200.nmf import ARD, _gamma, _observed_cells

pytestmark = pytest.mark.gpu
DEV = "cuda"
BIG = 2.0 ** 60

# ---- the paths: (name, builder of an engine on copies of W0 / H0, beta, the factors) ------------------------------------


def _nmf_factors(N, C, R, seed, vdtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    V = (torch.rand(N, 6, generator=g) @ torch.rand(6, C, generator=g) + 0.05 * torch.rand(N, C, generator=g))
    V[torch.rand(N, C, generator=g) < 0.05] = 0.0
    return V.to(vdtype).to(DEV), torch.rand(C, R, generator=g) + 0.1, torch.rand(N, R, generator=g) + 0.1


def _conv_factors(nd, R, seed):
    g = torch.Generator().manual_seed(seed)
    X, K = {1: ((200,), (7,)), 2: ((12, 40), (3, 5)), 3: ((6, 8, 20), (2, 3, 4))}[nd]
    B, C = 2, 12
    V = torch.rand(B, C, *X, generator=g) + 0.05
    W = torch.rand(C, R, *K, generator=g) + 0.1
    H = torch.rand(B, R, *(x - k + 1 for x, k in zip(X, K)), generator=g) + 0.1
    return V.to(DEV), W, H


def _path(name, beta, R=64, precision="f32"):
    """(make(W, H) -> engine, V, W0, H0) of one path."""
    if name in ("nmf", "f16v", "bf16v"):
        vd = {"nmf": torch.float32, "f16v": torch.float16, "bf16v": torch.bfloat16}[name]
        V, W0, H0 = _nmf_factors(640, 384, R, 1, vd)
        return (lambda W, H: E.CudaNmfEngine(V, W, H, precision)), V, W0, H0
    if name == "sparse":
        V, W0, H0 = _nmf_factors(640, 384, R, 2)
        Vs = (V * (V > 1.2)).to_sparse().coalesce()
        cls = E.CudaSparseNmfEngine if beta in (1, 2) else E.CudaSparseAnyBetaEngine
        return (lambda W, H: cls(Vs, W, H)), Vs, W0, H0
    if name in ("mask", "weight"):
        V, W0, H0 = _nmf_factors(640, 384, R, 3)
        g = torch.Generator().manual_seed(4)
        M = (torch.rand(V.shape, generator=g) < 0.7).to(DEV)
        Wt = (torch.rand(V.shape, generator=g) * 2 * (torch.rand(V.shape, generator=g) < 0.8)).to(DEV)

        def make(W, H):
            e = E.CudaNmfEngine(V, W, H, "f32")
            if name == "mask":
                e.set_mask(M)
            else:
                e.set_weight(Wt)
            return e
        return make, V, W0, H0
    if name == "smask":
        V, W0, H0 = _nmf_factors(640, 384, R, 5)
        g = torch.Generator().manual_seed(6)
        M = (torch.rand(V.shape, generator=g) < 0.2).to(DEV).to_sparse()
        O = _observed_cells(V, M, torch.device(DEV))
        return (lambda W, H: E.CudaObservedNmfEngine(O, W, H)), V, W0, H0
    nd = {"nmfd": 1, "nmf2d": 2, "nmf3d": 3}[name]
    V, W0, H0 = _conv_factors(nd, R, 7 + nd)
    return (lambda W, H: E.CudaNmfdEngine(V, W, H, precision)), V, W0, H0


PATHS = ([("nmf", b, R, p) for p in ("f32", "f16", "f16_split") for b in (1, 0.5, 2) for R in (16, 64, 128)] +
         [("sparse", b, 64, "f32") for b in (1, 2, 1.5)] +
         [(n, b, 64, "f32") for n in ("mask", "weight", "smask") for b in (1, 0.5)] +
         [(n, 1, 64, p) for n in ("f16v", "bf16v") for p in ("f32", "auto")] +
         [("nmfd", 0.5, 8, "f32"), ("nmfd", 1, 8, "f16"), ("nmf2d", 1, 8, "f16"), ("nmf3d", 1, 8, "f32"),
          ("nmf3d", 2, 8, "f32")])


def _ids(p):
    return f"{p[0]}-b{p[1]}-R{p[2]}-{p[3]}"


def _run(make, W0, H0, which, l1=0.0, ard=None, both=False):
    """Fresh copies of W0 / H0 on the device, an engine, optionally an ARD registration (b, c, phi), then one update of
    W (which 0) or H (which 1), or W then H (`both`).  Returns (W, H, pen or None)."""
    W, H = W0.to(DEV).contiguous(), H0.to(DEV).contiguous()
    eng = make(W, H)
    try:
        pen = None
        if ard is not None:
            eng.set_ard(*ard)
            pen = eng.ard_state()[1].cpu()
        beta, gamma = eng._beta, _gamma(eng._beta)
        if both or which == 0:
            eng.update_w(beta, gamma, l1, 0.0)
        if both or which == 1:
            eng.update_h(beta, gamma, l1, 0.0)
        torch.cuda.synchronize()
        return W.cpu(), H.cpu(), pen
    finally:
        eng.close()


def _with_beta(make, beta):
    def mk(W, H):
        e = make(W, H)
        e._beta = beta
        return e
    return mk


@pytest.mark.parametrize("path", PATHS, ids=_ids)
def test_equal_penalties_are_the_scalar_l1_update(path):
    name, beta, R, prec = path
    make, _, W0, H0 = _path(name, beta, R, prec)
    make = _with_beta(make, beta)
    p = 0.3
    Wa, Ha, pen = _run(make, W0, H0, 0, ard=(BIG, 1.0, p * BIG), both=True)
    assert torch.equal(pen, torch.full_like(pen, torch.tensor(p, dtype=torch.float32).item()))
    Ws, Hs, _ = _run(make, W0, H0, 0, l1=p, both=True)
    assert torch.equal(Wa, Ws) and torch.equal(Ha, Hs)
    assert not torch.equal(Wa, W0)


@pytest.mark.parametrize("path", PATHS[::2] + PATHS[1::6], ids=_ids)
def test_distinct_penalties_column_by_column(path):
    name, beta, R, prec = path
    make, _, W0, H0 = _path(name, beta, R, prec)
    make = _with_beta(make, beta)
    c = W0.numel() // R + H0.numel() // R + 6.0
    ard = (0.5, c, 20.0)
    for which in (0, 1):
        Wa, Ha, pen = _run(make, W0, H0, which, ard=ard)
        assert len(set(pen.tolist())) > R // 2            # the penalties differ from component to component
        got = Wa if which == 0 else Ha
        for k in sorted({0, R // 2, R - 1}):
            Ws, Hs, _ = _run(make, W0, H0, which, l1=float(pen[k]))
            want = Ws if which == 0 else Hs
            assert torch.equal(got[:, k], want[:, k]), (which, k)


def _lambda64(W, H, b, c):
    return (ao.comp_sums(W.double()) + ao.comp_sums(H.double()) + b) / c


@pytest.mark.parametrize("name", ["nmf", "nmfd", "nmf3d"])
def test_lambda_update_against_float64(name):
    make, _, W0, H0 = _path(name, 1, 64 if name == "nmf" else 8)
    R = W0.shape[1]
    b, c, phi = 0.7, W0.numel() // R + H0.numel() // R + 6.0, 1.5
    W, H = W0.to(DEV), H0.to(DEV)
    eng = make(W, H)
    try:
        eng.set_ard(b, c, phi)
        u = 2.0 ** -24
        n = max(W0.numel(), H0.numel()) // R
        for it in range(3):
            lam, pen, change = (t.cpu() if torch.is_tensor(t) else t for t in eng.ard_state())
            want = _lambda64(W.cpu(), H.cpu(), b, c)
            bound = 2 * n * u * (ao.comp_sums(W.cpu().double()) + ao.comp_sums(H.cpu().double())) / c + 2 * u * want
            assert torch.all((lam.double() - want).abs() <= bound), it
            assert torch.equal(pen, (phi / lam.double()).float())
            if it == 0:
                assert change == 0.0
            eng.update_w(1, 1.0, 0.0, 0.0)
            eng.update_h(1, 1.0, 0.0, 0.0)
            eng.ard_update()
            first = eng.ard_state()
            eng.ard_update()
            second = eng.ard_state()
            assert torch.equal(first[0], second[0]) and torch.equal(first[1], second[1]) and second[2] == 0.0
            want_change = float(((first[0].cpu().double() - lam.double()).abs() / lam.double()).max())
            assert math.isclose(first[2], want_change, rel_tol=1e-6, abs_tol=1e-12)
    finally:
        eng.close()


# ---- whole fits -----------------------------------------------------------------------------------------------------------

def _mean(V):
    return float(V.sum(dtype=torch.float64)) / V.numel()


def _close(a, b, rtol, atol_rel):
    return torch.allclose(a.double(), b.double(), rtol=rtol, atol=atol_rel * float(b.abs().max()))


def _scaled_err(a, b, rtol, atol_rel):
    """max |a - b| / (rtol |b| + atol): <= 1 inside the tolerance."""
    return float(((a.double() - b).abs() / (rtol * b.abs() + atol_rel * float(b.abs().max()))).max())


@pytest.mark.parametrize("precision,beta", [("f32", 1), ("f32", 0.5), ("f32", 2), ("auto", 1), ("f16", 1),
                                            ("f16_split", 1)])
def test_nmf_fit_matches_the_oracle(precision, beta):
    # the parity tests' kind of target: uniform and exact in bf16 (tests/test_gpu_parity.py)
    g = torch.Generator().manual_seed(11)
    N, C, R = 512, 320, 32
    V = torch.rand(N, C, generator=g).bfloat16().float()
    W0, H0 = torch.rand(C, R, generator=g) + 0.1, torch.rand(N, R, generator=g) + 0.1
    m = NMF(W=W0, H=H0).to(DEV)
    phi = 1.0 if beta != 2 else 0.01
    n = m.fit(V.to(DEV), beta, tol=float("-inf"), max_iter=50, precision=precision, ard=ARD(phi=phi))
    W, H, lam, n_ref, b, c = ao.fit(V, W0, H0, beta=beta, tol=float("-inf"), max_iter=50, phi=phi, mean_v=_mean(V))
    assert n == n_ref == 50
    tc = m.last_fit_precision != "f32"
    rtol, atol = (1e-3, 1e-5) if tc else (2e-4, 1e-6)
    for got, want in ((m.W.data.cpu(), W), (m.H.data.cpu(), H), (m.ard_lambda.cpu(), lam)):
        assert _close(got, want, rtol, atol), (m.last_fit_precision, _scaled_err(got, want, rtol, atol))
    assert m.ard_lambda.dtype == torch.float32 and m.ard_lambda.device.type == "cuda"
    assert math.isclose(m.ard_bound, b / c, rel_tol=1e-12)


@pytest.mark.parametrize("cls,nd,precision", [(NMFD, 1, "f32"), (NMFD, 1, "f16"), (NMF2D, 2, "f16"), (NMF3D, 3, "f32")])
def test_convolutive_fit_matches_the_oracle(cls, nd, precision):
    V, W0, H0 = _conv_factors(nd, 6, 12)
    V = V.cpu()
    m = cls(W=W0, H=H0).to(DEV)
    n = m.fit(V.to(DEV), 1, tol=float("-inf"), max_iter=50, precision=precision, ard=ARD())
    kind = {1: "nmfd", 2: "nmf2d", 3: "nmf3d"}[nd]
    W, H, lam, _, b, c = ao.fit(V, W0, H0, beta=1, tol=float("-inf"), max_iter=50, kind=kind, mean_v=_mean(V))
    assert n == 50
    tc = m.last_fit_precision != "f32"
    rtol, atol = (1e-3, 1e-5) if tc else (2e-4, 1e-6)
    for got, want in ((m.W.data.cpu(), W), (m.H.data.cpu(), H), (m.ard_lambda.cpu(), lam)):
        assert _close(got, want, rtol, atol), (m.last_fit_precision, _scaled_err(got, want, rtol, atol))


@pytest.mark.parametrize("precision", ["f32", "auto"])
def test_planted_nmf_keeps_the_oracles_components(precision):
    V, W0, H0 = planted_nmf()
    m = NMF(W=W0, H=H0).to(DEV)
    m.fit(V.to(DEV), 1, tol=float("-inf"), max_iter=PLANTED_ITERS, precision=precision, ard=ARD())
    _, _, lam, _, b, c = ao.fit(V, W0, H0, beta=1, tol=float("-inf"), max_iter=PLANTED_ITERS, mean_v=_mean(V))
    want = relevant(lam, b / c)
    assert len(want) == 4
    assert relevant(m.ard_lambda.cpu(), m.ard_bound) == want


def test_planted_nmfd_keeps_the_oracles_components():
    V, W0, H0 = planted_nmfd()
    m = NMFD(W=W0, H=H0).to(DEV)
    m.fit(V.to(DEV), 1, tol=float("-inf"), max_iter=PLANTED_ITERS, ard=ARD())
    _, _, lam, _, b, c = ao.fit(V, W0, H0, beta=1, tol=float("-inf"), max_iter=PLANTED_ITERS, kind="nmfd",
                                mean_v=_mean(V))
    want = relevant(lam, b / c)
    assert len(want) == 2
    assert relevant(m.ard_lambda.cpu(), m.ard_bound) == want


def test_stop_rule_fires_on_the_device_change():
    V, W0, H0 = planted_nmf()
    m = NMF(W=W0, H=H0).to(DEV)
    n = m.fit(V.to(DEV), 1, tol=1e-3, max_iter=400, precision="f32", ard=ARD())
    _, _, _, n_ref, _, _ = ao.fit(V, W0, H0, beta=1, tol=1e-3, max_iter=400, mean_v=_mean(V))
    assert n % 10 == 0 and n < 400 and abs(n - n_ref) <= 10


# ---- determinism and plumbing ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("precision,beta", [("f32", 1), ("f16", 1), ("f32", 0.5), ("f16_split", 2)])
def test_two_fits_give_identical_bits(precision, beta):
    V, W0, H0 = _nmf_factors(512, 320, 64, 13)
    outs = []
    for _ in range(2):
        m = NMF(W=W0, H=H0).to(DEV)
        m.fit(V, beta, tol=float("-inf"), max_iter=30, precision=precision, ard=ARD(phi=0.1 if beta == 2 else 1.0))
        outs.append((m.W.data.cpu(), m.H.data.cpu(), m.ard_lambda.cpu()))
    assert all(torch.equal(a, b) for a, b in zip(*outs))


@pytest.mark.parametrize("precision,beta", [("f32", 1), ("f16", 1), ("f32", 2), ("f16", 2)])
def test_fused_iterate_equals_per_update_calls(precision, beta):
    V, W0, H0 = _nmf_factors(512, 320, 64, 14)
    res = []
    for fused in (True, False):
        W, H = W0.to(DEV), H0.to(DEV)
        eng = E.CudaNmfEngine(V, W, H, precision)
        try:
            eng.set_ard(0.3, 320 + 512 + 6.0, 1.0)
            if fused:
                eng.iterate(7, beta, _gamma(beta), 0.0, 0.0)
            else:
                for _ in range(7):
                    eng.update_w(beta, _gamma(beta), 0.0, 0.0)
                    eng.update_h(beta, _gamma(beta), 0.0, 0.0)
                    eng.ard_update()
            lam, pen, change = eng.ard_state()
            res.append((W.cpu(), H.cpu(), lam.cpu(), pen.cpu(), change))
        finally:
            eng.close()
    a, b = res
    assert all(torch.equal(x, y) for x, y in zip(a[:4], b[:4])) and a[4] == b[4]


@pytest.mark.parametrize("path", [("nmf", 1, 64, "f16"), ("nmf", 2, 64, "f32"), ("nmfd", 1, 8, "f16"), ("smask", 1, 64, "f32")],
                         ids=_ids)
def test_registered_then_cleared_is_the_plain_update(path):
    name, beta, R, prec = path
    make, _, W0, H0 = _path(name, beta, R, prec)

    def cleared(W, H):
        e = make(W, H)
        e._beta = beta
        e.set_ard(1.0, 100.0, 1.0)
        e.set_ard(None, None, None)
        return e
    Wc, Hc, _ = _run(cleared, W0, H0, 0, both=True)
    Wp, Hp, _ = _run(_with_beta(make, beta), W0, H0, 0, both=True)
    assert torch.equal(Wc, Wp) and torch.equal(Hc, Hp)


def test_abi_refusals():
    V, W0, H0 = _nmf_factors(256, 128, 16, 15)
    W, H = W0.to(DEV), H0.to(DEV)
    eng = E.CudaNmfEngine(V, W, H, "f16")
    lib = _capi.load()
    try:
        assert lib.nmfb200_ard_update(eng._ctx, E._ptr(W), E._ptr(H), None) == 3          # NMFB200_ERR_STATE
        eng.set_ard(1.0, 400.0, 1.0)
        fixed = torch.zeros(16, dtype=torch.uint8, device=DEV)
        assert lib.nmfb200_set_fixed_w(eng._ctx, E._ptr(fixed), None) == 1
        red = torch.zeros(2 * 128 * 16, device=DEV)
        assert lib.nmfb200_w_apply(eng._ctx, E._ptr(W), E._ptr(red), 1.0, 1.0, 0.0, 0.0, None) == 1
        assert lib.nmfb200_nmf_peer_supported(eng._ctx, 1.0) == 0
        assert lib.nmfb200_nmf_cd_update(eng._ctx, E._ptr(W), E._ptr(H), 0, 0.0, 0.0, None) == 1
        assert lib.nmfb200_set_ard(eng._ctx, E._ptr(W), E._ptr(H), float("nan"), 1.0, 1.0, None) == 1
        assert lib.nmfb200_set_ard(eng._ctx, E._ptr(W), E._ptr(H), 1.0, 1.0, 0.0, None) == 1
        eng.set_ard(None, None, None)
        eng.set_fixed_w(fixed)
        assert lib.nmfb200_set_ard(eng._ctx, E._ptr(W), E._ptr(H), 1.0, 1.0, 1.0, None) == 1
    finally:
        eng.close()
    Vb = V.reshape(1, 256, 128).expand(2, 256, 128).contiguous()
    Wb, Hb = W0.to(DEV).expand(2, 128, 16).contiguous(), H0.to(DEV).expand(2, 256, 16).contiguous()
    beng = E.CudaBatchedNmfEngine(Vb, Wb, Hb)
    try:
        assert lib.nmfb200_set_ard(beng._ctx, E._ptr(Wb), E._ptr(Hb), 1.0, 1.0, 1.0, None) == 1
        assert b"batched" in lib.nmfb200_last_error()
    finally:
        beng.close()
