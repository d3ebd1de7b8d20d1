"""GPU parity tests (run with `-m gpu` on an H100).  Everything goes through the public module
surface -> ctypes -> libnmf_b200.so C ABI -> sm_90a kernels; the CPU oracle / reference-generated
golden vectors are only the checker.

Tolerances (floating-point path, stated per the task contract):
  * precision="f32" (fused CUDA-core kernels, fp32 everywhere): rtol 2e-4, atol 1e-6 * max|x| after
    <= 50 iterations -- only summation order and libm-vs-CUDA pow/log differ from the reference.
  * precision="f16" / "f16_split" (wgmma): rtol 1e-3, atol 1e-5 * max|x| (BASELINE.json north_star).
"""
import math

import numpy as np
import pytest
import torch

from conftest import GOLDEN, load_golden
from oracle import mu_oracle as orc
from torchnmf_b200 import NMF, NMFD, PLCA, _capi

pytestmark = pytest.mark.gpu
CASES = load_golden()


def _close(a, b, rtol, atol_rel):
    atol = atol_rel * float(b.abs().max())
    ok = torch.allclose(a, b, rtol=rtol, atol=atol)
    err = ((a - b).abs() / (b.abs() + atol)).max().item()
    return ok, err


def _run_case(c, precision, on_gpu=True):
    cls = NMF if c["kind"] == "nmf" else NMFD
    m = cls(W=c["W0"], H=c["H0"], trainable_W=bool(c.get("trainable_W", 1)),
            trainable_H=bool(c.get("trainable_H", 1)))
    V = c["V"]
    if on_gpu:
        m = m.cuda()
        V = V.cuda()
    n_iter = m.fit(V, c["beta"], c["tol"], int(c["max_iter"]), False, c["alpha"], c["l1_ratio"],
                   precision=precision)
    return m, n_iter


@pytest.mark.parametrize("name", sorted(CASES))
def test_f32_path_matches_reference_golden(name):
    c = CASES[name]
    m, n_iter = _run_case(c, "f32")
    assert m.last_fit_precision == "f32"
    assert n_iter == c["n_iter"]
    for got, want, nm in ((m.W.data.cpu(), c["W"], "W"), (m.H.data.cpu(), c["H"], "H")):
        ok, err = _close(got, want, 2e-4, 1e-6)
        assert ok, f"{name} {nm}: scaled err {err:.3e}"


def test_host_buffer_mode_updates_cpu_parameters_in_place():
    c = CASES["nmf_b1_a0_l0"]
    m = NMF(W=c["W0"], H=c["H0"])
    w_ptr, h_ptr = m.W.data_ptr(), m.H.data_ptr()
    n_iter = m.fit(c["V"], c["beta"], c["tol"], int(c["max_iter"]), precision="f32")   # CPU tensors in, staged via cuda
    assert n_iter == c["n_iter"] and m.W.device.type == "cpu"
    assert m.W.data_ptr() == w_ptr and m.H.data_ptr() == h_ptr
    assert _close(m.W.data, c["W"], 2e-4, 1e-6)[0] and _close(m.H.data, c["H"], 2e-4, 1e-6)[0]


@pytest.mark.parametrize("fit", ["nmf", "sparse_fit", "plca", "plca_masked"])
def test_non_contiguous_cuda_factors_are_staged_and_written_back(fit):
    """fp32 CUDA factors that are not contiguous (here transposed storages) are staged through contiguous copies and
    written back into the same storages: the fit equals the contiguous one bit for bit."""
    g = torch.Generator().manual_seed(7)
    N, C, R = 300, 200, 12
    V = (torch.rand(N, C, generator=g) + 0.01).cuda()
    M = (torch.rand(N, C, generator=g) > 0.3).cuda()
    W0, H0 = torch.rand(C, R, generator=g) + 0.1, torch.rand(N, R, generator=g) + 0.1
    runs = []
    for strided in (False, True):
        m = (PLCA(W=W0, H=H0, rank=R) if fit.startswith("plca") else NMF(W=W0, H=H0)).cuda()
        if strided:
            for p in (m.W, m.H):
                p.data = p.data.t().contiguous().t()
            assert not m.W.is_contiguous() and not m.H.is_contiguous()
        ptrs = [p.data_ptr() for p in m.parameters()]
        if fit == "nmf":
            out = (m.fit(V, 1, 1e-4, 50, precision="f32"),)
        elif fit == "sparse_fit":
            out = (m.sparse_fit(V, 2, 20, sW=0.5, sH=0.5),)
        else:
            out = m.fit(V, 1e-4, 50, mask=M if fit == "plca_masked" else None)
        assert [p.data_ptr() for p in m.parameters()] == ptrs
        runs.append((out[0], out[1:], [p.data.cpu() for p in m.parameters()]))
    (n1, norm1, f1), (n2, norm2, f2) = runs
    assert n1 == n2 and all(torch.equal(a, b) for a, b in zip(norm1, norm2))
    assert all(bool(torch.isfinite(a).all()) and torch.equal(a, b) for a, b in zip(f1, f2))


@pytest.mark.parametrize("beta", [-1, 0, 0.5, 1, 1.5, 2, 3])
@pytest.mark.parametrize("shape", [(1000, 700, 20), (130, 2049, 33), (64, 64, 256)])
def test_f32_path_matches_oracle_seeded(beta, shape):
    N, C, R = shape
    torch.manual_seed(N + C)
    V = torch.rand(N, C) + (0.01 if beta <= 0 else 0)
    W0 = torch.rand(C, R) + 0.1
    H0 = torch.rand(N, R) + 0.1
    iters = 3
    W, H, _, losses = orc.fit(V, W0, H0, beta=beta, tol=float("-inf"), max_iter=iters, alpha=0.05, l1_ratio=0.3)
    m = NMF(W=W0, H=H0).cuda()
    m.fit(V.cuda(), beta, float("-inf"), iters, False, 0.05, 0.3, precision="f32")
    assert _close(m.W.data.cpu(), W, 2e-4, 1e-6)[0]
    assert _close(m.H.data.cpu(), H, 2e-4, 1e-6)[0]


@pytest.mark.parametrize("beta", [-1, 0, 0.5, 1, 1.5, 2, 3])
@pytest.mark.parametrize("tol", [0, 1e-4])
@pytest.mark.parametrize("alpha,l1_ratio", [(0, 0), (0.1, 0), (0.1, 0.5), (0.1, 1.0)])
def test_fit_smoke_like_reference(beta, tol, alpha, l1_ratio):
    # reference tests/test_nmf.py:104-120: only n_iter <= max_iter and no NaN
    torch.manual_seed(0)
    V = torch.rand(100, 50) + (1e-3 if beta <= 0 else 0)
    m = NMF(V.shape, 8).cuda()
    n_iter = m.fit(V.cuda(), beta, tol, 100, False, alpha, l1_ratio)
    assert n_iter <= 100
    assert not torch.isnan(m.W).any() and not torch.isnan(m.H).any()
    assert (m.W >= 0).all() and (m.H >= 0).all()


def test_loss_matches_oracle_all_betas():
    torch.manual_seed(3)
    V = torch.rand(300, 170) + 0.01
    W0 = torch.rand(170, 12); H0 = torch.rand(300, 12)
    from torchnmf_b200.engine import CudaNmfEngine
    eng = CudaNmfEngine(V.cuda(), W0.cuda(), H0.cuda(), "f32")
    for beta in (-1, 0, 0.5, 1, 1.5, 2, 3):
        want = float(orc.beta_div(orc.nmf_reconstruct(H0, W0), V, beta))
        got = eng.loss(beta)
        assert math.isclose(got, want, rel_tol=2e-4), (beta, got, want)
    eng.close()


def test_validation_errors_on_gpu():
    V = torch.rand(12, 9).cuda()
    m = NMF((12, 9), 3).cuda()
    Vn = V.clone(); Vn[3, 3] = -0.5
    with pytest.raises(AssertionError, match="non-negative"):
        m.fit(Vn)
    Vz = V.clone(); Vz[0, 0] = 0
    with pytest.raises(ValueError):
        m.fit(Vz, beta=0)
    Vnan = V.clone(); Vnan[1, 1] = float("nan")
    with pytest.raises(AssertionError):
        m.fit(Vnan)


def test_frozen_factor_untouched_on_gpu():
    c = CASES["nmf_frozenW"]
    m, _ = _run_case(c, "f32")
    assert torch.equal(m.W.data.cpu(), c["W0"])


def test_kernels_were_launched_by_our_library():
    before = _capi.launch_count()
    c = CASES["nmf_b1_a0_l0"]
    _run_case(c, "f32")
    assert _capi.launch_count() - before >= 3 * int(c["max_iter"])


# ---- size-independent properties at a larger shape (no oracle run needed) ---------------------------
@pytest.mark.parametrize("precision", ["f32"])
def test_kl_update_preserves_marginals_and_decreases_loss(precision):
    # KL multiplicative updates (beta=1, no regularisation) have two exact invariants, up to eps:
    #   after the H update: rowsum(H W^T) == rowsum(V);  and the divergence never increases.
    torch.manual_seed(5)
    N, C, R = 4096, 1536, 32
    V = torch.rand(N, C).cuda()
    m = NMF((N, C), R).cuda()
    from torchnmf_b200.engine import CudaNmfEngine
    eng = CudaNmfEngine(V, m.W.data, m.H.data, precision)
    prev = eng.loss(1)
    for it in range(5):
        eng.update_w(1, 1.0, 0.0, 0.0)
        recon_colsum = m.W.data @ m.H.data.sum(0)          # colsum of H W^T
        assert torch.allclose(recon_colsum, V.sum(0), rtol=2e-3)
        eng.update_h(1, 1.0, 0.0, 0.0)
        recon_rowsum = m.H.data @ m.W.data.sum(0)
        assert torch.allclose(recon_rowsum, V.sum(1), rtol=2e-3)
        cur = eng.loss(1)
        assert cur <= prev * (1 + 1e-5), (it, cur, prev)
        prev = cur
    eng.close()


# ---- tensor-core (wgmma) path ---------------------------------------------------------------------------
TC_RTOL, TC_ATOL_REL = 1e-3, 1e-5     # north_star: rtol 1e-3 (atol = 1e-5 * max|x| for near-zero entries)


@pytest.mark.parametrize("name", ["nmf_tc", "nmf_tcragged"])
@pytest.mark.parametrize("precision", ["f16", "f16_split"])
def test_tc_path_matches_reference_golden(name, precision):
    c = CASES[name]
    m, n_iter = _run_case(c, precision)
    assert m.last_fit_precision == precision
    assert n_iter == c["n_iter"]
    for got, want, nm in ((m.W.data.cpu(), c["W"], "W"), (m.H.data.cpu(), c["H"], "H")):
        ok, err = _close(got, want, TC_RTOL, TC_ATOL_REL)
        assert ok, f"{name} {precision} {nm}: scaled err {err:.3e}"


@pytest.mark.parametrize("shape", [(128, 128, 64), (1000, 700, 20), (130, 2049, 33), (257, 129, 1), (4096, 1024, 64),
                                   (512, 384, 128), (300, 260, 100), (1100, 777, 65)])
@pytest.mark.parametrize("precision", ["f16", "f16_split"])
def test_tc_single_updates_match_oracle(shape, precision):
    N, C, R = shape
    torch.manual_seed(N + C + R)
    V = torch.rand(N, C)
    W0 = torch.rand(C, R) + 0.05
    H0 = torch.rand(N, R) * 3
    from torchnmf_b200.engine import CudaNmfEngine
    Wd, Hd = W0.cuda(), H0.cuda()
    eng = CudaNmfEngine(V.cuda(), Wd, Hd, precision)
    eng.update_w(1, 1.0, 0.0, 0.0)
    Wn = orc.nmf_update_w(V, W0, H0, 1)
    eng.update_h(1, 1.0, 0.01, 0.02)
    Hn = orc.nmf_update_h(V, Wn, H0, 1, 1.0, 0.01, 0.02)
    eng.close()
    # one update: only the fp16 rounding of V / P / factors separates the two (V here is NOT fp16-exact)
    assert _close(Wd.cpu(), Wn, 1e-3, 1e-5)[0], _close(Wd.cpu(), Wn, 1e-3, 1e-5)[1]
    assert _close(Hd.cpu(), Hn, 1e-3, 1e-5)[0], _close(Hd.cpu(), Hn, 1e-3, 1e-5)[1]


def test_tc_handles_extreme_scales():
    # power-of-two rescaling of the fp16 operand copies: results must be scale-covariant
    torch.manual_seed(11)
    V = torch.rand(256, 384)
    W0 = torch.rand(384, 32) + 0.1
    H0 = torch.rand(256, 32) + 0.1
    outs = []
    for sv, sw in ((1.0, 1.0), (1e-3, 1e4), (300.0, 1e-5)):
        m = NMF(W=W0 * sw, H=H0).cuda()
        m.fit((V * sv).cuda(), 1, float("-inf"), 5, precision="f16_split")
        outs.append((m.W.data.cpu() @ m.H.data.cpu().t()) / sv)
        assert not torch.isnan(outs[-1]).any()
    # after a few KL iterations the reconstruction H W^T no longer depends on the initial scale of W
    # (up to eps effects, which are absolute): compare reconstructions
    assert torch.allclose(outs[0], outs[1], rtol=5e-3, atol=1e-4)


def test_tc_sharded_pieces_match_full_update():
    torch.manual_seed(12)
    N, C, R = 1024, 512, 64
    V = torch.rand(N, C).bfloat16().float(); W0 = torch.rand(C, R) + 0.1; H0 = torch.rand(N, R) + 0.1
    from torchnmf_b200.engine import CudaNmfEngine
    full_W = W0.cuda(); full_H = H0.cuda()
    eng = CudaNmfEngine(V.cuda(), full_W, full_H, "f16_split")
    eng.update_w(1, 1.0, 0.0, 0.0); eng.close()
    parts = []
    Ws = W0.cuda()
    engs = []
    for lo, hi in ((0, 600), (600, N)):
        e = CudaNmfEngine(V[lo:hi].cuda().contiguous(), Ws, H0[lo:hi].cuda().contiguous(), "f16_split")
        parts.append(e.w_partial(1)); engs.append(e)
    red = parts[0] + parts[1]
    engs[0].w_apply(red, 1, 1.0, 0.0, 0.0)
    for e in engs: e.close()
    assert torch.allclose(Ws.cpu(), full_W.cpu(), rtol=2e-4, atol=1e-7)


def test_cfg2_200_iterations_match_reference_subsample():
    """BASELINE.json configs[1] at full size: 200 KL iterations from seeds 0/1 vs the reference's own CPU
    result (tests/golden/nmf_cfg2_kl_200.npz, generated by oracle/make_golden.py --cfg2)."""
    z = np.load(f"{GOLDEN}/nmf_cfg2_kl_200.npz")
    N, C, R = 65536, 4096, 64
    torch.manual_seed(0)
    V = torch.rand(N, C).bfloat16().float()
    torch.manual_seed(1)
    W0 = torch.randn(C, R).abs(); H0 = torch.randn(N, R).abs()
    assert math.isclose(V.double().sum().item(), float(z["v_sum"]), rel_tol=1e-12)      # same inputs as the fixture
    assert math.isclose(H0.double().sum().item(), float(z["h0_sum"]), rel_tol=1e-12)
    m = NMF(W=W0, H=H0).cuda()
    n = m.fit(V.cuda(), 1, float("-inf"), int(z["iters"]))
    assert n == int(z["n_iter"])
    Wg, Hg = torch.from_numpy(z["W_sub"]), torch.from_numpy(z["H_sub"])
    W, H = m.W.data.cpu()[::8], m.H.data.cpu()[::128]
    for got, want, mx, nm in ((W, Wg, float(z["w_absmax"]), "W"), (H, Hg, float(z["h_absmax"]), "H")):
        err = ((got - want).abs() / (want.abs() + TC_ATOL_REL * mx / TC_RTOL)).max().item()
        assert torch.allclose(got, want, rtol=TC_RTOL, atol=TC_ATOL_REL * mx), f"{nm} [{m.last_fit_precision}]: {err / TC_RTOL:.2f} x tol"


@pytest.mark.parametrize("precision", ["f16", "f16_split"])
def test_tc_loss_matches_oracle(precision):
    torch.manual_seed(21)
    N, C, R = 777, 515, 48
    V = (torch.rand(N, C) * 3).bfloat16().float()
    V[5, :7] = 0.0                              # exact zeros in the target are legal for beta = 1
    W0 = torch.rand(C, R) + 0.01; H0 = torch.rand(N, R) + 0.01
    from torchnmf_b200.engine import CudaNmfEngine
    eng = CudaNmfEngine(V.cuda(), W0.cuda(), H0.cuda(), precision)
    want = float(orc.beta_div(orc.nmf_reconstruct(H0, W0).double(), V.double(), 1))
    got = eng.loss(1)
    eng.close()
    assert math.isclose(got, want, rel_tol=5e-5), (got, want)


def test_cfg2_full_size_kl_invariants_on_tensor_cores():
    """Size-independent properties at BASELINE.json's full cfg2 shape (65536 x 4096, rank 64), default precision:
    after a KL W update colsum(H W^T) == colsum(V), after the H update rowsum(H W^T) == rowsum(V) (exact up to eps for
    beta = 1 without regularisation), and the divergence never increases (nmf.py:366-391, metrics.py:22)."""
    torch.manual_seed(11)
    N, C, R = 65536, 4096, 64
    V = torch.rand(N, C, device="cuda").bfloat16().float()
    m = NMF((N, C), R).cuda()
    from torchnmf_b200.engine import CudaNmfEngine
    eng = CudaNmfEngine(V, m.W.data, m.H.data, "auto")
    assert eng.precision_for(1) == "f16"
    vcol, vrow = V.sum(0), V.sum(1)
    prev = eng.loss(1)
    for it in range(3):
        eng.update_w(1, 1.0, 0.0, 0.0)
        assert torch.allclose(m.W.data @ m.H.data.sum(0), vcol, rtol=2e-3), it
        eng.update_h(1, 1.0, 0.0, 0.0)
        assert torch.allclose(m.H.data @ m.W.data.sum(0), vrow, rtol=2e-3), it
        cur = eng.loss(1)
        assert cur <= prev * (1 + 1e-4), (it, cur, prev)
        prev = cur
    eng.check_health()
    eng.close()


# ---- beta != 1 on tensor cores (two-output kernels: numerator and denominator accumulators) -------------------
@pytest.mark.parametrize("beta", [-1, 0, 0.5, 1.5, 3])
@pytest.mark.parametrize("shape", [(384, 256, 64), (1000, 700, 20), (130, 2049, 33)])
def test_tc_two_output_updates_match_oracle(beta, shape):
    N, C, R = shape
    torch.manual_seed(N + C + R)
    V = torch.rand(N, C) + 0.01
    W0 = torch.rand(C, R) + 0.05
    H0 = torch.rand(N, R) * 3 + 0.01
    from torchnmf_b200.engine import CudaNmfEngine
    Wd, Hd = W0.cuda(), H0.cuda()
    eng = CudaNmfEngine(V.cuda(), Wd, Hd, "f16_split")
    g = orc.gamma_of(beta)
    eng.update_w(beta, g, 0.0, 0.0)
    Wn = orc.nmf_update_w(V, W0, H0, beta)
    eng.update_h(beta, g, 0.01, 0.02)
    Hn = orc.nmf_update_h(V, Wn, H0, beta, g, 0.01, 0.02)
    eng.close()
    assert _close(Wd.cpu(), Wn, 1e-3, 1e-5)[0], _close(Wd.cpu(), Wn, 1e-3, 1e-5)[1]
    assert _close(Hd.cpu(), Hn, 1e-3, 1e-5)[0], _close(Hd.cpu(), Hn, 1e-3, 1e-5)[1]


@pytest.mark.parametrize("name", [n for n in sorted(CASES) if n.startswith("nmf_b") and "_b1_" not in n and "_b2_" not in n])
def test_tc_two_output_fit_matches_reference_golden(name):
    c = CASES[name]
    m, n_iter = _run_case(c, "f16")
    assert n_iter == c["n_iter"]
    for got, want, nm in ((m.W.data.cpu(), c["W"], "W"), (m.H.data.cpu(), c["H"], "H")):
        ok, err = _close(got, want, 2e-3, 1e-5)           # 20 iterations, fp16 ratio tiles, single-rounded factors
        assert ok, f"{name} {nm}: scaled err {err:.3e}"


@pytest.mark.parametrize("beta", [-1, 0, 0.5, 1.5, 3])
@pytest.mark.parametrize("precision", ["f16", "f16_split"])
def test_tc_loss_other_betas_match_oracle(beta, precision):
    torch.manual_seed(22)
    N, C, R = 777, 515, 48
    V = (torch.rand(N, C) * 3 + 0.02).bfloat16().float()
    W0 = torch.rand(C, R) + 0.01; H0 = torch.rand(N, R) + 0.01
    from torchnmf_b200.engine import CudaNmfEngine
    eng = CudaNmfEngine(V.cuda(), W0.cuda(), H0.cuda(), precision)
    assert eng.precision_for(beta) == "f16"
    want = float(orc.beta_div(orc.nmf_reconstruct(H0, W0).double(), V.double(), beta))
    got = eng.loss(beta)
    eng.close()
    assert math.isclose(got, want, rel_tol=3e-4), (beta, got, want)


# ---- beta == 2 on tensor cores: residual tile (V - WH), numerator = O + W (H^T H) -------------------------------
@pytest.mark.parametrize("shape", [(384, 256, 64), (1000, 700, 20), (130, 2049, 33), (512, 384, 128)])
@pytest.mark.parametrize("precision", ["f16", "f16_split"])
def test_tc_frobenius_updates_match_oracle(shape, precision):
    N, C, R = shape
    torch.manual_seed(N + C + R)
    V = torch.rand(N, C)
    W0 = torch.rand(C, R) + 0.05
    H0 = torch.rand(N, R) * 3 + 0.01
    from torchnmf_b200.engine import CudaNmfEngine
    Wd, Hd = W0.cuda(), H0.cuda()
    eng = CudaNmfEngine(V.cuda(), Wd, Hd, precision)
    assert eng.precision_for(2) == precision
    eng.update_w(2, 1.0, 0.0, 0.0)
    Wn = orc.nmf_update_w(V, W0, H0, 2)
    eng.update_h(2, 1.0, 0.01, 0.02)
    Hn = orc.nmf_update_h(V, Wn, H0, 2, 1.0, 0.01, 0.02)
    want = float(orc.beta_div(orc.nmf_reconstruct(Hn, Wn).double(), V.double(), 2))
    got = eng.loss(2)
    eng.close()
    tol = 1e-3 if precision == "f16_split" else 3e-3      # single-rounded fp16 factors enter S directly here
    assert _close(Wd.cpu(), Wn, tol, 1e-5)[0], _close(Wd.cpu(), Wn, tol, 1e-5)[1]
    assert _close(Hd.cpu(), Hn, tol, 1e-5)[0], _close(Hd.cpu(), Hn, tol, 1e-5)[1]
    assert math.isclose(got, want, rel_tol=5e-3), (got, want)


@pytest.mark.parametrize("name", ["nmf_cfg1", "nmf_b2_a0_l0", "nmf_b2_a0.1_l0.5"])
def test_tc_frobenius_fit_matches_reference_golden(name):
    c = CASES[name]                                     # nmf_cfg1 = BASELINE.json configs[0]: 256x512 R=16 beta=2, 50 iterations
    m, n_iter = _run_case(c, "f16_split")
    assert m.last_fit_precision == "f16_split" and n_iter == c["n_iter"]
    for got, want, nm in ((m.W.data.cpu(), c["W"], "W"), (m.H.data.cpu(), c["H"], "H")):
        ok, err = _close(got, want, TC_RTOL, TC_ATOL_REL)
        assert ok, f"{name} {nm}: scaled err {err:.3e}"


# ---- sparse targets (nmf.py:603-638): densified on the device; the reference's own check is sparse == dense ----------
@pytest.mark.parametrize("beta", [0.5, 1, 1.5, 2, 3])
@pytest.mark.parametrize("alpha,l1_ratio", [(0, 0), (0.1, 0.5)])
def test_fit_sparse_dense_like_reference(beta, alpha, l1_ratio):
    # reference tests/test_nmf_sparse.py:8-37
    torch.manual_seed(7)
    V = torch.rand(800, 800)
    idx = torch.nonzero(V > 0.95).T
    Vs = torch.sparse_coo_tensor(idx, V[idx[0], idx[1]], V.shape)
    dense = NMF(V.shape, 16)
    sparse = NMF(V.shape, 16)
    sparse.load_state_dict(dense.state_dict())
    dense, sparse = dense.cuda(), sparse.cuda()
    n1 = dense.fit(Vs.to_dense().cuda(), beta, 0, 5, False, alpha, l1_ratio, precision="f32")
    n2 = sparse.fit(Vs.cuda(), beta, 0, 5, False, alpha, l1_ratio, precision="f32")
    assert n1 == n2
    assert torch.allclose(dense.W, sparse.W) and torch.allclose(dense.H, sparse.H)


SP_CASES = load_golden("reference_sparse.npz")


@pytest.mark.parametrize("sparse_kernels", [True, False])
@pytest.mark.parametrize("name", sorted(SP_CASES))
def test_sparse_target_fit_matches_reference_sparse_golden(name, sparse_kernels):
    """Fits the reference ran through its sparse path (nmf.py:603-638; 7 % dense, an empty row and column): here on the
    library's sparse kernels (update terms at the non-zeros only) and on the densified target, same tolerance."""
    c = SP_CASES[name]
    m = NMF(W=c["W0"], H=c["H0"]).cuda()
    m._sparse_kernels = sparse_kernels
    n_iter = m.fit(c["V"].to_sparse().cuda(), c["beta"], c["tol"], int(c["max_iter"]), False, c["alpha"], c["l1_ratio"],
                   precision="f32")
    assert n_iter == c["n_iter"]
    for got, want, nm in ((m.W.data.cpu(), c["W"], "W"), (m.H.data.cpu(), c["H"], "H")):
        ok, err = _close(got, want, 2e-4, 1e-6)
        assert ok, f"{name} {nm}: scaled err {err:.3e}"


def test_sparse_kernels_at_scale_match_the_dense_path():
    """800 x 800 as in the reference's tests/test_nmf_sparse.py:8-37, rank 64 and a rank that is not a multiple of 32."""
    torch.manual_seed(0)
    D = torch.rand(800, 800)
    D = torch.where(D > 0.95, D, torch.zeros(()))
    for R, beta in ((64, 1), (16, 2), (40, 1)):
        W0, H0 = torch.rand(800, R) + 0.1, torch.rand(800, R) + 0.1
        a = NMF(W=W0, H=H0).cuda()
        a.fit(D.to_sparse().cuda(), beta, 0, 15, False, 0.1, 0.5)
        b = NMF(W=W0, H=H0).cuda()
        b.fit(D.cuda(), beta, 0, 15, False, 0.1, 0.5, precision="f32")
        assert a.last_fit_precision == "f32"
        assert _close(a.W.data.cpu(), b.W.data.cpu(), 2e-4, 1e-6)[0]
        assert _close(a.H.data.cpu(), b.H.data.cpu(), 2e-4, 1e-6)[0]
