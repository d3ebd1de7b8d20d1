"""NMF2D / NMF3D / SIPLCA2 / SIPLCA3 at precision "f16": beta 1 on the tensor-core sliding GEMMs with the outer axes
(csrc/tc_nmfd.cu, ND kernels), on the H100.

  * the raw terms of both updates and the loss on every case of tests/nd_tc_cases.py, against the model's bar and the
    float64 oracle (as tests/test_gpu_tc_terms.py::test_nmfd_terms_and_loss does for NMFD);
  * an NMF2D with a unit outer kernel axis against NMFD on the reshaped batch: the same k-blocks in the same order, so the
    same bits;
  * repeat calls and a poisoned workspace give the same bits; auto stays on the fp32 kernels;
  * fits on the reference fixtures at the north-star bar (rtol 1e-3, atol 1e-5 max).
"""
import numpy as np
import pytest
import torch

import nd_tc_cases as nc
import tc_model as tcm
from conftest import GOLDEN, load_golden
from torchnmf_b200 import NMF2D, NMF3D, NMFD, SIPLCA2, SIPLCA3
from torchnmf_b200.engine import CudaNmfdEngine, release_workspaces

pytestmark = pytest.mark.gpu


def _engine(V, W, H, prec="f16"):
    return CudaNmfdEngine(V.cuda(), W.cuda().clone(), H.cuda().clone(), prec)


@pytest.mark.parametrize("name", sorted(nc.CASES))
def test_nd_terms_and_loss(name):
    c = nc.CASES[name]
    V, W, H = nc.data(*c, seed=len(name))
    eng = _engine(V, W, H)
    assert eng.precision_for(1) == "f16"
    model = nc.NdModel(V.cuda(), W.cuda(), H.cuda())
    ws = nc.splits(*c)
    for which in (0, 1):
        num, den = eng.raw_terms(which, 1)
        mnum, _, bar = model.raw_terms(which, nchunks=ws[which])
        enum, eden = nc.exact_terms(V, W, H, which)
        tcm.check_terms(f"nd-raw{which}-{name}", num, mnum, bar, enum, nc.RTOL64)
        assert torch.allclose(den.double().cpu(), eden.reshape(-1), rtol=1e-5), "beta 1 denominator: column sums"
    tcm.check_loss(f"nd-loss-{name}", eng.loss(1), model.loss(), nc.exact_loss(V, W, H), "f16", 1)
    eng.close()


def test_nmf2d_with_unit_outer_kernel_is_nmfd_on_the_lines():
    """NMF2D V (B, C, X1, L), W (C, R, 1, T) is NMFD on V (B X1, C, L): both contract over the same k-blocks in the same
    order, so W, H and n_iter are the same bits."""
    B, C, X1, L, R, T = 2, 20, 5, 150, 6, 9
    g = torch.Generator().manual_seed(7)
    V = torch.rand(B, C, X1, L, generator=g) + 0.1
    W0 = torch.rand(C, R, 1, T, generator=g) + 0.1
    H0 = torch.rand(B, R, X1, L - T + 1, generator=g) + 0.1
    m2 = NMF2D(W=W0, H=H0).cuda()
    n2 = m2.fit(V.cuda(), 1, 1e-6, 30, precision="f16")
    assert m2.last_fit_precision == "f16"
    Vd = V.permute(0, 2, 1, 3).reshape(B * X1, C, L)
    Hd = H0.permute(0, 2, 1, 3).reshape(B * X1, R, L - T + 1)
    md = NMFD(W=W0[:, :, 0].contiguous(), H=Hd.contiguous()).cuda()
    nd = md.fit(Vd.contiguous().cuda(), 1, 1e-6, 30, precision="f16")
    assert md.last_fit_precision == "f16"
    assert n2 == nd
    assert torch.equal(m2.W.data[:, :, 0], md.W.data)
    assert torch.equal(m2.H.data.permute(0, 2, 1, 3).reshape(B * X1, R, -1), md.H.data)


def test_shapes_with_unit_outer_axes_take_the_nmfd_kernels():
    """An NMF2D / NMF3D context whose outer axes are all 1 is an NMFD context: same plan, same terms bit for bit."""
    B, C, L, R, T = 2, 30, 200, 5, 12
    V, W, H = nc.data(B, C, (L,), R, (T,), seed=11)
    e1 = _engine(V, W, H)
    for shape in ((1,), (1, 1)):
        e2 = _engine(V.view(B, C, *shape, L), W.view(C, R, *shape, T), H.view(B, R, *shape, L - T + 1))
        assert e2.precision_for(1) == "f16"
        for which in (0, 1):
            a, b = e1.raw_terms(which, 1), e2.raw_terms(which, 1)
            assert torch.equal(a[0].reshape(-1), b[0].reshape(-1)) and torch.equal(a[1], b[1])
        assert torch.equal(e1.loss_tensor(1).clone(), e2.loss_tensor(1).clone())
        e2.close()
    e1.close()


@pytest.mark.parametrize("name", ["border-3d", "single-channel", "r129"])
def test_repeat_and_poisoned_workspace_are_bit_identical(name):
    c = nc.CASES[name]
    V, W, H = nc.data(*c, seed=1)
    eng = _engine(V, W, H)
    first = [t.clone() for which in (0, 1) for t in eng.raw_terms(which, 1)] + [eng.loss_tensor(1).clone()]
    again = [t.clone() for which in (0, 1) for t in eng.raw_terms(which, 1)] + [eng.loss_tensor(1).clone()]
    assert all(torch.equal(a, b) for a, b in zip(first, again))
    eng.close()
    release_workspaces()
    # a fresh context on device memory that held 0xFF bytes: every byte the kernels read is written or zeroed first
    junk = torch.full((1 << 28,), 0xFF, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    del junk
    torch.cuda.empty_cache()
    fresh = _engine(V, W, H)
    poisoned = [t.clone() for which in (0, 1) for t in fresh.raw_terms(which, 1)] + [fresh.loss_tensor(1).clone()]
    assert all(torch.equal(a, b) for a, b in zip(first, poisoned))
    fresh.close()


def test_auto_and_other_betas_stay_on_the_fp32_kernels():
    V, W, H = nc.data(*nc.CASES["border-2d"], seed=2)
    eng = _engine(V, W, H, "auto")
    assert eng.precision_for(1) == "f32"
    eng.close()
    eng = _engine(V, W, H, "f16")
    assert eng.precision_for(1) == "f16"
    assert eng.precision_for(2) == "f32" and eng.precision_for(0.5) == "f32"
    eng.close()
    m = NMF2D(W=W, H=H).cuda()
    m.fit(V.cuda(), 1, float("-inf"), 3)
    assert m.last_fit_precision == "f32"


def test_f16_refusal_names_the_limit():
    V = torch.rand(1, 1, 16, 16, 8, device="cuda")
    W = torch.rand(1, 256, 16, 16, 1, device="cuda")
    H = torch.rand(1, 256, 1, 1, 8, device="cuda")
    with pytest.raises(Exception, match="wgrad grid needs R T1 T2"):
        CudaNmfdEngine(V, W, H, "f16")


def _close(got, want, rtol=1e-3, atol_rel=1e-5):
    atol = atol_rel * float(want.abs().max())
    return float(((got - want).abs() / (rtol * want.abs() + atol)).max())


ND_CASES = load_golden("reference_nd.npz")
ND_CLS = {"nmf2d": NMF2D, "nmf3d": NMF3D}


@pytest.mark.parametrize("name", sorted(n for n in ND_CASES if "_b1_" in n))
def test_nd_fit_at_f16_matches_reference_golden(name):
    c = ND_CASES[name]
    m = ND_CLS[c["kind"]](W=c["W0"], H=c["H0"]).cuda()
    n_iter = m.fit(c["V"].cuda(), c["beta"], c["tol"], int(c["max_iter"]), False, c["alpha"], c["l1_ratio"],
                   precision="f16")
    assert m.last_fit_precision == "f16"
    assert n_iter == c["n_iter"]
    for got, want, nm in ((m.W.data.cpu(), c["W"], "W"), (m.H.data.cpu(), c["H"], "H")):
        err = _close(got, want)
        assert err <= 1.0, f"{name} {nm}: {err:.3f} x the north-star tolerance"


ZP = np.load(f"{GOLDEN}/reference_plca.npz", allow_pickle=False)
PLCA_CLS = {2: SIPLCA2, 3: SIPLCA3}


def _plca_case(name):
    c = {k.split("/", 1)[1]: ZP[k] for k in ZP.files if k.startswith(name + "/")}
    c.setdefault("tol", np.array(float("-inf")))
    for k in ("trainable_W", "trainable_H", "trainable_Z"):
        c.setdefault(k, np.array(1))
    return c


@pytest.mark.parametrize("name", sorted({k.split("/")[0] for k in ZP.files if k.startswith(("siplca2_", "siplca3_"))}))
def test_siplca_nd_fit_at_f16_matches_reference_golden(name):
    c = _plca_case(name)
    t = lambda k: torch.from_numpy(c[k].copy())  # noqa: E731
    m = PLCA_CLS[int(c["cls"])](W=t("W0"), H=t("H0"), Z=t("Z0"), trainable_W=bool(int(c["trainable_W"])),
                                trainable_H=bool(int(c["trainable_H"])), trainable_Z=bool(int(c["trainable_Z"]))).cuda()
    n_iter, norm = m.fit(t("V").cuda(), float(c["tol"]), int(c["iters"]), False, float(c["W_alpha"]), float(c["H_alpha"]),
                         float(c["Z_alpha"]), precision="f16")
    assert m.last_fit_precision == "f16"
    assert n_iter == int(c["n_iter"])
    for nm in ("W", "H", "Z"):
        err = _close(getattr(m, nm).data.cpu(), t(nm))
        assert err <= 1.0, f"{name} {nm}: {err:.3f} x the north-star tolerance"
