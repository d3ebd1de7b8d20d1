"""CPU tests of the float64 model of the tensor-core arithmetic (tests/tc_model.py).

With rounding off the model is the oracle (oracle/mu_oracle.py), term by term; with rounding on its error against exact
float64 shows what the split mode is for (split <= fast / 2); and the GPU cases of tests/test_gpu_tc_terms.py are ones where
the model's bar and a kernel that rounds as the model passes the float64 bar.
"""
import pytest
import torch

import tc_model as tcm
import test_gpu_tc_terms as gt
from oracle import mu_oracle as orc


def _rel(a, b):
    return float(((a - b).abs() / b.abs()).max())


def _nmf(N, C, R, seed, vmin=0.01):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(N, C, generator=g) + vmin, torch.rand(C, R, generator=g) + 0.1, torch.rand(N, R, generator=g) + 0.1


@pytest.mark.parametrize("beta", [1, 2, 0, 0.5, 1.5, 3, -1])
def test_nmf_model_without_rounding_is_the_oracle(beta):
    V, W, H = _nmf(70, 50, 9, seed=1)
    V, W, H = V.double(), W.double(), H.double()
    m = tcm.NmfModel(V, W, H, "f16", rounding=False)
    num, den, _, _ = m.raw_terms(0, beta)
    onum, oden = orc.nmf_w_contractions(V, W, H, beta)
    assert torch.allclose(num, onum, rtol=1e-12) and torch.allclose(den.reshape(oden.shape), oden, rtol=1e-12)
    num, den, _, _ = m.raw_terms(1, beta)
    Pn, Pp = orc.phi(V, orc.nmf_reconstruct(H, W), beta)
    assert torch.allclose(num, Pn @ W, rtol=1e-12)
    assert torch.allclose(den, W.sum(0) if beta == 1 else Pp @ W, rtol=1e-12)
    want = float(orc.beta_div(orc.nmf_reconstruct(H, W), V, beta))
    assert abs(m.loss(beta)[0] - want) <= 1e-12 * abs(want)
    assert abs(m.loss(beta, fold=True)[0] - want) <= 1e-12 * abs(want)


def test_nmfd_model_without_rounding_is_the_oracle():
    g = torch.Generator().manual_seed(2)
    V, W, H = torch.rand(2, 7, 40, generator=g), torch.rand(7, 3, 6, generator=g) + 0.1, torch.rand(2, 3, 35, generator=g) + 0.1
    V, W, H = V.double(), W.double(), H.double()
    m = tcm.NmfdModel(V, W, H, rounding=False)
    P = V / (orc.nmfd_reconstruct(H, W) + orc.EPS)
    num, den, _ = m.raw_terms(0)
    assert torch.allclose(num, orc.nmfd_grad_w(P, H, 6), rtol=1e-12) and torch.allclose(den, H.sum((0, 2)), rtol=1e-12)
    num, den, _ = m.raw_terms(1)
    assert torch.allclose(num, orc.nmfd_grad_h(P, W, 35), rtol=1e-12) and torch.allclose(den, W.sum((0, 2)), rtol=1e-12)
    want = float(orc.beta_div(orc.nmfd_reconstruct(H, W), V, 1))
    assert abs(m.loss()[0] - want) <= 1e-12 * abs(want)


def test_operand_copies():
    """fp16 copies at the power-of-two scale that puts the maximum in [2^13, 2^14); split: hi + lo carries ~22 bits."""
    x = torch.rand(1000, dtype=torch.float64).float().double() * 3.7 + 0.01
    assert tcm.pow2_exp(3.71) == 12 and tcm.pow2_exp(0.0) == 0 and tcm.ratio_exp(1.0) == -4
    hi, lo = tcm.operand(x, False)
    assert torch.equal(lo, torch.zeros_like(x)) and _rel(hi, x) <= 2.0 ** -11
    hi, lo = tcm.operand(x, True)
    assert _rel(hi + lo, x) <= 2.0 ** -21 and not torch.equal(lo, torch.zeros_like(x))


@pytest.mark.parametrize("shape,ratio", [((1000, 700, 20), 0.5), ((4096, 1024, 64), 0.5), ((300, 260, 100), 0.7)])
def test_split_model_is_more_accurate_than_fast(shape, ratio):
    """The raw W and H numerators of the model against exact float64 (max relative error): the split mode's error is at
    most half the fast mode's where the factors' rounding dominates.  At 300 x 260 x 100 the fast mode's S error already
    averages over 100 rank terms while the rounding both modes share (fp16 V, the ratio tile) averages over only ~300
    columns: the split mode gains less there (0.51 and 0.63 of the fast mode's error for the H and W sides)."""
    V, W, H = _nmf(*shape, seed=sum(shape), vmin=0.0)
    exact = tcm.NmfModel(V, W, H, "f16", rounding=False)
    for which in (0, 1):
        want = exact.raw_terms(which, 1)[0]
        fast = _rel(tcm.NmfModel(V, W, H, "f16").raw_terms(which, 1)[0], want)
        split = _rel(tcm.NmfModel(V, W, H, "f16_split").raw_terms(which, 1)[0], want)
        assert split <= fast * ratio, (which, fast, split)
        assert fast <= gt.RTOL64["f16"] / 2 and split <= gt.RTOL64["f16_split"] / 2, (which, fast, split)


@pytest.mark.parametrize("case", gt.NMF_CASES + gt.CHUNK_CASES, ids=gt._id)
def test_gpu_nmf_cases_are_passable(case):
    """Every beta 1 GPU case: a kernel within the model bar of the model is within the float64 bar."""
    prec, N, C, R = case
    V, W, H = gt._data(N, C, R, seed=N * 7 + C + R)
    model, exact = tcm.NmfModel(V, W, H, prec), tcm.NmfModel(V, W, H, prec, rounding=False)
    for which in (0, 1):
        num, _, bar, _ = model.raw_terms(which, 1)
        want = exact.raw_terms(which, 1)[0]
        tight = float((bar / want).max())
        assert _rel(num, want) + tight <= gt.RTOL64[prec], which


@pytest.mark.parametrize("case", gt.NMFD_CASES, ids=gt._id)
def test_gpu_nmfd_cases_are_passable(case):
    V, W, H = gt._nmfd_data(*case, seed=sum(case))
    model, exact = tcm.NmfdModel(V, W, H), tcm.NmfdModel(V, W, H, rounding=False)
    for which in (0, 1):
        num, _, bar = model.raw_terms(which)
        want = exact.raw_terms(which)[0]
        tight, rtol64 = float((bar / want).max()), gt.nmfd_rtol64(case, V, W, H)
        assert _rel(num, want) + tight <= rtol64, which


def _mutated_numerator(m, which, drop):
    """The beta 1 numerator of the split model with one term of the split arithmetic dropped."""
    Fh, Fl, Gh, Gl, Vm, _, G32 = m._orient(which)
    S = Fh @ Gh.t() + (0 if drop == "Flo Ghi" else Fl @ Gh.t()) + (0 if drop == "Fhi Glo" else Fh @ Gl.t())
    P = Vm / (S + tcm.EPS)
    tile = tcm._round_tile(P - m.kappa, tcm.ratio_exp(m.kappa), True)
    return tile @ (Gh if drop == "P Glo" else Gh + Gl) + m.kappa * G32.sum(0)


@pytest.mark.parametrize("case", gt.STRUCT_CASES, ids=gt._id)
def test_structured_split_cases_see_every_split_term(case):
    """On the structured split inputs a kernel that dropped Flo Ghi, Fhi Glo or P Glo would miss the model by more than
    twice the model bar, in both orientations; a kernel within the model bar passes the float64 bar."""
    prec, N, C, R = case
    V, W, H = gt._structured_data(N, C, R, seed=N + C + R)
    model, exact = tcm.NmfModel(V, W, H, prec), tcm.NmfModel(V, W, H, prec, rounding=False)
    for which in (0, 1):
        num, _, bar, _ = model.raw_terms(which, 1)
        want = exact.raw_terms(which, 1)[0]
        assert _rel(num, want) + float((bar / want).max()) <= gt.RTOL64["f16"], which
        for drop in ("Flo Ghi", "Fhi Glo", "P Glo"):
            miss = float(((_mutated_numerator(model, which, drop) - num).abs() / bar).max())
            assert miss >= 2.0, (which, drop, miss)
