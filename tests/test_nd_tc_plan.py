"""The tensor-core plan of NMF2D / NMF3D contexts (nmfb200_nmfnd_tc_plan), its refusals, the case catalogue of
tests/test_gpu_nd_tc.py, and the float64 model of the ND terms (tests/nd_tc_cases.py) -- all without a GPU."""
import pytest
import torch

import nd_tc_cases as nc
import tc_model as tcm
from oracle import mu_oracle as orc
from torchnmf_b200 import _capi
from torchnmf_b200._capi import NmfB200Error

EXTRA_SHAPES = [
    (1, 1, (4, 64), 1, (1, 64)),              # Lin = 1
    (70000, 2, (2, 10), 3, (2, 3)),           # more target lines than one grid.z: two recon launches, one dgrad launch
    (40000, 2, (2, 2, 10), 3, (1, 2, 3)),     # both slice counts above one
    (1, 300, (2, 3, 500), 7, (2, 2, 129)),
]


@pytest.mark.parametrize("name", sorted(nc.CASES))
def test_plan_matches_restatement(name):
    c = nc.CASES[name]
    p, why = nc.plan(*c)
    assert why is None
    got = _capi.nmfnd_tc_plan(*c)
    for k, v in got.items():
        want = p[k]
        assert (tuple(want) if isinstance(want, tuple) else want) == v, (name, k, v, want)


@pytest.mark.parametrize("shape", EXTRA_SHAPES, ids=str)
def test_plan_matches_restatement_on_more_shapes(shape):
    p, why = nc.plan(*shape)
    assert why is None
    got = _capi.nmfnd_tc_plan(*shape)
    assert all((tuple(p[k]) if isinstance(p[k], tuple) else p[k]) == v for k, v in got.items()), (got, p)
    if shape[0] >= 40000:
        assert got["slices"] > 1


@pytest.mark.parametrize("case", [(1, 1, 200, 1, 200), (3, 43, 400, 2, 3), (1, 24, 96, 256, 8), (70000, 3, 50, 4, 5)],
                         ids=str)
def test_outer_axes_of_size_one_plan_as_one_axis(case):
    """NMF2D / NMF3D shapes whose outer axes are all 1 plan exactly what their one-axis NMFD shape plans."""
    B, C, L, R, T = case
    a = _capi.nmfnd_tc_plan(B, C, (L,), R, (T,))
    assert (a["hslice"], a["hslices"]) == (a["bslice"], a["slices"])
    for vd, kd in (((1, L), (1, T)), ((1, 1, L), (1, 1, T))):
        assert _capi.nmfnd_tc_plan(B, C, vd, R, kd) == a


ND = "the tensor-core NMF2D / NMF3D path needs "
REFUSALS = [
    # (shape, message); each crosses the limit it is named for and no earlier one
    ((1, 4, (3, 10), 257, (2, 2)), "rank > 256 is not supported"),
    ((1, 1, (16, 16, 8), 256, (16, 16, 1)), "the tensor-core NMFD wgrad grid needs R T1 T2 ceil(T / 128) <= 65535"),
    ((1, 1, (8388608, 1), 256, (1, 1)), "a tensor-core NMFD grid passes the CUDA grid limits"),               # prep_h
    ((1, 65536, (32768, 1), 1, (1, 1)), ND + "B X1 X2 C < 2^31 - 128 (TMA row coordinate of the ratio tile)"),
    ((128, 1, (8192, 1024, 128), 1, (1, 1, 1)), ND + "B J1 J2 ceil(L / 64) < 2^31 (wgrad k-blocks)"),
    ((1, 4194240, (16, 16, 129), 1, (16, 16, 129)), ND + "C T1 T2 Tp / 64 < 2^31 (dgrad k-blocks)"),
]


@pytest.mark.parametrize("shape,msg", REFUSALS, ids=[m[-40:] for _, m in REFUSALS])
def test_refusals_name_their_limit(shape, msg):
    with pytest.raises(NmfB200Error, match=msg.replace("(", r"\(").replace(")", r"\)").replace("^", r"\^")):
        _capi.nmfnd_tc_plan(*shape)
    if shape[3] <= 256:
        assert nc.plan(*shape) == (None, msg)


def test_unreachable_bounds_are_implied():
    """The remaining 32-bit checks of the ND plan cannot fire on a shape the context accepts: nmfd_shape_of caps C at
    4194240 (so Cpad R <= 2^30), the target at 2^30 elements per (b, c) (so Lp, Lq < 2^31) and 2^40 in all (so at most
    2^26 loss partials), and the wgrad grid caps R T1 T2 ceil(T / 128) at 65535 (so R T1 T2 Tp < 2^24)."""
    assert nc.round_up(4194240, 128) * 256 <= 2 ** 30
    assert nc.plan(1, 1, (2 ** 30,), 1, (1,))[0]["Lq"] < 2 ** 31
    assert 65535 * 128 < 2 ** 24


def test_catalogue_reaches_every_branch():
    assert nc.BRANCHES <= nc.covers(), sorted(nc.BRANCHES - nc.covers())


def test_recon_kblocks_skip_border_offsets():
    """A border line runs fewer k-blocks than an interior one: no MMA on the zero rows beyond the activation's edge."""
    C, vd, R, kd = 5, (6, 40), 3, (3, 8)
    counts = [nc.recon_kblocks(C, vd, R, kd, 0, x)[0] for x in range(6)]     # NMF2D: the outer axis is X2
    assert counts == [3, 6, 9, 9, 6, 3]


@pytest.mark.parametrize("name", ["border-2d", "border-3d", "x-eq-k", "t1-1", "b3", "single-channel"])
def test_restatement_matches_oracle(name):
    """The line-by-line float64 restatement (1-D contractions summed over the outer offsets) against the oracle's ND
    contractions, and the model without rounding against both."""
    V, W, H = nc.data(*nc.CASES[name], seed=3)
    V, W, H = V.double(), W.double(), H.double()
    S = nc.reconstruct(H, W)
    assert torch.allclose(S, orc.nmfnd_reconstruct(H, W), rtol=1e-12)
    G = torch.rand_like(V)
    assert torch.allclose(nc.grad_w(G, H, tuple(W.shape[2:])), orc.nmfnd_grad_w(G, H, tuple(W.shape[2:])), rtol=1e-12)
    assert torch.allclose(nc.grad_h(G, W, tuple(H.shape[2:])), orc.nmfnd_grad_h(G, W, tuple(H.shape[2:])), rtol=1e-12)
    m = nc.NdModel(V.float(), W.float(), H.float(), rounding=False)
    for which in (0, 1):
        num, den, _ = m.raw_terms(which)
        enum, eden = nc.exact_terms(V, W, H, which)
        assert torch.allclose(num, enum, rtol=1e-12) and torch.allclose(den, eden, rtol=1e-12)
    assert abs(m.loss()[0] - nc.exact_loss(V, W, H)) <= 1e-12 * m.loss()[2]


@pytest.mark.parametrize("name", ["border-2d", "border-3d", "x-eq-k", "t-above-128", "r1", "single-channel"])
def test_model_within_its_bar_of_float64(name):
    """The rounding model lands within the f16 float64 bar of the exact terms, and its own bar is below that bar (so a
    kernel within the model's bar passes the float64 one)."""
    c = nc.CASES[name]
    V, W, H = nc.data(*c, seed=5)
    m = nc.NdModel(V, W, H)
    ws = nc.splits(*c)
    for which in (0, 1):
        num, _, bar = m.raw_terms(which, nchunks=ws[which])
        enum, _ = nc.exact_terms(V, W, H, which)
        assert float(((num - enum).abs() / enum.abs()).max()) <= nc.RTOL64, (name, which)
        assert float((bar / enum.abs()).max()) < nc.RTOL64, (name, which)
    val, bar, terms = m.loss()
    assert bar < (tcm.LOSS_RELS["f16"] + 2.0 ** -12) * terms
    assert abs(val - nc.exact_loss(V, W, H)) <= (tcm.LOSS_RELS["f16"] + 2.0 ** -12) * terms


def test_workspace_estimate_counts_the_fp16_copies():
    """A cached f16 NMF2D / NMF3D context holds the line-major ratio tile, two W copies and the padded H lines on top of
    what an fp32 context holds; an NMFD key's estimate is unchanged."""
    from torchnmf_b200.engine import _workspace_bytes
    B, C, vd, R, kd = nc.CASES["border-3d"]
    p, _ = nc.plan(B, C, vd, R, kd)
    (X1, X2, L), (T1, T2, T) = nc.outer(vd, kd)
    J12 = (X1 - T1 + 1) * (X2 - T2 + 1)
    extra = 2 * p["Lq"] * B * C * X1 * X2 + 4 * p["Cpad"] * R * T1 * T2 * p["Tp"] + 2 * p["Lp"] * B * R * J12
    f16 = _workspace_bytes(("nmfd", 0, B, C, vd, R, kd, "f16"))
    assert f16 - _workspace_bytes(("nmfd", 0, B, C, vd, R, kd, "auto")) == extra
    assert _workspace_bytes(("nmfd", 0, 1, 5, (40,), 3, (8,), "f16")) == _workspace_bytes(("nmfd", 0, 1, 5, (40,), 3, (8,), "auto"))
