"""The tensor-core contractions one term at a time, against exact float64 and against the float64 model of their rounding
(tests/tc_model.py), at the tile edges of every kernel configuration.

Every case compares what the kernels return before any MU rule can hide an error: the raw numerator / denominator of one
update (`raw_terms`), the loss, for beta 1 the loss folded into the W update's contraction (`loss_prefetch_w`), and for
beta 2 (no tensor-core raw terms) one W and one H update.  Every case asserts the path that ran (`precision_for`).

Two bars per case:
  * against the model: the per-element bound of tc_model's error model (fp32 accumulation truncating at most 8 ulp per
    16-term k-step, rcp.approx, the one-ulp steps of the ratio tile's double rounding, the fp32 chunk sums).  Each case
    reports how this bound compares with the float64 bar below (TIGHTER).
  * against exact float64 (the oracle at the same fp32 inputs, computed in float64), the accuracy of the mode:
      f16        1.25e-3 relative (2^-10 + 2^-12): the fp16 rounding of each factor (unit roundoff 2^-11) goes into S and
                 so into the ratio, up to 2^-10 where S has a single term (rank 1) and averaged over the rank and shift
                 terms otherwise; fp16 V and the ratio tile add up to 2^-11 per term, averaged over the >= 64-term sums
      f16_split  2.5e-4 relative (~2^-12): hi + lo factors are ~22-bit, S is good to ~2^-20; what remains is fp16 V and the
                 ratio tile, up to 2^-11 per term averaged over the sum (the split mode exists to be this much tighter)
      two-output tiles (beta not 1 or 2; fast mode only): S enters as x^(beta-2) (numerator) and x^(beta-1) (denominator),
                 so the f16 bar is multiplied by max(1, |exponent|)
    Losses are held relative to the sum of the absolute values of their summed terms ("terms"): f16 (2^-11 g + 2^-12),
    f16_split (2^-20 g + 2^-12) with g = max(1, |beta|, |beta - 1|) the power S enters with; 2^-12 is fp16 V in the cross
    term, never averaged in the worst case.
"""
import json

import pytest
import torch

import tc_model as tcm
from tc_model import LOSS_RELS, RTOL64, TIGHTER, cdiv, nmfd_rtol64  # noqa: F401  (shared with the sequence harness)
from tc_model import check_loss as _check_loss, check_terms as _check_terms, nmfd_splits as _nmfd_splits, plan as _plan, tn as _tn
from oracle import mu_oracle as orc
from oracle_engine import OracleNmfEngine, OracleNmfdEngine
from torchnmf_b200 import NMFD
from torchnmf_b200.engine import CudaNmfdEngine, CudaNmfEngine

pytestmark = pytest.mark.gpu

# ---- NMF cases: every configuration <RP, SPLIT, TN> meets every edge -------------------------------------------------------
# N and C each run through the residues 1, 63, 64, 65, 127, 0 mod 128: rows of F mod 128 in {1, 64, 65, 127, 0} and
# contracted columns mod TN in {1, 63, 64, 65, 0} (TN = 64 for Split128) in both orientations.
RES = [1, 63, 64, 65, 127, 0]
RANKS = {64: [1, 8, 63, 64, 8, 63], 128: [65, 100, 127, 128, 100, 65]}
CONFIGS = [("f16", 64), ("f16_split", 64), ("f16", 128), ("f16_split", 128)]


def _nmf_cases():
    cases = []
    for prec, rp in CONFIGS:
        for i, rn in enumerate(RES):
            rc = RES[(i + 2) % len(RES)]
            N = 256 + (rn or 128)
            C = 128 * (1 + i % 3) + (rc or 128)
            cases.append((prec, N, C, RANKS[rp][i]))
    return cases


NMF_CASES = _nmf_cases()
# make_plan splits the contracted columns into chunks with a short last one (mirrored by _plan): W side, H side
# (fast mode: a split-mode model bar over 4161-term sums is not 5x tighter than the split mode's float64 bar)
CHUNK_CASES = [("f16", 4161, 200, 20), ("f16", 200, 4161, 20), ("f16", 200, 2113, 100), ("f16", 2113, 200, 100)]
TWO_BETAS = [0, 0.5, 1.5, 3, -1]


def _data(N, C, R, seed, vmin=0.0, fmin=0.1):
    g = torch.Generator().manual_seed(seed)
    V = torch.rand(N, C, generator=g) + vmin
    W = torch.rand(C, R, generator=g) + fmin
    H = torch.rand(N, R, generator=g) + fmin
    return V, W, H


def _biased(x, frac=0.375):
    """x moved so that its fp16 operand copy (tc_model.operand) rounds every entry down by `frac` of an fp16 ulp: the lo
    halves of the split copy all have one sign and add up instead of cancelling."""
    x = x.double()
    a = tcm.pow2_exp(x.max())
    xs = x * 2.0 ** a

    def ulp(h):
        return torch.exp2(torch.frexp(h.abs().clamp_min(2.0 ** -14))[1].double() - 11)
    h = tcm.f16(xs)
    h = torch.where(h > xs, h - ulp(h), h)
    return ((h + frac * ulp(h)) * 2.0 ** -a).float()


def _structured_data(N, C, R, seed):
    """Split-mode inputs on which every term of the split arithmetic shows: factors whose fp16 copies all lose 3/8 ulp in
    the same direction (Flo Ghi, Fhi Glo and P Glo do not average out over the sums), and a target with 1/64 of its rows
    and columns 32x hotter, where P >> kappa and the centred tile carries the sum."""
    g = torch.Generator().manual_seed(seed)
    V = torch.rand(N, C, generator=g) + 0.05
    V[torch.randperm(N, generator=g)[:max(1, N // 64)]] *= 32
    V[:, torch.randperm(C, generator=g)[:max(1, C // 64)]] *= 32
    W = _biased(torch.rand(C, R, generator=g) + 0.1)
    H = _biased(torch.rand(N, R, generator=g) + 0.1)
    return V, W, H


# both split configurations, ranks 1 to 128; rows / columns with the residues of NMF_CASES
STRUCT_CASES = [("f16_split", N, C, R) for N, C, R in
                [(257, 192, 1), (319, 321, 8), (384, 447, 63), (321, 256, 64), (257, 192, 65), (383, 257, 100),
                 (320, 511, 127), (321, 256, 128)]]


def _engine(prec, V, W, H):
    eng = CudaNmfEngine(V.cuda(), W.cuda().clone(), H.cuda().clone(), prec)
    return eng


def _nchunks(prec, N, C, R, which):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return _plan(C, N, sms, _tn(prec, R))[2] if which == 0 else _plan(N, C, sms, _tn(prec, R))[2]


def _id(c):
    return "-".join(str(x) for x in c)


@pytest.mark.parametrize("case", NMF_CASES + CHUNK_CASES, ids=_id)
def test_nmf_kl_terms_and_loss(case):
    """beta 1 on all four configurations: raw numerator / denominator of both updates, the loss pass and the folded loss."""
    prec, N, C, R = case
    V, W, H = _data(N, C, R, seed=N * 7 + C + R)
    eng = _engine(prec, V, W, H)
    assert eng.precision_for(1) == prec
    model = tcm.NmfModel(V.cuda(), W.cuda(), H.cuda(), prec)
    ora = OracleNmfEngine(V.double(), W.double(), H.double())
    for which in (0, 1):
        num, den = eng.raw_terms(which, 1)
        mnum, mden, bar, _ = model.raw_terms(which, 1, nchunks=_nchunks(prec, N, C, R, which))
        enum, eden = ora.raw_terms(which, 1)
        _check_terms(f"kl-raw{which}-{_id(case)}", num, mnum, bar, enum, RTOL64[prec])
        assert torch.allclose(den.double().cpu(), eden.reshape(-1), rtol=1e-5), "beta 1 denominator: column sums"
    exact = ora.loss(1)
    _check_loss(f"kl-loss-{_id(case)}", eng.loss(1), model.loss(1), exact, prec, 1)
    fold = prec == "f16"                       # the split mode evaluates loss_prefetch_w with the loss pass
    _check_loss(f"kl-fold-{_id(case)}", eng.loss_prefetch_w(1), model.loss(1, fold=fold), exact, prec, 1)
    eng.close()


@pytest.mark.parametrize("case", STRUCT_CASES, ids=_id)
def test_nmf_split_terms_on_structured_inputs(case):
    """beta 1 raw terms of the split configurations on _structured_data, where dropping any of the three split terms
    (Flo Ghi, Fhi Glo in S; P Glo in O) moves the numerator by 3 to 10 times the model bar (tests/test_tc_model.py).
    Against float64 these cases are held to the fast mode's bar: a handful of hot terms carries each sum, and their ratio
    tile rounding (up to 2^-11 each) does not average out."""
    prec, N, C, R = case
    V, W, H = _structured_data(N, C, R, seed=N + C + R)
    eng = _engine(prec, V, W, H)
    assert eng.precision_for(1) == prec
    model = tcm.NmfModel(V.cuda(), W.cuda(), H.cuda(), prec)
    ora = OracleNmfEngine(V.double(), W.double(), H.double())
    for which in (0, 1):
        num, _ = eng.raw_terms(which, 1)
        mnum, _, bar, _ = model.raw_terms(which, 1, nchunks=_nchunks(prec, N, C, R, which))
        _check_terms(f"split-struct-raw{which}-{_id(case)}", num, mnum, bar, ora.raw_terms(which, 1)[0], RTOL64["f16"])
    eng.close()


@pytest.mark.parametrize("case", NMF_CASES[::2] + NMF_CASES[1::4], ids=_id)
def test_nmf_eu_updates_and_loss(case):
    """beta 2 (the residual kernel; no tensor-core raw terms): one W update, then one H update from the new W, each
    against the model's numerator / denominator through the ratio stage; and the loss."""
    prec, N, C, R = case
    V, W, H = _data(N, C, R, seed=N + 3 * C + R)
    eng = _engine(prec, V, W, H)
    assert eng.precision_for(2) == prec
    exact = orc.beta_div(orc.nmf_reconstruct(H.double(), W.double()), V.double(), 2).item()
    _check_loss(f"eu-loss-{_id(case)}", eng.loss(2), tcm.NmfModel(V.cuda(), W.cuda(), H.cuda(), prec).loss(2), exact, prec, 2)
    for which in (0, 1):
        Wc, Hc = eng.W.clone(), eng.H.clone()
        model = tcm.NmfModel(V.cuda(), Wc, Hc, prec)
        num, den, bar, _ = model.raw_terms(which, 2, nchunks=_nchunks(prec, N, C, R, which))
        enum, eden, _, _ = tcm.NmfModel(V.cuda(), Wc, Hc, prec, rounding=False).raw_terms(which, 2)
        (eng.update_w if which == 0 else eng.update_h)(2, 1.0, 0.0, 0.0)
        old = (Wc if which == 0 else Hc).double()
        got = (eng.W if which == 0 else eng.H).double()

        def upd(n, d):
            return old * (n.clamp_min(0) + tcm.EPS) / (d.clamp_min(0) + tcm.EPS)
        want, want64 = upd(num, den), upd(enum, eden)
        # the ratio stage's fp32 Gram (<= 72 ulp), its product with F (R ulp), num + kappa den and the division (8 ulp)
        ratio_bar = tcm.U * (R + 80) * (1 + model.kappa * den.abs() / num.abs())
        _check_terms(f"eu-upd{which}-{_id(case)}", got, want, want * (bar / num.abs() + ratio_bar), want64, RTOL64[prec])
    eng.close()


@pytest.mark.parametrize("beta", TWO_BETAS)
@pytest.mark.parametrize("case", [c for c in NMF_CASES if c[3] <= 64] + CHUNK_CASES[:2], ids=_id)
def test_nmf_two_output_terms_and_loss(case, beta):
    """beta not in {1, 2}: the two-output kernel (hi halves of the operand copies, rank <= 64) in both orientations, and
    the loss pass (which uses the full split product in split mode, with the out-of-range rows / columns masked)."""
    prec, N, C, R = case
    # factors in [0.5, 1.5): at rank 1 with factors in [0.1, 1.1), V x^(beta - 2) spans more than the fp16 range under the
    # tile's one power-of-two scale (beta -1: 1e8) and the kernel loses the small entries, as the model does
    V, W, H = _data(N, C, R, seed=N + C + 5 * R, vmin=0.01, fmin=0.5)
    eng = _engine(prec, V, W, H)
    assert eng.precision_for(beta) == "f16"
    model = tcm.NmfModel(V.cuda(), W.cuda(), H.cuda(), prec)
    ora = OracleNmfEngine(V.double(), W.double(), H.double())
    for which in (0, 1):
        num, den = eng.raw_terms(which, beta)
        mnum, mden, bar, dbar = model.raw_terms(which, beta, nchunks=_nchunks(prec, N, C, R, which))
        enum, eden = ora.raw_terms(which, beta)
        _check_terms(f"b{beta}-num{which}-{_id(case)}", num, mnum, bar, enum, RTOL64["f16"] * max(1, abs(beta - 2)))
        _check_terms(f"b{beta}-den{which}-{_id(case)}", den, mden, dbar, eden, RTOL64["f16"] * max(1, abs(beta - 1)))
    _check_loss(f"b{beta}-loss-{_id(case)}", eng.loss(beta), model.loss(beta), ora.loss(beta), prec, beta)
    eng.close()


@pytest.mark.parametrize("beta", [0.5, 3])
@pytest.mark.parametrize("prec", ["f16", "f16_split"])
def test_nmf_two_output_beta_above_rank_64_falls_back_to_fp32(prec, beta):
    """R > 64 with a two-output beta has no tensor-core kernel: the engine says so and the fp32 kernels still match."""
    N, C, R = 321, 193, 100
    V, W, H = _data(N, C, R, seed=11, vmin=0.01)
    eng = _engine(prec, V, W, H)
    assert eng.precision_for(beta) == "f32"
    ora = OracleNmfEngine(V.double(), W.double(), H.double())
    for which in (0, 1):
        for got, want in zip(eng.raw_terms(which, beta), ora.raw_terms(which, beta)):
            # fp32 sums of <= 321 positive terms: a few ulp per term in the worst case, 1e-5 relative
            err = float(((got.double().cpu() - want) / want).abs().max())
            assert err <= 1e-5, (which, err)
    eng.close()


def test_chunk_cases_hit_a_short_last_chunk():
    """The chunked cases above are what they claim on this device: more than one chunk, the last one short."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for prec, N, C, R in CHUNK_CASES:
        rows, cols = (C, N) if N > C else (N, C)          # the orientation whose contracted side is long
        rb, tiles, nch, tpc = _plan(rows, cols, sms, _tn(prec, R))
        assert nch > 1 and tiles - (nch - 1) * tpc < tpc, (prec, N, C, R, rb, tiles, nch, tpc)


# ---- NMFD (beta 1, the sliding-GEMM kernels) --------------------------------------------------------------------------------
# (B, C, L, R, T): T in {1, 2, 63, 64, 65, 127, 128, 129, 200}, R in {1, 5, 16, 128, 129, 160, 256}, C in {1, 127, 128,
# 129}, B in {1, 3}, L = T and L ragged against 64 and 128; R T and C T kept small enough for the model bar to stay tight
NMFD_CASES = [
    (1, 1, 200, 1, 200),        # T > 128, L = T (Lin = 1), C = 1
    (3, 12, 333, 5, 200),       # T > 128, B = 3, split wgrad and dgrad
    (1, 31, 300, 16, 129),      # T = 129
    (1, 20, 257, 3, 128),       # T = 128, L = 2 x 128 + 1
    (3, 17, 191, 7, 127),
    (1, 127, 130, 1, 65),
    (1, 128, 64, 5, 64),        # L = T = 64
    (3, 129, 127, 16, 63),
    (1, 40, 200, 128, 2),       # R = 128: one dgrad slice
    (1, 33, 150, 129, 2),       # R = 129: a second slice of one component
    (3, 9, 100, 160, 1),
    (1, 24, 96, 256, 8),        # R = 256: two full slices
    (3, 43, 400, 2, 3),         # ws_w = 2 and ws_h = 5, both with a short last split
]


def _nmfd_data(B, C, L, R, T, seed):
    # a target bounded away from zero: where a sum has a single term (L = T) the centred numerator (P - kappa) G + kappa G
    # is only good to u kappa / P relative, which a V near zero would turn into the bar of the case
    g = torch.Generator().manual_seed(seed)
    V = torch.rand(B, C, L, generator=g) + 0.1
    W = torch.rand(C, R, T, generator=g) + 0.1
    H = torch.rand(B, R, L - T + 1, generator=g) + 0.1
    return V, W, H


@pytest.mark.parametrize("case", NMFD_CASES, ids=_id)
def test_nmfd_terms_and_loss(case):
    B, C, L, R, T = case
    V, W, H = _nmfd_data(*case, seed=sum(case))
    eng = CudaNmfdEngine(V.cuda(), W.cuda().clone(), H.cuda().clone(), "f16")
    assert eng.precision_for(1) == "f16"
    model = tcm.NmfdModel(V.cuda(), W.cuda(), H.cuda())
    ora = OracleNmfdEngine(V.double(), W.double(), H.double())
    ws_w, _, _, ws_h, _, _ = _nmfd_splits(*case)
    rtol64 = nmfd_rtol64(case, V, W, H)
    for which, ns in ((0, ws_w), (1, ws_h)):
        num, den = eng.raw_terms(which, 1)
        mnum, mden, bar = model.raw_terms(which, nchunks=ns)
        enum, eden = ora.raw_terms(which, 1)
        _check_terms(f"nmfd-raw{which}-{_id(case)}", num, mnum, bar, enum, rtol64)
        assert torch.allclose(den.double().cpu(), eden.reshape(-1), rtol=1e-5), "beta 1 denominator: column sums"
    _check_loss(f"nmfd-loss-{_id(case)}", eng.loss(1), model.loss(), ora.loss(1), "f16", 1)
    eng.close()


def test_nmfd_split_case_has_short_last_splits():
    ws_w, kbs_w, last_w, ws_h, kbs_h, last_h = _nmfd_splits(*NMFD_CASES[-1])
    assert ws_w > 1 and last_w < kbs_w and ws_h > 1 and last_h < kbs_h


def test_nmfd_fit_with_kernel_wider_than_128_shifts_matches_oracle():
    """A T = 200 fit on the tensor-core path against the oracle at the north-star bar (rtol 1e-3, atol 1e-5 max)."""
    V, W0, H0 = _nmfd_data(1, 20, 300, 4, 200, seed=200)
    W, H, _, _ = orc.fit(V, W0, H0, beta=1, tol=float("-inf"), max_iter=10, kind="nmfd")
    m = NMFD(W=W0, H=H0).cuda()
    m.fit(V.cuda(), 1, float("-inf"), 10, precision="f16")
    assert m.last_fit_precision == "f16"
    for got, want in ((m.W.data.cpu(), W), (m.H.data.cpu(), H)):
        atol = 1e-5 * float(want.abs().max())
        err = float(((got - want).abs() / (1e-3 * want.abs() + atol)).max())
        assert err <= 1.0, f"{err:.2f} x the north-star tolerance"
