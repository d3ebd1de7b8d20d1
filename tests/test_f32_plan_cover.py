"""The fp32 kernel cases of tests/test_gpu_f32_terms.py reach every tile plan they claim, asked of the library's own planners
(nmfb200_nmf_plan / nmfb200_nmfd_plan: host only, no device needed); every exact case is exact by a bound below 2^24; and the
float64 bars of the other cases hold for fp32 arithmetic on the CPU and are not vacuous.
"""
import math

import pytest
import torch

import f32_cases as fc
from oracle import mu_oracle as orc
from torchnmf_b200 import _capi


def cdiv(a, b):
    return -(-a // b)


def _chunk_shape(tiles, nch, tpc):
    """'short' if the last chunk holds fewer tiles than the others, 'empty' if some chunks hold none."""
    out = set()
    if nch > 1 and (nch - 1) * tpc >= tiles:
        out.add("empty")
    elif nch > 1 and tiles - (nch - 1) * tpc < tpc:
        out.add("short")
    return out


def nmf_branches(cases):
    hit = set()
    for N, C, R in cases:
        p = _capi.nmf_plan(N, C, R)
        hit.add(f"rb={p['rb']}")
        if (N, C, R) == (1, 1, 1):
            hit.add("1x1x1")
        if R == 1:
            hit.add("rank 1")
        for side, rows, cols, nch, tpc in (("W", C, N, p["nch_w"], p["tpc_w"]), ("H", N, C, p["nch_h"], p["tpc_h"])):
            tiles = cdiv(cols, 64)
            hit.add(f"rows%64={rows % 64}" if rows % 64 in (0, 1, 63) else "rows other")
            hit.add(f"cols%64={cols % 64}" if cols % 64 in (0, 1, 63) else "cols other")
            if tiles <= 3:
                hit.add(f"{tiles} contracted tiles")
            for k in _chunk_shape(tiles, nch, tpc):
                hit.add(f"{k} chunk ({side} update)")
            if nch == 32:
                hit.add("32 chunks")
        nb = p["colsum_blocks_n"]
        if nb == 1024:
            rpb = cdiv(N, nb)
            last = N - (nb - 1) * rpb
            if 0 < last < rpb:
                hit.add("column sum over 1024 blocks, short last block")
    return hit


NMF_REQUIRED = ({f"rb={rb}" for rb in (1, 2, 4, 8, 16)} | {"1x1x1", "rank 1", "32 chunks",
                "column sum over 1024 blocks, short last block"}
                | {f"rows%64={r}" for r in (0, 1, 63)} | {f"cols%64={r}" for r in (0, 1, 63)}
                | {f"{t} contracted tiles" for t in (1, 2, 3)}
                | {f"{k} chunk ({s} update)" for k in ("short", "empty") for s in ("W", "H")})

NMFD_T = {1, 2, 31, 32, 33, 63, 64, 65, 128, 129, 200}


def _split_shape(n, ns):
    per = cdiv(n, ns)
    last = n - (ns - 1) * per
    return "empty" if last <= 0 else ("short" if ns > 1 and last < per else None)


def nmfd_branches(cases):
    hit = set()
    for case in cases:
        B, C, X, R, K, J = fc.nmfd_dims(case)
        p = _capi.nmfd_plan(B, C, list(X), R, list(K))
        w = p["wgrad"]
        L, T, Lin = X[-1], K[-1], J[-1]
        hit |= {f"recon MT={p['recon_mt']}", f"dgrad MT={p['dgrad_mt']}", f"B={B}"}
        if T in NMFD_T:
            hit.add(f"T={T}")
        if w["ntt"] > 1:
            hit.add("wgrad ntt>1")
        if T % 4:
            hit.add("T%4!=0 (tp rounds up)")
        if L % 64:
            hit.add("L%64!=0")
        if Lin % 64 and Lin > 1:
            hit.add("Lin%64!=0")
        if L == T:
            hit.add("L=T (Lin=1)")
        for k in ("nrg", "no", "nog"):
            if w[k] > 1:
                hit.add(f"wgrad {k}>1")
        shape = _split_shape(B * math.prod(J[:-1]), p["wgrad_nsplit"])
        if shape and p["wgrad_nsplit"] > 1:
            hit.add(f"wgrad {shape} last split")
        shape = _split_shape(C, p["dgrad_nsplit"])
        if shape and p["dgrad_nsplit"] > 1:
            hit.add(f"dgrad {shape} last split")
        if len(X) > 1:
            hit.add(f"{len(X)}D")
            if len(X) == 3 and K[0] == X[0]:
                hit.add("3D T1=X1 (J1=1)")
            if K[-2] > 1:
                hit.add(f"{len(X)}D T2>1")
            if math.prod(X[:-1]) % (64 // p["recon_mt"]):
                hit.add("recon lines not a multiple of XT")
            if math.prod(J[:-1]) % (64 // p["dgrad_mt"]):
                hit.add("dgrad lines not a multiple of XT")
    return hit


NMFD_REQUIRED = ({f"recon MT={m}" for m in (4, 8, 16, 32, 64)} | {f"dgrad MT={m}" for m in (4, 8, 16, 32, 64)}
                 | {f"T={t}" for t in NMFD_T} | {"B=1", "B=3", "wgrad ntt>1", "T%4!=0 (tp rounds up)", "L%64!=0",
                 "Lin%64!=0", "L=T (Lin=1)", "wgrad nrg>1", "wgrad no>1", "wgrad nog>1", "wgrad short last split",
                 "dgrad short last split", "wgrad empty last split", "dgrad empty last split", "2D", "3D",
                 "3D T1=X1 (J1=1)", "2D T2>1", "3D T2>1",
                 "recon lines not a multiple of XT", "dgrad lines not a multiple of XT"})


def ratio_branches(cases):
    hit = set()
    for kind, case in cases:
        if kind == "nmf":
            hit.add("NMF (scalar, inner 1)")
            continue
        B, C, X, R, K, J = fc.nmfd_dims(case)
        p = _capi.nmfd_plan(B, C, list(X), R, list(K))
        for side, inner, vec in (("W", math.prod(K), p["vec4_w"]), ("H", math.prod(J), p["vec4_h"])):
            assert vec == (inner % 4 == 0), (case, side)
            hit.add(f"NMFD {side} {'vec4' if vec else 'scalar'}")
            if inner % 4 == 2 and R % 2 == 0:
                hit.add("inner 2 mod 4, even rank")
    return hit


RATIO_REQUIRED = {"NMF (scalar, inner 1)", "NMFD W vec4", "NMFD W scalar", "NMFD H vec4", "NMFD H scalar",
                  "inner 2 mod 4, even rank"}


def _missing(required, hit):
    return sorted(required - hit)


def test_nmf_cases_cover_every_plan_branch():
    assert not _missing(NMF_REQUIRED, nmf_branches(fc.NMF_EXACT)), _missing(NMF_REQUIRED, nmf_branches(fc.NMF_EXACT))
    ranks = {R for _, _, R in fc.NMF_EXACT}
    assert {1, 16, 17, 32, 33, 64, 65, 128, 129, 200, 256} <= ranks
    assert fc.NMF_F16 and all(R <= 128 for _, _, R in fc.NMF_F16)
    assert "short chunk (H update)" in nmf_branches(fc.NMF_F16) and "32 chunks" in nmf_branches(fc.NMF_F16)


def test_nmfd_cases_cover_every_plan_branch():
    miss = _missing(NMFD_REQUIRED, nmfd_branches(fc.NMFD_EXACT))
    assert not miss, miss
    C = {c[1] for c in fc.NMFD_EXACT}
    R = {c[3] for c in fc.NMFD_EXACT}
    assert {1, 4, 5, 8, 9, 16, 17, 32, 33, 65, 129} <= C and {1, 4, 5, 9, 17, 33, 65, 129, 256} <= R
    assert fc.NMFD_LOSS and {"recon MT=4", "recon MT=64", "2D", "3D"} <= nmfd_branches(fc.NMFD_LOSS)


def test_ratio_cases_cover_both_kernels():
    miss = _missing(RATIO_REQUIRED, ratio_branches(fc.RATIO_CASES))
    assert not miss, miss
    exact = set(fc.NMF_EXACT) | set(fc.NMFD_EXACT)
    assert all(c in exact for _, c in fc.RATIO_CASES), "the ratio stage runs on exact raw terms"


def test_removing_a_category_names_the_missing_branch():
    """The coverage checks fail by name when a category of cases is left out."""
    cut = [c for c in fc.NMF_EXACT if c not in ((64, 2112, 17), (2112, 64, 200))]
    assert {"empty chunk (W update)", "empty chunk (H update)"} <= set(_missing(NMF_REQUIRED, nmf_branches(cut)))
    cut = [c for c in fc.NMFD_EXACT if len(c[2]) < 3]
    assert {"3D", "3D T1=X1 (J1=1)", "3D T2>1"} <= set(_missing(NMFD_REQUIRED, nmfd_branches(cut)))
    cut = [c for c in fc.NMFD_EXACT if c[4][-1] < 128]
    assert {"T=128", "T=129", "T=200"} <= set(_missing(NMFD_REQUIRED, nmfd_branches(cut)))


@pytest.mark.parametrize("case", fc.NMF_EXACT + fc.NMF_F16)
def test_nmf_exact_bounds(case):
    N, C, R = case
    f = fc.nmf_range(N, C, R)
    assert fc.nmf_bound(N, C, R, f, f * f) < fc.EXACT
    assert fc.nmf_kl_bound(N, C, R) < fc.EXACT
    f = fc.nmf_range(N, C, R, loss=True)
    assert fc.loss_bound(R * f * f, f * f) < fc.EXACT_LOSS
    V, W, H = fc.nmf_eu_data(N, C, R, seed=1, loss=True)
    assert float(V.max()) <= f * f and float(W.max()) <= f and float(H.max()) <= f and float(V.min()) >= 0


@pytest.mark.parametrize("case", fc.NMFD_EXACT, ids=str)
def test_nmfd_exact_bounds_and_kl_floor(case):
    f = fc.nmfd_range(case)
    assert fc.nmfd_bound(case, f, f * f) < fc.EXACT
    assert fc.nmfd_kl_bound(case) < fc.EXACT
    # a full convolution covers every position with at least one product of two factors >= 2: S >= 4 everywhere
    B, C, X, R, K, J = fc.nmfd_dims(case)
    assert all(x == j + k - 1 for x, j, k in zip(X, J, K))
    if B * C * math.prod(X) * fc.nmfd_terms(case)[0] <= 5e7:
        V, W, H, Q = fc.nmfd_kl_data(case, seed=3)
        S = fc.recon(H.double(), W.double())
        assert float(S.min()) >= 4 and torch.equal(V.double(), Q.double() * S)
        assert torch.equal(((S.float() + orc.EPS) == S.float()).all(), torch.tensor(True))


@pytest.mark.parametrize("case", [c for c in fc.NMF_EXACT if c[0] * c[1] * c[2] <= 5e7])
def test_nmf_kl_data_is_exact(case):
    V, W, H, Q = fc.nmf_kl_data(*case, seed=3)
    S = H.double() @ W.double().t()
    assert float(S.min()) >= 4 and torch.equal(V.double(), Q.double() * S)
    assert bool(((S.float() + orc.EPS) == S.float()).all())
    Pn = V / (S.float() + orc.EPS)
    assert torch.equal(Pn, Q), "fp32 v / (s + eps) is q"


# ---- float64 bars: fp32 arithmetic on the CPU stays inside them; one average term is above them where the sums are short ---
def _nmf_small(N, C, R, seed):
    return fc.bar_data((N, C), (C, R), (N, R), seed)


@pytest.mark.parametrize("beta", fc.TWO_BETAS)
@pytest.mark.parametrize("case", [(65, 129, 17), (1, 63, 1), (40, 70, 200)])
def test_term_bars_hold_for_fp32_on_the_cpu(case, beta):
    N, C, R = case
    V, W, H = _nmf_small(N, C, R, seed=N + C + R)
    for which, n in ((0, N), (1, C)):
        want = fc.nmf_terms64(which, *orc.phi(V.double(), H.double() @ W.double().t(), beta), W.double(), H.double())
        got = fc.nmf_terms64(which, *orc.phi(V, H @ W.t(), beta), W, H)
        for g, w, bar in zip(got, want, fc.terms_bar(beta, R, n, 1)):
            err = float(((g.double() - w).abs() / w.abs()).max())
            assert err <= bar, (which, err, bar)
            if n <= 200:
                # one average term of the shortest sums is well above the bar: dropping it cannot pass
                assert 1.0 / n > 10 * bar, (n, bar)


@pytest.mark.parametrize("beta", fc.LOSS_BETAS)
def test_loss_bars_hold_for_fp32_on_the_cpu(beta):
    N, C, R = 130, 70, 9
    V, W, H = _nmf_small(N, C, R, seed=5)
    want, bar = fc.loss_bar(beta, (H.double() @ W.double().t()).reshape(-1), V.double().reshape(-1), R, orc.EPS)
    got = float(orc.beta_div(H @ W.t(), V, beta))
    assert abs(got - want) <= bar, (got, want, bar)
    # and the bar is below the smallest term's contribution on average: a dropped row of 70 terms shows
    term, _ = fc.loss_pieces(beta, (H.double() @ W.double().t()).reshape(-1), V.double().reshape(-1), orc.EPS)
    assert bar < 70 * float(term.abs().mean()), (bar, float(term.abs().mean()))


def test_ratio_bar_holds_for_fp32_on_the_cpu():
    g = torch.Generator().manual_seed(9)
    p = torch.rand(4096, generator=g) + 0.01
    num = torch.randint(0, 5000, (4096,), generator=g).float()
    den = torch.randint(0, 5000, (4096,), generator=g).float()
    gamma = orc.gamma_of(0.5)
    got = orc._ratio_update(p, num, den, gamma, fc.RATIO_L1, fc.RATIO_L2, False)
    want, mult = fc.ratio64(p.double(), num.double(), den.double(), gamma, fc.RATIO_L1, fc.RATIO_L2, False)
    assert bool(((got.double() - want).abs() <= fc.ratio_bar(mult, gamma) * want).all())
