"""The fp32 kernel cases of tests/test_gpu_f32_terms.py reach every tile plan they claim, asked of the library's own planners
(nmfb200_nmf_plan / nmfb200_nmfd_plan: host only, no device needed); every exact case is exact by a bound below 2^24; and the
float64 bars of the other cases hold for fp32 arithmetic on the CPU and are not vacuous.
"""
import math

import pytest
import torch

import f32_cases as fc
import sparse_cases as sc
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


# ---- sparse-target kernels (tests/sparse_cases.py, tests/test_gpu_sparse_terms.py) ------------------------------------------
def sparse_branches(cases):
    hit = set()
    for N, C, R, kind in cases:
        p = _capi.sparse_plan(N, C, R)
        hit |= {f"rpl={p['rpl']}", f"gram passes={p['gram_passes']}", f"pattern {kind}"}
        if (N, C) == (800, 800):
            hit.add(f"800x800 R={R}")
        if kind == "lines" and max(N, C) > 1024:
            hit.add("segment longer than 1024")
        for side, rows, rpb, nb, gb in (("N", N, p["rpb_n"], p["nb_n"], p["gather_blocks_n"]),
                                        ("C", C, p["rpb_c"], p["nb_c"], p["gather_blocks_c"])):
            assert gb == cdiv(rows, 8) and nb <= 128 and rpb % 32 == 0 and (nb - 1) * rpb < rows <= nb * rpb
            if rows % 8 in (0, 1, 7):
                hit.add(f"gather tail {side}%8={rows % 8}")
            last = rows - (nb - 1) * rpb
            if nb == 1 and rows < 32:
                hit.add(f"Gram one partial slab ({side})")
            if nb == 2 and rpb == 32 and last == 1:
                hit.add(f"Gram 2 blocks, 1 row in the last ({side})")
            if nb == 128 and rpb == 32 and last == 32:
                hit.add(f"Gram 128 blocks of 32 rows ({side})")
            if rpb == 64 and last == 1:
                hit.add(f"Gram rpb 64, 1-row last block ({side})")
            if rpb == 64 and last == 63:
                hit.add(f"Gram rpb 64, 63-row last block, short last slab ({side})")
    return hit


SPARSE_REQUIRED = ({f"rpl={r}" for r in (1, 2, 4, 8)} | {f"gram passes={n}" for n in (1, 2, 3, 4, 5, 10, 16)}
                   | {f"pattern {k}" for k in ("random", "edges", "lines", "empty")}
                   | {"800x800 R=64", "800x800 R=200", "segment longer than 1024"}
                   | {f"gather tail {s}%8={t}" for s in "NC" for t in (0, 1, 7)}
                   | {f"Gram {k} ({s})" for s in "NC" for k in ("one partial slab", "2 blocks, 1 row in the last",
                                                               "128 blocks of 32 rows", "rpb 64, 1-row last block",
                                                               "rpb 64, 63-row last block, short last slab")})


def test_sparse_cases_cover_every_plan_branch():
    miss = _missing(SPARSE_REQUIRED, sparse_branches(sc.SPARSE_EXACT))
    assert not miss, miss
    assert {1, 31, 32, 33, 64, 65, 96, 128, 129, 200, 256} <= {c[2] for c in sc.SPARSE_EXACT}
    sizes = {1, 7, 8, 9, 31, 32, 33, 4096, 4097, 8191}
    assert sizes <= {c[0] for c in sc.SPARSE_EXACT} and sizes <= {c[1] for c in sc.SPARSE_EXACT}
    assert {f"rpl={r}" for r in (1, 2, 4, 8)} | {"gram passes=16"} <= sparse_branches(sc.SPARSE_BAR)
    assert all(c in sc.SPARSE_EXACT for c in sc.SPARSE_RATIO), "the ratio stage runs on exact raw terms"
    cut = [c for c in sc.SPARSE_EXACT if c[0] != 8191 and c[1] != 8191]
    assert {"Gram rpb 64, 63-row last block, short last slab (N)",
            "Gram rpb 64, 63-row last block, short last slab (C)"} <= set(_missing(SPARSE_REQUIRED, sparse_branches(cut)))
    cut = [c for c in sc.SPARSE_EXACT if c[2] <= 128]
    assert {"rpl=8", "gram passes=10", "gram passes=16"} <= set(_missing(SPARSE_REQUIRED, sparse_branches(cut)))


def test_sparse_plan_matches_its_formulas():
    for R, rpl, passes in ((1, 1, 1), (32, 1, 1), (33, 2, 1), (64, 2, 1), (65, 4, 2), (128, 4, 4), (129, 8, 5), (256, 8, 16)):
        p = _capi.sparse_plan(5, 6, R)
        assert (p["rpl"], p["gram_passes"]) == (rpl, passes), R
    p = _capi.sparse_plan(8191, 4097, 7)
    assert (p["rpb_n"], p["nb_n"], p["rpb_c"], p["nb_c"]) == (64, 128, 64, 65)
    with pytest.raises(_capi.NmfB200Error):
        _capi.sparse_plan(5, 6, 257)


@pytest.mark.parametrize("case", sc.SPARSE_EXACT, ids=str)
def test_sparse_exact_bounds(case):
    N, C, R, kind = case
    f = sc.sparse_range(N, C, R)
    assert sc.sparse_eu_bound(N, C, R, f, f * f) < fc.EXACT
    assert sc.sparse_kl_bound(N, C, R) < fc.EXACT
    rows, cols, vals, W, H = sc.sparse_eu_data(case, seed=1)
    assert sc.sparse_eu_loss_bound(N, C, R, f, f * f, rows.numel()) < sc.EXACT_DOUBLE
    assert float(W.max()) <= f and float(H.max()) <= f and (not vals.numel() or float(vals.max()) <= f * f)
    assert rows.numel() <= sc.MAX_NNZ + N + C
    if kind == "empty":
        assert rows.numel() == 0
    if kind == "edges":
        assert not ({0, N - 1} & set(rows.tolist())) and not ({0, C - 1} & set(cols.tolist()))
    rows, cols, vals, W, H, Q = sc.sparse_kl_data(case, seed=3)
    d = sc.dots(rows, cols, W.double(), H.double())
    assert torch.equal(vals.double(), Q.double() * d)
    if rows.numel():
        assert float(d.min()) >= 4 and bool(((d.float() + orc.EPS) == d.float()).all())
        assert torch.equal(vals / (d.float() + orc.EPS), Q), "fp32 v / (dot + eps) is q"


def test_sparse_cases_store_explicit_zeros():
    """Stored zero values reach the kernels in the exact data of both betas (a zero v still occupies its slot)."""
    for case in sc.SPARSE_EXACT[:10]:
        for vals in (sc.sparse_eu_data(case, seed=1)[2], sc.sparse_kl_data(case, seed=3)[2]):
            assert vals.numel() < 100 or bool((vals == 0).any()), case
    S = sc.sparse_tensor(3, 3, torch.tensor([0, 2]), torch.tensor([1, 2]), torch.tensor([0.0, 1.0]))
    assert S._nnz() == 2


@pytest.mark.parametrize("beta", [1, 2])
@pytest.mark.parametrize("case", [(9, 32, 33, "random"), (31, 33, 64, "edges"), (200, 150, 17, "lines")], ids=str)
def test_sparse_restatement_is_the_reference(case, beta):
    """The float64 restatement of nmf.py:603-638 at the non-zeros equals the dense reference: loss = beta_div(H W^T, V)
    up to the eps of log(v + eps) (at most eps per stored positive value), and the terms equal the dense gradients."""
    N, C, R, _ = case
    rows, cols, vals, W, H = sc.sparse_bar_data(case, seed=11)
    vals[::7] = 0.0                                                  # stored zeros
    W, H = W.double(), H.double()
    V = sc.sparse_tensor(N, C, rows, cols, vals.double()).to_dense()
    got = sc.sp_loss64(beta, rows, cols, vals, W, H)
    want = float(orc.beta_div(H @ W.t(), V, beta))
    slack = (rows.numel() * orc.EPS if beta == 1 else 0.0) + 1e-12 * abs(want)
    assert abs(got - want) <= slack, (got, want)
    Pn, Pp = orc.phi(V, H @ W.t(), beta)
    for which in (0, 1):
        for g, w in zip(sc.sp_terms64(which, beta, rows, cols, vals, W, H), fc.nmf_terms64(which, Pn, Pp, W, H)):
            assert torch.allclose(g, w, rtol=1e-12, atol=0), which


def _gram32(F, rpb, nb):
    """F^T F in fp32 in the kernel's grouping: 32-row slabs, summed in order within each block of rpb rows, then the blocks."""
    out = torch.zeros(F.shape[1], F.shape[1])
    for b in range(nb):
        acc = torch.zeros_like(out)
        for r in range(b * rpb, min(F.shape[0], (b + 1) * rpb), 32):
            s = F[r:r + 32]
            acc += s.t() @ s
        out += acc
    return out


def _sp_terms32(which, beta, rows, cols, vals, W, H, plan):
    num, den = sc.sp_terms64(which, beta, rows, cols, vals, W, H)
    if beta == 2:
        F, O, key = (W, H, "n") if which == 0 else (H, W, "c")
        den = F @ _gram32(O, plan[f"rpb_{key}"], plan[f"nb_{key}"])
    return num, den


def _rel(got, want):
    """Relative error per entry; an entry whose reference is 0 must be 0."""
    assert bool((got[want == 0] == 0).all())
    return (got.double() - want).abs() / want.abs().clamp_min(1e-300)


@pytest.mark.parametrize("beta", [1, 2])
@pytest.mark.parametrize("case", sc.SPARSE_BAR, ids=str)
def test_sparse_bars_hold_for_fp32_and_catch_one_dropped_term(case, beta):
    """fp32 arithmetic on the CPU (the Gram in the kernel's grouping) stays inside the float64 bars; dropping the last stored
    entry of a segment of up to 64 entries, or the last row of a Gram sum, exceeds them."""
    N, C, R, _ = case
    rows, cols, vals, W, H = sc.sparse_bar_data(case, seed=N + C + R)
    plan = _capi.sparse_plan(N, C, R)
    W64, H64 = W.double(), H.double()
    order = torch.argsort(cols * N + rows)
    for which in (0, 1):
        n = sc.seg_lengths(which, rows, cols, N, C)
        want = sc.sp_terms64(which, beta, rows, cols, vals, W64, H64)
        got = _sp_terms32(which, beta, rows, cols, vals, W, H, plan)
        nbar = sc.num_bar(beta, R, n)[:, None]
        assert bool((_rel(got[0], want[0]) <= nbar).all()), which
        if beta == 2:
            rpb, nb = (plan["rpb_n"], plan["nb_n"]) if which == 0 else (plan["rpb_c"], plan["nb_c"])
            dbar = sc.den_bar(R, rpb, nb)
            assert float(_rel(got[1], want[1]).max()) <= dbar, which
            O = H64 if which == 0 else W64
            cut = (W64 if which == 0 else H64) @ (O[:-1].t() @ O[:-1])
            assert float(((cut - want[1]).abs() / want[1]).min()) > dbar, "a dropped Gram row shows"
        # the last stored entry of every segment dropped
        keep = torch.ones(rows.numel(), dtype=torch.bool)
        ends = torch.cumsum(n, 0)[n > 0] - 1
        keep[(order[ends] if which == 0 else ends)] = False
        cut = sc.sp_terms64(which, beta, rows[keep], cols[keep], vals[keep], W64, H64)[0]
        short = (n > 0) & (n <= 64)
        if bool(short.any()):
            assert bool(((cut[short] - want[0][short]).abs() / want[0][short] > nbar[short]).all()), which
    assert bool((sc.seg_lengths(1, rows, cols, N, C) <= 64).any() | (sc.seg_lengths(0, rows, cols, N, C) <= 64).any())


@pytest.mark.parametrize("beta", [1, 2])
@pytest.mark.parametrize("case", sc.SPARSE_BAR, ids=str)
def test_sparse_loss_bar_holds_for_fp32(case, beta):
    N, C, R, _ = case
    rows, cols, vals, W, H = sc.sparse_bar_data(case, seed=N + C + R)
    want = sc.sp_loss64(beta, rows, cols, vals, W.double(), H.double())
    bar = sc.loss_bar(beta, rows, cols, vals, W.double(), H.double())
    d = sc.dots(rows, cols, W, H)                                       # fp32 pieces, double sums
    if beta == 2:
        pos = 0.5 * float((_gram32(W, 32, cdiv(C, 32)).double() * _gram32(H, 32, cdiv(N, 32)).double()).sum())
        neg = float((vals * d).double().sum())
    else:
        pos = float(W.sum(0).double() @ H.sum(0).double())
        neg = float((vals * (d + orc.EPS).log()).double().sum())
    got = sc.v_norm(vals, beta) + pos - neg
    assert abs(got - want) <= bar, (got, want, bar)
    if case == sc.SPARSE_BAR[0]:
        # on a small case one stored entry is above the bar: a dropped or duplicated non-zero shows
        lost = sc.sp_loss64(beta, rows[1:], cols[1:], vals[1:], W.double(), H.double())
        assert abs(lost - want) > bar, (lost, want, bar)
