"""The tensor-core NMF contraction's launch plan (nmfb200_nmf_tc_plan) against tests/tc_model.py's mirror of make_plan, the
shared-memory layouts of its four configurations, and the walk state each case of tests/tc_walk_cases.py reaches -- all
without a GPU."""
import pytest
import torch

import tc_model as tcm
import tc_walk_cases as wc
import test_gpu_tc_terms as gt
from torchnmf_b200 import _capi
from torchnmf_b200._capi import NmfB200Error

TERM_SHAPES = sorted(set(gt.NMF_CASES + gt.CHUNK_CASES + gt.STRUCT_CASES))
WALK_SHAPES = sorted({(c["prec"], c["N"], c["C"], c["R"]) for S in wc.SM_COUNTS for c in wc.cases(S)})


def _id(c):
    return "-".join(str(x) for x in c)


@pytest.mark.parametrize("S", wc.SM_COUNTS)
@pytest.mark.parametrize("shape", TERM_SHAPES + WALK_SHAPES, ids=_id)
def test_plan_query_is_the_mirror(shape, S):
    """tc_model.plan and tc_model.tn, which the term tests take their chunk counts from, are what the library plans."""
    prec, N, C, R = shape
    got = _capi.nmf_tc_plan(N, C, R, prec, S)
    assert got == wc.mirror_plan(N, C, R, prec, S)
    assert got["tn"] == tcm.tn(prec, R)
    for which, (rows, cols) in ((0, (C, N)), (1, (N, C))):
        pl = wc.side(got, which)
        assert (pl["row_blocks"], pl["tiles"], pl["nchunks"], pl["tpc"]) == tcm.plan(rows, cols, S, tcm.tn(prec, R))
        assert pl["items"] == pl["row_blocks"] * pl["nchunks"] and pl["grid"] == min(pl["items"], S)


@pytest.mark.parametrize("prec,R", [(p, r) for p in ("f16", "f16_split") for r in (1, 40, 64, 65, 100, 128)])
def test_shared_memory_layouts(prec, R):
    """TN, NS and NF of the configuration serving (precision, rank): only the fast rank-64 kernel has two F slots."""
    p = _capi.nmf_tc_plan(1000, 1000, R, prec, 132)
    assert (p["tn"], p["ns"], p["nf"]) == wc.layout(prec, R)
    want = {("f16", 64): (128, 4, 2), ("f16_split", 64): (128, 3, 1), ("f16", 128): (128, 3, 1),
            ("f16_split", 128): (64, 3, 1)}[(prec, 64 if R <= 64 else 128)]
    assert (p["tn"], p["ns"], p["nf"]) == want


def test_auto_plans_as_f16():
    assert _capi.nmf_tc_plan(300, 200, 40, "auto", 132) == _capi.nmf_tc_plan(300, 200, 40, "f16", 132)


@pytest.mark.parametrize("args", [
    (300, 200, 40, "f32", 132),                 # no tensor-core kernel
    (300, 200, 0, "f16", 132), (300, 200, 129, "f16", 132), (300, 200, 129, "auto", 132),
    (0, 200, 40, "f16", 132), (300, 0, 40, "f16_split", 132), (300, 200, 40, "f16", 0),
    (65535 * 64 + 1, 8, 4, "f16", 132),         # past the conversion kernel's row limit: create takes f32 only
], ids=str)
def test_plan_query_refuses(args):
    with pytest.raises(NmfB200Error):
        _capi.nmf_tc_plan(*args)


def test_plan_query_is_host_only():
    """No device, no allocation: the query answers for any SM count, on a machine without a GPU too."""
    assert _capi.nmf_tc_plan(65535 * 64, 8, 4, "f16", 1)["grid_h"] == 1
    assert _capi.nmf_tc_plan(65535 * 64, 8, 4, "f16", 100000)["grid_h"] == 32768


@pytest.mark.parametrize("S", wc.SM_COUNTS)
@pytest.mark.parametrize("i", range(len(wc.cases(132))))
def test_catalogue_reaches_its_walk_state(i, S):
    """From the library's plan: the walked orientation's busiest CTA walks at least 2 NF + 1 items (each F slot flips its
    phase and comes back), the items do not divide evenly over the CTAs, the period prime does not divide the grid, the
    tiles of an item are not a multiple of NS and the last tile is short; chunked cases have a short last chunk that CTAs
    alternate with full ones."""
    c = wc.cases(S)[i]
    p = _capi.nmf_tc_plan(c["N"], c["C"], c["R"], c["prec"], S)
    pl = wc.side(p, c["which"])
    cols = c["C"] if c["which"] == 1 else c["N"]
    w = wc.walk_state(pl, p["ns"], p["nf"], c["P"], p["tn"], cols)
    assert pl["grid"] == S and pl["grid"] % c["P"] != 0 and c["P"] == wc.period_prime(S)
    assert w["max_items"] >= 2 * p["nf"] + 1 and w["slot_back_to_phase0"], w
    assert w["uneven"] and w["min_items"] < w["max_items"], w
    assert pl["tpc"] % p["ns"] != 0 and w["short_last_tile"] and w["item_inside_ring"], w
    assert w["distinct_consecutive_f"], w
    if c["kind"] == "chunked":
        assert pl["nchunks"] > 1 and w["short_last_chunk"] and w["alternating_chunk_lengths"], w
    else:
        assert pl["nchunks"] == 1 and (c["N"] if c["which"] == 1 else c["C"]) % 128 == 65
    if c["kind"] in ("tall", "wide"):
        assert pl["items"] == 4 * S + 5 and (w["max_items"], w["min_items"]) == (5, 4)


def test_chunked_case_at_132_sms():
    """At 132 SMs: 141 row blocks over 7 chunks of 5 tiles, the last of 3, 987 items, up to 8 on a CTA."""
    c = wc.case(132, "chunked", "f16", 64)
    pl = wc.side(_capi.nmf_tc_plan(c["N"], c["C"], c["R"], c["prec"], 132), 1)
    assert (pl["row_blocks"], pl["nchunks"], pl["tpc"], pl["tiles"] - 6 * pl["tpc"], pl["items"]) == (141, 7, 5, 3, 987)
    assert wc.walk_state(pl, 4, 2, c["P"], 128, c["C"])["max_items"] == 8


@pytest.mark.parametrize("kind", ["tall", "wide", "chunked"])
def test_periodic_data(kind):
    """Walked factor rows and the matching rows / columns of V repeat their first 128 P rows exactly."""
    c = dict(wc.case(132, kind, "f16", 64))
    per = 128 * c["P"]
    c["N" if c["which"] == 1 else "C"] = 3 * per + 65            # a smaller copy of the case: the same layout
    V, W, H = wc.periodic_data(c, seed=3)
    F, Vm = (W, V.t()) if c["which"] == 0 else (H, V)
    for X in (F, Vm):
        assert torch.equal(X, X[torch.arange(X.shape[0]) % per])
        assert not torch.equal(X[:128], X[128:256])              # consecutive row blocks differ
    lo = 1 - 2.0 ** -20                                          # the fp32 offsets sit just below 0.05, 0.1, 0.01
    assert float(V.min()) >= 0.05 * lo and float(F.min()) >= 0.1 * lo
    V2, W2, H2 = wc.periodic_data(c, seed=3, two_output=True)
    assert float(V2.min()) >= 0.01 * lo and float(min(W2.min(), H2.min())) >= 0.5 and float(max(W2.max(), H2.max())) < 1.5


@pytest.mark.parametrize("chunks", [1, 3])
def test_period_breaks_flags_one_ulp(chunks):
    """The periodicity check finds a one-ulp change in one row of one period and names the items, CTAs and walk
    positions that produced the row."""
    per, rows, grid = 128 * 5, 128 * 17 + 65, 4
    pl = {"row_blocks": -(-rows // 128), "nchunks": chunks, "grid": grid}
    g = torch.Generator().manual_seed(0)
    X = (torch.rand(per, 40, generator=g) + 0.1).repeat(4, 1)[:rows].contiguous()
    assert wc.period_breaks(X, per, pl) == []
    r = 2 * per + 3 * 128 + 17                                   # row block 13
    Y = X.clone()
    Y[r, 11] = torch.nextafter(Y[r, 11], torch.tensor(2.0))
    bad = wc.period_breaks(Y, per, pl)
    assert len(bad) == 1
    b = bad[0]
    items = [ch * pl["row_blocks"] + 13 for ch in range(chunks)]
    assert b["row"] == r and b["representative"] == 3 * 128 + 17 and b["items"] == items
    assert b["ctas"] == [i % grid for i in items] and b["walk_positions"] == [i // grid for i in items]
    assert b["got"] != b["want"]
    with pytest.raises(AssertionError, match="first period"):
        wc.assert_periodic("t", Y, per, pl)
    # the last, short row block and float64 tensors too
    Z = X.double()
    Z[rows - 1, 0] += 2.0 ** -40
    assert [b["row"] for b in wc.period_breaks(Z, per, pl)] == [rows - 1]
