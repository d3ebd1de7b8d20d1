"""The tensor-core NMF contraction where every CTA walks several work items (cases: tests/tc_walk_cases.py), against exact
float64, against the float64 model of its rounding (tests/tc_model.py) and bit for bit across the walk.

tc_contract_kernel is persistent: CTA b walks items b, b + grid, ...  The F slot and its barrier parity, the stage ring's
counter, the ping-pong token of the two consumer warpgroups and the loss accumulators all carry over from one item to the
next.  The cases of tests/test_gpu_tc_terms.py give every CTA one item; here the walked orientation's busiest CTA walks at
least 2 NF + 1 items (both F slots of the fast rank-64 kernel come back to phase 0), the items do not divide evenly, item
boundaries fall inside the stage ring, and the chunked cases alternate full and short chunks.  Each case asserts that walk
state from the library's own plan (nmfb200_nmf_tc_plan) at this card's SM count.

Per case, on the walked update (H for tall and chunked, W for wide):
  * beta 1: the raw numerator through tc_model.check_terms (model bar and float64 bar RTOL64), the denominator (column
    sums) at rtol 1e-5, and the loss (tall, chunked: the loss pass; wide: the loss folded into the W update, which must then
    give the bits of a plain W update);
  * beta 2: one update through the ratio-stage bar of test_gpu_tc_terms.test_nmf_eu_updates_and_loss, and loss(2);
  * beta in {0, 0.5, 1.5, 3, -1} (tall, fast rank 64: the two-output kernels): numerator and denominator with the f16 bar
    times max(1, |exponent|), and the loss.
Every output row must equal its representative in the first period of the periodic data bit for bit.

Each case checks the card's free memory first and skips naming the shortfall; it prints one WALK JSON line with the plan,
the walk state, the peak device memory of its tensors and its wall time.
"""
import gc
import json
import time

import pytest
import torch

import tc_model as tcm
import tc_walk_cases as wc
from torchnmf_b200 import _capi
from torchnmf_b200.engine import CudaNmfEngine, release_workspaces

pytestmark = pytest.mark.gpu

TWO_BETAS = [0, 0.5, 1.5, 3, -1]
WALKS = [(k, p, r) for p, r in wc.CONFIGS for k in ("tall", "wide")] + [("chunked", "f16", r) for r in wc.CHUNK_RANKS]
# float64 N x C matrices alive at the peak of a case (V and its rounded copy in two models, S, P, the tile and the
# temporaries of flip_ulps), plus V and the engine's fp16 copies.  Measured on an H100 SXM (132 SMs): 5.4 to 5.9 GiB of
# torch allocations on the tall and wide cases, 9.6 GiB on the chunked ones (~137 bytes per cell); WALK lines print it.
BYTES_PER_CELL = 8 * 18 + 16


def _id(c):
    return "-".join(str(x) for x in c)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _need(c):
    nbytes = BYTES_PER_CELL * c["N"] * c["C"]
    torch.cuda.synchronize()
    free, _ = torch.cuda.mem_get_info()
    if free < nbytes:
        pytest.skip(f"needs {nbytes / 2**30:.1f} GiB of device memory, {free / 2**30:.1f} GiB free "
                    f"(short by {(nbytes - free) / 2**30:.1f} GiB)")


def _cleanup():
    release_workspaces()
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


class _Case:
    """One catalogue case on this card: its data on the device, the engine, both models, and the walk its plan reaches."""

    def __init__(self, kind, prec, R, seed, two_output=False):
        S = _sms()
        self.c = wc.case(S, kind, prec, R)
        c = self.c
        _cleanup()
        _need(c)
        torch.cuda.reset_peak_memory_stats()
        self.t0 = time.time()
        p = _capi.nmf_tc_plan(c["N"], c["C"], c["R"], c["prec"], S)
        self.pl = wc.side(p, c["which"])
        cols = c["C"] if c["which"] == 1 else c["N"]
        self.walk = wc.walk_state(self.pl, p["ns"], p["nf"], c["P"], p["tn"], cols)
        w = self.walk
        # the walk state this case exists for
        assert self.pl["grid"] == S and S % c["P"] != 0
        assert w["max_items"] >= 2 * p["nf"] + 1 and w["uneven"] and w["item_inside_ring"], w
        assert self.pl["tpc"] % p["ns"] != 0 and w["short_last_tile"] and w["distinct_consecutive_f"], w
        if kind == "chunked":
            assert w["short_last_chunk"] and w["alternating_chunk_lengths"], w
        self.plan = p
        self.which = c["which"]
        self.period = 128 * c["P"]
        V, W, H = wc.periodic_data(c, seed, two_output)
        self.V, self.W0, self.H0 = V.cuda(), W.cuda(), H.cuda()
        self.eng = CudaNmfEngine(self.V, self.W0.clone(), self.H0.clone(), prec)
        self.tag = c["name"]

    def models(self, W=None, H=None):
        W = self.W0 if W is None else W
        H = self.H0 if H is None else H
        return (tcm.NmfModel(self.V, W, H, self.c["prec"]),
                tcm.NmfModel(self.V, W, H, self.c["prec"], rounding=False))

    def periodic(self, what, X):
        wc.assert_periodic(f"{self.tag} {what}", X, self.period, self.pl)

    def close(self):
        self.eng.check_health()
        self.eng.close()
        peak = torch.cuda.max_memory_allocated() / 2 ** 30
        print("WALK " + json.dumps({"case": self.tag, "sms": _sms(), "plan": self.pl, "layout": [self.plan[k] for k in
                                    ("tn", "ns", "nf")], "walk": self.walk, "peak_gib": round(peak, 2),
                                    "seconds": round(time.time() - self.t0, 1)}))
        self.eng = self.V = self.W0 = self.H0 = None
        _cleanup()


@pytest.mark.parametrize("walk", WALKS, ids=_id)
def test_kl_terms_and_loss_across_the_walk(walk):
    kind, prec, R = walk
    k = _Case(kind, prec, R, seed=11 + R)
    eng, which, c = k.eng, k.which, k.c
    try:
        assert eng.precision_for(1) == prec
        num, den = eng.raw_terms(which, 1)
        eng.check_health()
        model, exact = k.models()
        mnum, _, bar, _ = model.raw_terms(which, 1, nchunks=k.pl["nchunks"])
        enum, eden, _, _ = exact.raw_terms(which, 1)
        tcm.check_terms(f"kl-raw{which}-{k.tag}", num, mnum, bar, enum, tcm.RTOL64[prec])
        del mnum, bar, enum
        assert torch.allclose(den.double(), eden.reshape(-1), rtol=1e-5), "beta 1 denominator: column sums"
        k.periodic("beta 1 numerator", num)
        want = exact.loss(1)[0]
        if kind != "wide":
            tcm.check_loss(f"kl-loss-{k.tag}", eng.loss(1), model.loss(1), want, prec, 1)
            return
        # wide: the loss folded into the walked W update, then that update from the prefetched partial numerators
        plain = eng.loss(1)
        W, W_before = eng.W, eng.W.clone()
        eng.update_w(1.0, 1.0, 0.0, 0.0)
        eng.check_health()
        W_plain = W.clone()
        k.periodic("beta 1 W update", W_plain)
        W.copy_(W_before)
        eng.sync()
        got = eng.loss_prefetch_w(1.0)
        assert got == pytest.approx(plain, rel=2e-6)
        tcm.check_loss(f"kl-fold-{k.tag}", got, model.loss(1, fold=prec == "f16"), want, prec, 1)
        eng.update_w(1.0, 1.0, 0.0, 0.0)
        eng.check_health()
        assert torch.equal(W, W_plain), "the W update after the folded loss is not the plain W update"
    finally:
        k.close()


@pytest.mark.parametrize("walk", WALKS, ids=_id)
def test_eu_update_and_loss_across_the_walk(walk):
    """beta 2 (the residual kernel): one update of the walked factor against the model's numerator / denominator through
    the ratio stage, and the loss pass (which walks the H orientation)."""
    kind, prec, R = walk
    k = _Case(kind, prec, R, seed=23 + R)
    eng, which = k.eng, k.which
    try:
        assert eng.precision_for(2) == prec
        model, exact = k.models()
        if kind != "wide":
            tcm.check_loss(f"eu-loss-{k.tag}", eng.loss(2), model.loss(2), exact.loss(2)[0], prec, 2)
        num, den, bar, _ = model.raw_terms(which, 2, nchunks=k.pl["nchunks"])
        enum, eden, _, _ = exact.raw_terms(which, 2)
        kappa = model.kappa
        del model, exact
        old = (k.W0 if which == 0 else k.H0).double()
        (eng.update_w if which == 0 else eng.update_h)(2, 1.0, 0.0, 0.0)
        eng.check_health()
        got = eng.W if which == 0 else eng.H
        k.periodic("beta 2 update", got)

        def upd(n, d):
            return old * (n.clamp_min(0) + tcm.EPS) / (d.clamp_min(0) + tcm.EPS)
        want, want64 = upd(num, den), upd(enum, eden)
        # the ratio stage's fp32 Gram (<= 72 ulp), its product with F (R ulp), num + kappa den and the division (8 ulp)
        ratio_bar = tcm.U * (R + 80) * (1 + kappa * den.abs() / num.abs())
        tcm.check_terms(f"eu-upd{which}-{k.tag}", got, want, want * (bar / num.abs() + ratio_bar), want64, tcm.RTOL64[prec])
    finally:
        k.close()


@pytest.mark.parametrize("beta", TWO_BETAS)
def test_two_output_terms_and_loss_across_the_walk(beta):
    """beta not in {1, 2}: the two-output kernel (fast, rank 64, NF = 2) on the tall case: numerator and denominator of the
    H update, both periodic, and the loss."""
    k = _Case("tall", "f16", 64, seed=31, two_output=True)
    eng = k.eng
    try:
        assert eng.precision_for(beta) == "f16"
        num, den = eng.raw_terms(1, beta)
        eng.check_health()
        model, exact = k.models()
        mnum, mden, bar, dbar = model.raw_terms(1, beta, nchunks=k.pl["nchunks"])
        enum, eden, _, _ = exact.raw_terms(1, beta)
        tcm.check_terms(f"b{beta}-num1-{k.tag}", num, mnum, bar, enum, tcm.RTOL64["f16"] * max(1, abs(beta - 2)))
        del mnum, bar, enum
        tcm.check_terms(f"b{beta}-den1-{k.tag}", den, mden, dbar, eden, tcm.RTOL64["f16"] * max(1, abs(beta - 1)))
        del mden, dbar, eden
        k.periodic(f"beta {beta} numerator", num)
        k.periodic(f"beta {beta} denominator", den)
        tcm.check_loss(f"b{beta}-loss-{k.tag}", eng.loss(beta), model.loss(beta), exact.loss(beta)[0], "f16", beta)
    finally:
        k.close()
