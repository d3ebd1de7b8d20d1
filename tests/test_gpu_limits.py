"""The kernels past 2^31 elements and at the CUDA grid-dimension limits (cases: tests/limit_cases.py).

Big cases: the raw terms of both factors' updates (`raw_terms`) against float64, every row, from targets of just over 2^31
elements (NMF tall and wide, an NMF factor of more than 2^31 elements, a long NMFD batch).  fp32 at beta 2 on integer data
is bit-exact; otherwise the float64 bars of the fp32 suite (f32_cases.terms_bar) and, on the tensor cores, the f16 bar.
Each case first checks the card's free memory against the need its shape implies and skips naming the shortfall; it frees
its tensors and the cached contexts afterwards.  Each prints one LIMITS JSON line: worst err / bar, peak device memory,
wall time.

Grid cases: shapes on both sides of every grid limit (batches past 65535 on grid.z, B R past 65535, channels past
65535 x 64, R ceil(T / 128) = 65535 / 65536, the NMF tensor-core N limit) run one update of each factor's raw terms and
the loss against float64, or are rejected by create with NMFB200_ERR_INVALID and a message naming the limit.  Every case
asserts the path that ran (`precision_for`).
"""
import gc
import json
import time

import pytest
import torch

import f32_cases as fc
import limit_cases as lc
from oracle import mu_oracle as orc
from torchnmf_b200 import _capi
from torchnmf_b200.engine import CudaNmfdEngine, CudaNmfEngine, release_workspaces

pytestmark = pytest.mark.gpu


def _report(**kw):
    print("LIMITS " + json.dumps(kw))


def _need(nbytes):
    torch.cuda.synchronize()
    free, _ = torch.cuda.mem_get_info()
    if free < nbytes:
        pytest.skip(f"needs {nbytes / 2**30:.1f} GiB of device memory, {free / 2**30:.1f} GiB free "
                    f"(short by {(nbytes - free) / 2**30:.1f} GiB)")
    return free


def _cleanup():
    release_workspaces()
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


class _Peak:
    """Lowest free device memory seen (mem_get_info), sampled after each step."""

    def __init__(self, free0):
        self.free0, self.low = free0, free0

    def sample(self):
        torch.cuda.synchronize()
        self.low = min(self.low, torch.cuda.mem_get_info()[0])

    @property
    def gib(self):
        return (self.free0 - self.low) / 2 ** 30


def _compare(tag, got, want, bar):
    """bar None: bit-exact.  Else relative per entry.  Returns err / bar (0 for exact)."""
    got = got.double().reshape(want.shape)
    if bar is None:
        if not torch.equal(got, want):
            bad = (got != want).nonzero()[0].tolist()
            raise AssertionError(f"{tag}: {int((got != want).sum())} entries differ, first at {bad}: "
                                 f"{float(got[tuple(bad)])} vs {float(want[tuple(bad)])}")
        return 0.0
    diff, lim = (got - want).abs(), bar * want.abs()
    r = float((diff / lim.clamp_min(1e-300)).max())
    assert bool((diff <= lim).all()), f"{tag}: {r:.3f} x the relative bar {bar:.3e}"
    return r


def _nmf_runs():
    return [(name, prec, beta) for name, c in lc.NMF_BIG.items() for prec, betas in c["runs"].items() for beta in betas]


def _check_loss(tag, got, want, bar):
    assert abs(got - want) <= bar, f"{tag}: {got!r} vs {want!r}, bar {bar:.3e}"
    return abs(got - want) / bar


def _check_update(tag, got, old, num, den, beta, term_rel):
    """One ratio stage (gamma 1, no l1 / l2) from float64 terms: relative bar = ratio stage + the terms' relative bars
    (term_rel: a scalar or per-entry tensor; 0 for exact terms)."""
    kl = beta == 1
    if kl:                                         # the column sums of the other factor, one per component (dim 1)
        den = den.reshape((1, -1) + (1,) * (num.dim() - 2))
    want, mult = fc.ratio64(old.double(), num, den, 1.0, 0.0, 0.0, kl)
    bar = (fc.ratio_bar(mult, 1.0) + term_rel) * want.abs()
    err = (got.double() - want).abs()
    r = float((err / bar.clamp_min(1e-300)).max()) if bool((bar > 0).any()) else 0.0
    bad = (~(err <= bar)).nonzero()
    if bad.numel():
        i = tuple(bad[0].tolist())
        raise AssertionError(f"{tag}: {bad.shape[0]} entries past the bar, first at {i}: got {float(got[i])!r}, want "
                             f"{float(want[i])!r}, old {float(old[i])!r}, num {float(num[i])!r}, bar {float(bar[i])!r}")
    return r


@pytest.mark.parametrize("name,prec,beta", _nmf_runs())
def test_nmf_past_2p31(name, prec, beta):
    """The loss, the raw terms of both factors on every row, then one W update and one H update on the sampled rows."""
    case = lc.NMF_BIG[name]
    N, C, R = case["N"], case["C"], case["R"]
    _cleanup()
    free0 = _need(lc.nmf_device_bytes(case, prec, beta))
    t0 = time.time()
    peak = _Peak(free0)
    V, W, H = lc.nmf_data(case, beta, "cuda")
    eng = CudaNmfEngine(V, W, H, prec)
    try:
        assert eng.precision_for(beta) == prec
        plan = _capi.nmf_plan(N, C, R)
        want, lbar = lc.loss_bar_of(beta, lc.nmf_loss_ref(V, W, H, beta), R, prec)
        worst = _check_loss("loss", eng.loss(beta), want, lbar)
        peak.sample()
        bars = {}
        for which in (0, 1):
            n_other, nch = (N, plan["nch_w"]) if which == 0 else (C, plan["nch_h"])
            if prec == "f16":
                bars[which] = (lc.F16_BAR, lc.F16_BAR)
            elif beta == 2:
                assert lc.nmf_exact_bound(case) < fc.EXACT
                bars[which] = (None, None)
            elif case.get("kl_exact"):
                bars[which] = (lc.KL_EXACT_BAR, lc.KL_EXACT_BAR)
            else:
                bars[which] = fc.terms_bar(beta, R, n_other, nch)
        for which in case.get("which", [0, 1]):
            num, den = eng.raw_terms(which, beta)
            peak.sample()
            for rows in lc.row_ranges(case, which):
                enum, eden = lc.nmf_terms_ref(V, W, H, beta, which, rows)
                worst = max(worst, _compare(f"num{which}[{rows.start}:{rows.stop}]", num[rows.start:rows.stop], enum,
                                            bars[which][0]))
                if beta != 1:
                    worst = max(worst, _compare(f"den{which}[{rows.start}:{rows.stop}]", den[rows.start:rows.stop],
                                                eden, bars[which][1]))
            if beta == 1:                          # the column sums of the other factor (R values)
                worst = max(worst, _compare(f"den{which}", den, eden, bars[which][1]))
            del num, den, enum, eden
            _cleanup()
        for which in (0, 1):                       # W first, then H from the updated W
            F = W if which == 0 else H
            rows = lc.update_rows(case, which).cuda()
            old = F[rows].clone()
            (eng.update_w if which == 0 else eng.update_h)(beta, 1.0, 0.0, 0.0)
            peak.sample()
            num, den = lc.nmf_terms_ref(V, W, H, beta, which, rows, F_rows=old)
            if which == 1 and prec == "f32":       # the updated W is no longer integer: the fp32 bars of the H terms,
                # over the nonzero terms only (a banded W stays zero outside its hot rows; adding zeros is exact)
                n = len(lc.nmf_hot_rows(case)) if case["fac"] == "W" else C
                bars[1] = fc.terms_bar(beta, R, n, plan["nch_h"])
            rel = sum(b or 0.0 for b in bars[which])
            worst = max(worst, _check_update(f"update{which}", F[rows], old, num, den, beta, rel))
        peak.sample()
        _report(case=name, prec=prec, beta=beta, err_over_bar=worst, peak_gib=round(peak.gib, 2),
                need_gib=round(lc.nmf_device_bytes(case, prec, beta) / 2 ** 30, 2), wall_s=round(time.time() - t0, 1))
    finally:
        eng.close()
        del eng, V, W, H
        _cleanup()


def _nmfd_runs():
    return [(name, prec, beta) for name, c in lc.NMFD_BIG.items() for prec, betas in c["runs"].items() for beta in betas]


def _nmfd_term_bars(case, prec, beta, want, which):
    """Relative bars (numerator: scalar or per entry, denominator) of one factor's NMFD raw terms."""
    B, C, L, R, T = lc.nmfd_dims(case)
    if prec == "f16":
        # the f16 bar, plus what the fp32 accumulation of one split truncates (tests/tc_model.py): a sum of ~10^6 centred
        # terms on the tensor cores is not held to 1.25e-3 by the float64 bar alone
        tcp = _capi.nmfnd_tc_plan(B, C, [L], R, [T])
        trunc = lc.nmfd_tc_trunc(tcp["kbs_w"] if which == 0 else tcp["kbs_h"]) * want[2][which][0]
        return lc.F16_BAR + trunc / want[which][0].abs(), lc.F16_BAR
    plan = _capi.nmfd_plan(B, C, [L], R, [T])
    n, nch = (B * (L - T + 1), plan["wgrad_nsplit"]) if which == 0 else (C * T, plan["dgrad_nsplit"])
    return fc.terms_bar(beta, R * T, n, nch)


@pytest.mark.parametrize("name,prec,beta", _nmfd_runs())
def test_nmfd_terms_and_updates_past_2p31(name, prec, beta):
    """The loss, the raw terms of both factors, then one W update and one H update, every entry."""
    case = lc.NMFD_BIG[name]
    B, C, L, R, T = lc.nmfd_dims(case)
    _cleanup()
    free0 = _need(lc.nmfd_device_bytes(case, prec))
    t0 = time.time()
    peak = _Peak(free0)
    V, W, H = lc.nmfd_data(case, "cuda")
    eng = CudaNmfdEngine(V, W, H, prec)
    try:
        assert eng.precision_for(beta) == prec
        kappa = (lambda: lc.nmfd_kappa(V, W, H)) if prec == "f16" else (lambda: None)
        want, lbar = lc.loss_bar_of(beta, lc.nmfd_loss_ref(V, W, H, beta), R * T, prec)
        worst = _check_loss("loss", eng.loss(beta), want, lbar)
        got = [eng.raw_terms(which, beta) for which in (0, 1)]
        peak.sample()
        want = lc.nmfd_terms_ref(V, W, H, beta, kappa=kappa())
        peak.sample()
        for which in (0, 1):
            bn, bd = _nmfd_term_bars(case, prec, beta, want, which)
            g, w = got[which][0].double().reshape(want[which][0].shape), want[which][0]
            r = float(((g - w).abs() / (bn * w.abs())).max())
            assert r <= 1.0, f"num{which}: {r:.3f} x the bar"
            worst = max(worst, r, _compare(f"den{which}", got[which][1], want[which][1], bd))
        del got
        for which in (0, 1):                       # W first, then H from the updated W
            if which == 1:
                want = lc.nmfd_terms_ref(V, W, H, beta, kappa=kappa())
            F = W if which == 0 else H
            old = F.clone()
            (eng.update_w if which == 0 else eng.update_h)(beta, 1.0, 0.0, 0.0)
            peak.sample()
            bn, bd = _nmfd_term_bars(case, prec, beta, want, which)
            worst = max(worst, _check_update(f"update{which}", F, old, want[which][0], want[which][1], beta, bn + bd))
            del old
        del want
        _report(case=name, prec=prec, beta=beta, err_over_bar=worst, peak_gib=round(peak.gib, 2),
                need_gib=round(lc.nmfd_device_bytes(case, prec) / 2 ** 30, 2), wall_s=round(time.time() - t0, 1))
    finally:
        eng.close()
        del eng, V, W, H
        _cleanup()


# ---- grid limits ---------------------------------------------------------------------------------------------------------
def _create_error(kind, shape, prec):
    """(rc, message) of create for this shape (no target, no launch)."""
    import ctypes
    lib = _capi.load()
    ctx = ctypes.c_void_p()
    if kind == "nmf":
        rc = lib.nmfb200_nmf_create(ctypes.byref(ctx), 0, *shape, _capi.PRECISIONS[prec])
    else:
        B, C, L, R, T = shape
        rc = lib.nmfb200_nmfnd_create(ctypes.byref(ctx), 0, B, C, 1, (ctypes.c_int64 * 1)(L), R, (ctypes.c_int64 * 1)(T),
                                      _capi.PRECISIONS[prec])
    if rc == 0:
        lib.nmfb200_destroy(ctx)
        return 0, ""
    return rc, lib.nmfb200_last_error().decode()


def _grid_data(kind, shape, seed):
    g = torch.Generator().manual_seed(seed)
    if kind == "nmf":
        N, C, R = shape
        dims = ((N, C), (C, R), (N, R))
    else:
        B, C, L, R, T = shape
        dims = ((B, C, L), (C, R, T), (B, R, L - T + 1))
    return tuple((torch.rand(*d, generator=g) + 0.5).cuda() for d in dims)


def _nmfd_refused(case):
    return case[1] == "nmfd" and case[4] != "runs"


NMFD_REFUSED = [c for c in lc.GRID_CASES if _nmfd_refused(c)]


@pytest.mark.parametrize("name,kind,shape,prec,expected", NMFD_REFUSED, ids=[c[0] for c in NMFD_REFUSED])
def test_nmfnd_create_refuses_past_the_grid_limit(name, kind, shape, prec, expected):
    rc, msg = _create_error(kind, shape, prec)
    assert rc == 1 and expected[1] in msg, (rc, msg)


GRID_CASES = [c for c in lc.GRID_CASES if not _nmfd_refused(c)]


@pytest.mark.parametrize("name,kind,shape,prec,expected", GRID_CASES, ids=[c[0] for c in GRID_CASES])
def test_grid_limit(name, kind, shape, prec, expected):
    _cleanup()
    if expected != "runs":
        rc, msg = _create_error(kind, shape, prec)
        assert rc == 1 and expected[1] in msg, (rc, msg)
        return
    _need(lc.grid_bytes(kind, shape, prec))
    t0 = time.time()
    V, W, H = _grid_data(kind, shape, seed=sum(shape))
    resolved = prec
    if prec == "auto":
        resolved = "f32"
    eng = (CudaNmfEngine if kind == "nmf" else CudaNmfdEngine)(V, W, H, prec)
    try:
        assert eng.precision_for(1) == resolved
        W64, H64, V64 = W.double(), H.double(), V.double()
        worst = 0.0
        if kind == "nmf":
            N, C, R = shape
            S = H64 @ W64.t()
            Pn, _ = orc.phi(V64, S, 1)
            plan = _capi.nmf_plan(N, C, R)
            for which, n, nch in ((0, N, plan["nch_w"]), (1, C, plan["nch_h"])):
                num, den = eng.raw_terms(which, 1)
                enum, eden = fc.nmf_terms64(which, Pn, None, W64, H64)
                bar = lc.F16_BAR if resolved == "f16" else fc.terms_bar(1, R, n, nch)[0]
                worst = max(worst, _compare(f"num{which}", num, enum, bar), _compare(f"den{which}", den, eden, bar))
        else:
            B, C, L, R, T = shape
            S = fc.recon(H64, W64)
            Pn, _ = orc.phi(V64, S, 1)
            plan = _capi.nmfd_plan(B, C, [L], R, [T])
            for which, n, nch in ((0, B * (L - T + 1), plan["wgrad_nsplit"]), (1, C * T, plan["dgrad_nsplit"])):
                num, den = eng.raw_terms(which, 1)
                enum, eden = fc.nmfd_terms64(which, Pn, None, W64, H64)
                bar = lc.F16_BAR if resolved == "f16" else fc.terms_bar(1, R * T, n, nch)[0]
                worst = max(worst, _compare(f"num{which}", num, enum, bar), _compare(f"den{which}", den, eden, bar))
        want, lbar = fc.loss_bar(1, S.reshape(-1), V64.reshape(-1), R * (T if kind == "nmfd" else 1), orc.EPS)
        got = eng.loss(1)
        lbar = max(lbar, abs(want) * lc.F16_BAR) if resolved == "f16" else lbar
        assert abs(got - want) <= lbar, (got, want, lbar)
        worst = max(worst, abs(got - want) / lbar)
        _report(case=name, prec=resolved, err_over_bar=worst, wall_s=round(time.time() - t0, 1))
    finally:
        eng.close()
        del eng, V, W, H
        _cleanup()


@pytest.mark.parametrize("name,shape,prec,words", lc.REJECT_CASES, ids=[c[0] for c in lc.REJECT_CASES])
def test_nmfnd_create_rejects_past_the_narrowing_bounds(name, shape, prec, words):
    rc, msg = _create_error("nmfd", shape, prec)
    assert rc == 1 and words in msg, (rc, msg)
