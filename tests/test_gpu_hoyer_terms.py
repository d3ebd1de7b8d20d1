"""`nmfb200_hoyer_project` (csrc/project.cu) slice by slice, and the target min / max of fit()'s validation.

Cases, references and bars: tests/hoyer_cases.py.  Every slice of every case is held to the model of the kernel's arithmetic
at the model's bar, with the same zero set except where the model's trajectories disagree; stable slices are also held to
float64 at the conditioning bar.  Whatever the class: no NaN or Inf except where the reference algorithm yields NaN, no
negative entry, and sum y = k1, sum y^2 = k2 within bars from the final round.

Degenerate slices: where the surviving support is uniform, a = w.w = 0 and alphap = 0 / 0: the reference returns NaN for the
slice and so does the kernel (the NaN is not negative, so the round ends the loop).  Where a round zeroes every coordinate,
the reference divides by zero (nmf.py:32 raises ZeroDivisionError); the kernel leaves the slice at zero through its
`nzero >= n` exit.  The fp32 rounds need not meet these where float64 does: they are pinned to the model.

Each case prints one HOYER JSON line with the worst error over bar per group.
"""
import ctypes
import gc
import json

import numpy as np
import pytest
import torch

import hoyer_cases as hc
from torchnmf_b200 import _capi
from torchnmf_b200 import engine as _engine
from torchnmf_b200.engine import CudaNmfdEngine, CudaNmfEngine, release_workspaces

pytestmark = pytest.mark.gpu

NAMES = [c.name for c in hc.CASES]


def _report(**kw):
    print("HOYER " + json.dumps(kw))


def _project(x, dim, k1, k2, poison=None):
    """One launch through the C ABI; `poison` fills the zeroed workspace first (None: zeros)."""
    outer, D, inner = hc.layout(tuple(x.shape), dim)
    ws = torch.full((x.numel(),), 0 if poison is None else poison, dtype=torch.uint8, device=x.device)
    k1 = torch.as_tensor(k1, dtype=torch.float32).cuda()
    k2 = torch.as_tensor(k2, dtype=torch.float32).cuda()
    lib = _capi.load()
    _capi.check(lib.nmfb200_hoyer_project(torch.cuda.current_device(), ctypes.c_void_p(x.data_ptr()), outer, D, inner,
                                          ctypes.c_void_p(k1.data_ptr()), ctypes.c_void_p(k2.data_ptr()),
                                          ctypes.c_void_p(ws.data_ptr()), _engine._stream(x.device)))
    torch.cuda.synchronize()
    return x


FORMS_SEEN = set()


def match_form(mb, got):
    """(err / bar, form) of the model form the kernel slice matches best: same NaN pattern, same zero set outside the
    form's ambiguous entries, error over that form's bar."""
    best = None
    for name, f in mb.forms.items():
        want = f.y.astype(np.float64)
        nan = np.isnan(want)
        if not np.array_equal(nan, np.isnan(got)) or (((got == 0) != (want == 0)) & ~f.ambiguous).any():
            continue
        e = float((np.abs(got - want)[~nan] / f.bar[~nan]).max()) if (~nan).any() else 0.0
        if best is None or e < best[0]:
            best = (e, name)
    assert best is not None, "the NaN pattern or the zero set matches no form of the model"
    return best


def check_slice(a, got):
    """Errors over bar of one kernel slice `got` (float64 numpy): (model, float64 or None, sum, sum of squares)."""
    mb = a["mb"]
    em, form = match_form(mb, got)
    FORMS_SEEN.add(form)
    if a["ref"].outcome in ("nan", "overflow"):  # a = 0 in float64 (fp32 rounding may leave w != 0: the model decides
        return em, None, 0.0, 0.0                # NaN or not), or b^2 / 4ac past the fp32 range: the model only
    assert np.isfinite(got).all() and (got >= 0).all()
    e64 = None
    if a["cls"] == "stable":
        e64 = float(np.abs(got - a["ref"].y).max()) / a["bar64"]
    b1, b2 = hc.invariant_bars(mb, a["k1"], a["k2"])
    es = abs(got.sum() - float(a["k1"])) / b1
    eq = abs((got * got).sum() - float(a["k2"])) / b2
    if mb.model.exit == "all-zeroed":            # every coordinate zeroed: the kernel leaves zeros, no constraint holds
        assert not got.any()
        es = eq = 0.0
    return em, e64, es, eq


@pytest.mark.parametrize("name", NAMES)
def test_kernel_matches_model_and_float64(name):
    c = hc.BY_NAME[name]
    x, k1, k2 = hc.case_tensor(c)
    y = _project(torch.from_numpy(x).cuda(), c.dim, k1, k2).cpu().numpy()
    ys = hc.slices(y, c.dim).astype(np.float64)
    worst = dict(model=0.0, float64=0.0, sum=0.0, sumsq=0.0)
    for j, a in enumerate(hc.analyse(name)):
        em, e64, es, eq = check_slice(a, ys[j])
        for k, v in (("model", em), ("float64", e64), ("sum", es), ("sumsq", eq)):
            if v is not None:
                worst[k] = max(worst[k], v)
    classes = [a["cls"] for a in hc.analyse(name)]
    _report(case=name, n=c.n, D=c.D, classes={k: classes.count(k) for k in set(classes)},
            rounds=max(a["mb"].model.rounds for a in hc.analyse(name)),
            model_bar_rel=max(a["mb"].rel() for a in hc.analyse(name)), forms=sorted(FORMS_SEEN), **worst)
    for k, v in worst.items():
        assert v <= 1.0, f"{name}: {k} error {v:.3g} x the bar"


def test_many_slices_past_int32():
    """D n > 2^31: every slice is one of 8 patterns; identical slices give bit-identical outputs and the 8 patterns are
    held to the model and float64."""
    c = hc.HUGE
    outer, D, inner = c.layout
    need = int(D * outer * inner * 5 * 1.1) + (1 << 30)
    torch.cuda.synchronize()
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f"needs {need / 2**30:.1f} GiB of device memory, {free / 2**30:.1f} GiB free "
                    f"(short by {(need - free) / 2**30:.1f} GiB)")
    P, k1p, k2p = hc.huge_patterns()
    reps = D // hc.HUGE_PATTERNS
    try:
        x = torch.from_numpy(P).cuda().repeat(1, reps)
        k1 = torch.from_numpy(np.tile(k1p, reps)).cuda()
        k2 = torch.from_numpy(np.tile(k2p, reps)).cuda()
        _engine.hoyer_project_(x, 1, k1, k2)
        torch.cuda.synchronize()
        first = x[:, :hc.HUGE_PATTERNS].clone()
        v = x.view(outer, reps, hc.HUGE_PATTERNS)
        step = 4096
        for r0 in range(0, reps, step):
            blk = v[:, r0:r0 + step, :]
            same = (blk == first[:, None, :]) | (torch.isnan(blk) & torch.isnan(first[:, None, :]))
            assert bool(same.all()), f"a repeat of a pattern differs in repeats {r0}..{r0 + step}"
        ys = first.cpu().numpy().T.astype(np.float64)
        worst = [0.0, 0.0]
        for j, a in enumerate(hc.analyse("huge")):
            em, e64, _, _ = check_slice(a, ys[j])
            worst = [max(worst[0], em), max(worst[1], e64 or 0.0)]
        _report(case="huge", n=outer * inner, D=D, model=worst[0], float64=worst[1])
        assert max(worst) <= 1.0
    finally:
        x = v = blk = same = None
        gc.collect()
        torch.cuda.empty_cache()


@pytest.mark.parametrize("name", ["decays", "h_cfg1", "nmfd_w", "negative", "all_zeroed", "n1025"])
def test_poisoned_workspace_and_repeat_launches_are_bit_identical(name):
    """zeroed_ws is scratch: a workspace left at 0xFF by an earlier user must not change a bit (round 0 clears it), and
    two launches give the same bits."""
    c = hc.BY_NAME[name]
    x, k1, k2 = hc.case_tensor(c)
    xc = torch.from_numpy(x).cuda()
    clean = _project(xc.clone(), c.dim, k1, k2)
    again = _project(xc.clone(), c.dim, k1, k2)
    poisoned = _project(xc.clone(), c.dim, k1, k2, poison=0xFF)
    for got in (again, poisoned):
        assert torch.equal(got.view(torch.int32), clean.view(torch.int32))


@pytest.mark.parametrize("name", ["n4097", "nmf3d_w", "dim2_4d", "dim3_4d", "dim0_3d", "dim2_5d", "dim3_5d", "sp_high"])
def test_any_dim_is_dim_1_of_the_moved_tensor(name):
    """Along dim d the kernel enumerates slice elements as (outer, inner), the order x.movedim(d, 1) has along dim 1:
    the outputs are bit-identical."""
    c = hc.BY_NAME[name]
    x, k1, k2 = hc.case_tensor(c)
    xc = torch.from_numpy(x).cuda()
    a = _project(xc.clone(), c.dim, k1, k2)
    b = _project(xc.movedim(c.dim, 1).contiguous(), 1, k1, k2)
    assert torch.equal(a.movedim(c.dim, 1).contiguous().view(torch.int32), b.view(torch.int32))


# ------------------------------------------------------------------------------------------------------------------
# target_minmax: minmax_stage1 / minmax_stage2 (csrc/update.cu), NaN-sticky, exact
# ------------------------------------------------------------------------------------------------------------------
def _bits(v):
    return np.float32(v).view(np.uint32)


def _assert_minmax(got, V):
    want = torch.aminmax(V) if not torch.isnan(V).any() else (torch.tensor(float("nan")),) * 2
    for g, w, nm in ((got[0], want[0], "min"), (got[1], want[1], "max")):
        w = float(w)
        if w != w:
            assert g != g, f"{nm}: {g} where V holds NaN"
        else:
            assert _bits(g) == _bits(w), f"{nm}: {g!r} vs {w!r}"
    return 0.0


MM_N, MM_C = 2100, 2049                  # 4.3M entries: 1024 blocks of 256 x 16, a grid-stride second pass


@pytest.mark.parametrize("where", ["first", "last", "last_partial_block", "past_grid_stride", "signed_zero_inf",
                                   "subnormal"])
def test_target_minmax_is_exact_and_nan_sticky(where):
    g = torch.Generator().manual_seed(9)
    V = torch.rand(MM_N, MM_C, generator=g) + 0.5
    flat = V.view(-1)
    total = flat.numel()
    if where == "first":
        flat[0] = float("nan")
    elif where == "last":
        flat[-1] = float("nan")
    elif where == "last_partial_block":
        flat[total - 3] = float("nan")
    elif where == "past_grid_stride":            # the second grid-stride pass: index >= 1024 blocks x 256 threads
        flat[1024 * 256 + 1000] = float("nan")
    elif where == "signed_zero_inf":
        flat[12345] = -0.0
        flat[total // 2] = float("inf")
    else:
        flat[777] = 1e-45                        # the smallest subnormal
        flat[778] = 3e-39
    eng = CudaNmfEngine(V.cuda(), torch.rand(MM_C, 2, generator=g).cuda(), torch.rand(MM_N, 2, generator=g).cuda(), "f32")
    got = eng.minmax()
    eng.close()
    release_workspaces()
    _assert_minmax(got, V)
    if where == "signed_zero_inf":
        assert str(got[0]) == "-0.0" and got[1] == float("inf")
    _report(case=f"minmax-{where}", minmax=0.0)


@pytest.mark.parametrize("nan_pad", [False, True])
def test_minmax_of_a_strided_target_ignores_its_padding(nan_pad):
    """nmfb200_nmf_set_target with ldv > C: the padding columns (NaN, -Inf, +Inf) must not reach the min / max."""
    g = torch.Generator().manual_seed(10)
    N, C, ldv = 1500, 1111, 1200
    Vp = torch.rand(N, ldv, generator=g) + 0.25
    Vp[:, C:] = float("nan") if nan_pad else -float("inf")
    Vp[0, C] = float("inf")
    V = Vp[:, :C].contiguous()
    eng = CudaNmfEngine(V.cuda(), torch.rand(C, 3, generator=g).cuda(), torch.rand(N, 3, generator=g).cuda(), "f32")
    Vpd = Vp.cuda()
    _capi.check(eng._lib.nmfb200_nmf_set_target(eng._ctx, ctypes.c_void_p(Vpd.data_ptr()), ldv, _capi.DTYPE_F32,
                                                 _engine._stream(Vpd.device)))
    got = eng.minmax()
    eng.close()
    release_workspaces()
    del Vpd
    _assert_minmax(got, V)
    _report(case=f"minmax-ldv-nan{int(nan_pad)}", minmax=0.0)


@pytest.mark.parametrize("nan", [False, True])
def test_nmfd_target_minmax(nan):
    g = torch.Generator().manual_seed(11)
    V = torch.rand(3, 7, 4100, generator=g) + 0.125
    V[1, 3, 17] = 2.0 ** -140
    if nan:
        V[2, 6, 4099] = float("nan")
    eng = CudaNmfdEngine(V.cuda(), torch.rand(7, 2, 5, generator=g).cuda(), torch.rand(3, 2, 4096, generator=g).cuda(), "f32")
    got = eng.minmax()
    eng.close()
    release_workspaces()
    _assert_minmax(got, V)
    _report(case=f"minmax-nmfd-nan{int(nan)}", minmax=0.0)


# ------------------------------------------------------------------------------------------------------------------
# sparse_fit and SparsityProj call by call: every engine call is read back and held to float64 from its own inputs, so
# that errors do not accumulate; every projection to the model.
# ------------------------------------------------------------------------------------------------------------------
import f32_cases as fc                                       # noqa: E402
from oracle import mu_oracle as orc                          # noqa: E402
from torchnmf_b200 import NMF, NMF2D, NMFD, SparsityProj    # noqa: E402
from torchnmf_b200 import trainer as _trainer                # noqa: E402
from torchnmf_b200.metrics import beta_div                   # noqa: E402

F16_RTOL, F16_LOSS = 1.25e-3, 2.0 ** -11                     # the f16 bars of tests/sequence_cases.float64_check


def check_projection(x_in, dim, k1, k2, got, worst):
    """Every slice of one projection launch against the model (and float64 where stable).  Returns how many slices
    overflowed the fp32 quadratic."""
    xs = hc.slices(x_in.cpu().numpy(), dim)
    gs = hc.slices(got.cpu().numpy(), dim).astype(np.float64)
    k1 = np.asarray(torch.as_tensor(k1, dtype=torch.float32).cpu(), np.float32)
    k2 = np.asarray(torch.as_tensor(k2, dtype=torch.float32).cpu(), np.float32)
    over = 0
    for j in range(xs.shape[0]):
        cls, ref, bar64 = hc.classify(xs[j], k1[j], k2[j], seed=j)
        a = dict(cls=cls, ref=ref, bar64=bar64, mb=hc.model_bar(xs[j], k1[j], k2[j]), k1=k1[j], k2=k2[j])
        em, e64, es, eq = check_slice(a, gs[j])
        worst["project"] = max(worst["project"], em, e64 or 0.0, es, eq)
        over += ref.outcome == "overflow"
    assert worst["project"] <= 1.0, f"projection {worst['project']:.3g} x the bar"
    return over


def _err_over(got, want, rel):
    """Max relative error over bar on the finite entries; NaN and Inf must sit where float64 of the same inputs has them
    (a fit whose trial factors overflowed carries NaN, in the reference as here)."""
    nf = ~torch.isfinite(want)
    assert torch.equal(nf, ~torch.isfinite(got)) and torch.equal(torch.isnan(want), torch.isnan(got)), "NaN / Inf placement"
    fin = ~nf
    if not bool(fin.any()):
        return 0.0
    rel = torch.as_tensor(rel, dtype=torch.float64).expand_as(want)
    return float(((got - want).abs()[fin] / (rel * want.abs())[fin].clamp_min(1e-300)).max())


class Recorder:
    """Wraps a CudaNmfEngine / CudaNmfdEngine: reads back the inputs of every call and checks its result in float64."""

    def __init__(self, inner, kind):
        self.inner, self.kind_ = inner, kind
        self.worst = dict(raw=0.0, loss=0.0, update=0.0, project=0.0, renorm=0.0)
        self.calls, self.flips, self.decisions, self.renorms, self.overflow = {}, 0, 0, 0, 0
        self._loss = None                     # (kernel, float64, bar) of the last loss()
        self._prev = None                     # (W, H) at the last sync
        self._h_step = False
        self._last = None

    def __getattr__(self, name):
        return getattr(self.inner, name)

    def _count(self, name):
        self.calls[name] = self.calls.get(name, 0) + 1
        self._last = name

    def _snap(self, W=None, H=None):
        W = self.inner.W if W is None else W
        H = self.inner.H if H is None else H
        return W.detach().double().cpu(), H.detach().double().cpu()

    def _recon(self, W, H):
        return orc.nmf_reconstruct(H, W) if self.kind_ == "nmf" else fc.recon(H, W)

    def _f16(self, beta):
        return self.inner.precision_for(beta) != "f32"

    def _loss64(self, W, H, beta):
        s, v = self._recon(W, H).reshape(-1), self.inner.V.double().cpu().reshape(-1)
        ks = W[0].numel()                                      # products per reconstruction entry: R x prod(K)
        if self._f16(beta):
            term, M = fc.loss_pieces(beta, s, v, 2.0 ** -23)
            g = max(1.0, abs(beta), abs(beta - 1))
            return float(term.sum()), float((F16_LOSS * g + 2.0 ** -12) * M.sum())
        return fc.loss_bar(beta, s, v, ks, 2.0 ** -23)

    def _check_loss(self, got, W, H, beta):
        want, bar = self._loss64(W, H, beta)
        if want != want:                      # a trial factor holding NaN (an overflowed projection): NaN, rejected
            assert got != got, f"loss {got} where float64 gives NaN"
            return want, 0.0
        self.worst["loss"] = max(self.worst["loss"], abs(got - want) / bar)
        assert abs(got - want) <= bar, f"loss {got} vs {want} (bar {bar})"
        return want, bar

    def _terms64(self, W, H, which, beta):
        V = self.inner.V.double().cpu()
        Pn, Pp = orc.phi(V, self._recon(W, H), beta)
        if self.kind_ == "nmf":
            return fc.nmf_terms64(which, Pn, None if beta == 1 else Pp, W, H)
        return fc.nmfd_terms64(which, Pn, None if beta == 1 else Pp, W, H)

    def _term_bars(self, W, H, which, beta):
        if self._f16(beta):
            return (F16_RTOL * max(1, abs(beta - 2)), F16_RTOL * max(1, abs(beta - 1))) if beta not in (1, 2) else \
                (F16_RTOL, F16_RTOL)
        V = self.inner.V
        n = V.numel() // (W.shape[0] if which == 0 else H.shape[0])        # terms per entry, at most
        return fc.terms_bar(beta, W[0].numel(), n, n)

    # ---- the engine interface ----
    def loss(self, beta):
        W, H = self._snap()
        got = self.inner.loss(beta)
        self._count("loss")
        self._loss = (got,) + self._check_loss(got, W, H, beta)
        return got

    def loss_at(self, W, H, beta):
        Wc, Hc = self._snap(W, H)
        got = self.inner.loss_at(W, H, beta)
        self._count("loss_at")
        want, bar = self._check_loss(got, Wc, Hc, beta)
        cur, cur64, cbar = self._loss
        self.decisions += 1
        if (got <= cur) != (want <= cur64):                 # a flipped line-search decision: only within the loss bars
            assert want == want and cur64 == cur64
            self.flips += 1
            assert abs(want - cur64) <= bar + cbar, f"line search decided {got} <= {cur}, float64 {want} vs {cur64}"
        return got

    def raw_terms(self, which, beta):
        W, H = self._snap()
        num, den = self.inner.raw_terms(which, beta)
        self._count("raw_terms")
        self._h_step = which == 1
        wn, wd = self._terms64(W, H, which, beta)
        rn, rd = self._term_bars(W, H, which, beta)
        if beta == 1:
            rd = fc.gam(self.inner.V.numel()) + 2 * fc.U
        for got, want, r in ((num, wn, rn), (den, wd, rd)):
            e = _err_over(got.double().cpu().reshape(want.shape), want, r)
            self.worst["raw"] = max(self.worst["raw"], e)
            assert e <= 1.0, f"raw terms {which} beta {beta}: {e:.3g} x the bar"
        return num, den

    def project(self, x, dim, k1, k2):
        x_in = x.detach().clone()
        out = self.inner.project(x, dim, k1, k2)
        torch.cuda.synchronize()
        self._count("project")
        self.overflow += check_projection(x_in, dim, k1, k2, x, self.worst)
        return out

    def _update(self, which, beta, gamma, l1, l2):
        W, H = self._snap()
        (self.inner.update_w if which == 0 else self.inner.update_h)(beta, gamma, l1, l2)
        self._count("update_w" if which == 0 else "update_h")
        self._h_step = which == 1
        num, den = self._terms64(W, H, which, beta)
        p = W if which == 0 else H
        if beta == 1:
            den = den.reshape((1, -1) + (1,) * (p.dim() - 2))
        want, mult = fc.ratio64(p, num, den, gamma, l1, l2, beta == 1)
        rn, rd = self._term_bars(W, H, which, beta)
        rel = gamma * (rn + (rd if beta != 1 else 1e-5)) + fc.ratio_bar(mult, gamma)
        got = (self.inner.W if which == 0 else self.inner.H).double().cpu()
        if which == 1:
            self._prev = self._snap()                         # what the renormalisation starts from
        e = _err_over(got, want, rel)
        self.worst["update"] = max(self.worst["update"], e)
        assert e <= 1.0, f"update {which} beta {beta}: {e:.3g} x the bar"

    def update_w(self, beta, gamma, l1, l2):
        self._update(0, beta, gamma, l1, l2)

    def update_h(self, beta, gamma, l1, l2):
        self._update(1, beta, gamma, l1, l2)

    def sync(self):
        W, H = self._snap()
        if self._h_step and self._last in ("update_h", "sync") and self._prev is not None:
            W0, H0 = self._prev                               # nmf.py:588: H / |H[:, r]|, W * |H[:, r]|
            nrm = H0.pow(2).sum([d for d in range(H0.dim()) if d != 1]).sqrt()
            hs = (slice(None),) + (None,) * (H0.dim() - 2)
            ws = (slice(None),) + (None,) * (W0.dim() - 2)
            bar = 4 * fc.U + fc.gam(H0[:, 0].numel())
            e = max(_err_over(H, H0 / nrm[hs], bar), _err_over(W, W0 * nrm[ws], bar))
            self.worst["renorm"] = max(self.worst["renorm"], e)
            assert e <= 1.0, f"renormalisation {e:.3g} x the bar"
            self._h_step = False
            self.renorms += 1
        self.inner.sync()
        self._count("sync")
        self._prev = (W, H)


SFIT = [  # (name, module, V shape, W shape, H shape, beta, sW, sH, precision)
    # with both constraints at beta 1 and 0.5 the reference's own fit blows up (rows of S at 0: gradients of 1e12, trial
    # projections past the fp32 quadratic's range, NaN trials): the calls are still checked one by one, NaN included
    *[(f"nmf_{tag}_b{b}", "nmf", (64, 48), (48, 8), (64, 8), b, sw, sh, "auto")
      for b in (2, 1, 0.5, 1.5) for tag, sw, sh in (("sW", 0.5, None), ("sH", None, 0.4), ("both", 0.5, 0.4))],
    ("nmfd_sW_b1", "nmfd", (2, 6, 40), (6, 3, 5), (2, 3, 36), 1, 0.5, None, "auto"),
    ("nmfd_sH_b1", "nmfd", (2, 6, 40), (6, 3, 5), (2, 3, 36), 1, None, 0.6, "auto"),
    ("nmf2d_both_b2", "nmf2d", (2, 5, 12, 10), (5, 3, 3, 2), (2, 3, 10, 9), 2, 0.5, 0.5, "auto"),
    ("nmf_sH_f16_b1", "nmf", (256, 192), (192, 8), (256, 8), 1, None, 0.25, "f16"),
]
MODULES = {"nmf": NMF, "nmfd": NMFD, "nmf2d": NMF2D}


@pytest.mark.parametrize("case", SFIT, ids=lambda c: c[0])
def test_sparse_fit_call_by_call(case):
    name, mod, vs, wsh, hsh, beta, sW, sH, prec = case
    g = torch.Generator().manual_seed(sum(vs) + int(beta * 10))
    V = (torch.rand(*vs, generator=g) + 0.1).cuda()
    m = MODULES[mod](W=torch.rand(*wsh, generator=g) + 0.05, H=torch.rand(*hsh, generator=g) + 0.05).cuda()
    recs = []

    def factory(Vd, W, H):                              # the precision sparse_fit resolves: "auto" is "f32" under a constraint
        p = "f32" if prec == "auto" else prec
        inner = CudaNmfEngine(Vd, W, H, p) if mod == "nmf" else CudaNmfdEngine(Vd, W, H, p)
        recs.append(Recorder(inner, "nmf" if mod == "nmf" else "nd"))
        recs[-1].prec = inner.precision_for(beta)
        return recs[-1]
    m._engine_factory = factory
    try:
        m.sparse_fit(V, beta, 4, False, sW, sH, precision=prec)
    finally:
        release_workspaces()
    r = recs[0]
    if prec == "f16":                                   # the unconstrained W update ran on the tensor cores
        assert r.prec == "f16" and r.calls.get("update_w", 0) == 4
    assert r.calls.get("project", 0) >= 4 and r.decisions >= 4
    assert r.renorms == 4                               # after every H step
    _report(case=f"sfit-{name}", calls=r.calls, decisions=r.decisions, flips=r.flips, overflow_slices=r.overflow,
            **r.worst)


@pytest.mark.parametrize("dim", [0, 1])
def test_sparsity_proj_call_by_call(dim, monkeypatch):
    """SparsityProj.step: every projection of every parameter, at each line-search trial, against the model."""
    g = torch.Generator().manual_seed(20 + dim)
    V = (torch.rand(96, 80, generator=g) + 0.1).cuda()
    m = NMF(W=torch.rand(80, 5, generator=g) + 0.05, H=torch.rand(96, 5, generator=g) + 0.05).cuda()
    worst = dict(project=0.0)
    count = [0]
    real = _trainer._project_slices_

    def recording(p, d, k1, k2):
        x_in = p.detach().clone()
        real(p, d, k1, k2)
        torch.cuda.synchronize()
        count[0] += 1
        check_projection(x_in, d, k1, k2, p.detach(), worst)
    monkeypatch.setattr(_trainer, "_project_slices_", recording)
    tr = SparsityProj([m.W, m.H], 0.6, dim=dim)
    tr.param_groups[0]["lr"] = 0.01

    def closure():
        tr.zero_grad()
        return beta_div(m(), V, 1)
    for _ in range(3):
        tr.step(closure)
    assert count[0] >= 6
    _report(case=f"sproj-dim{dim}", projections=count[0], **worst)
