"""Long-lived engine contexts, call by call (tests/sequence_cases.py): every step of a scripted sequence on ONE context is
checked against a float64 evaluation of that step from the factors it started from.

Per step:
  * the path that ran (`precision_for`) is the one the host-side state machine (sequence_cases.simulate) says;
  * a W update after a prefetch skips its contraction exactly when it may (`nmfb200_launch_count`);
  * tensor-core steps: the model bar and the float64 bar of tests/test_gpu_tc_terms.py (tc_model.check_terms /
    check_loss) for raw terms and losses; an update is its model terms through the float64 ratio stage, with the model bar
    of the terms carried through it (plus the ratio stage's own fp32 bar, tests/f32_cases.py);
  * fp32 steps (the fp32 kernels, sparse targets, NMFD beta 2): bit-equal to the same call on a fresh context, and within
    the float64 bars of the f16 mode.
The tensor-core sequences run at target scales 2^s, s in sequence_cases.SCALES, with the factors matched so that W H ~ V,
and once with unbalanced factors (W 2^8, H 2^-8).
"""
import ctypes
import json

import pytest
import torch

import f32_cases as fc
import sequence_cases as sc
import sparse_cases as spc
import tc_model as tcm
from torchnmf_b200 import _capi, engine as E

pytestmark = pytest.mark.gpu

U = tcm.U


def _report(**kw):
    print("SEQ " + json.dumps(kw))


def _make(seq, V, W, H):
    if seq.kind == "nmfd":
        return E.CudaNmfdEngine(V, W, H, seq.precision)
    if seq.kind == "sparse":
        return E.CudaSparseNmfEngine(V, W, H)
    return E.CudaNmfEngine(V, W, H, seq.precision)


def _fresh_f32(seq, eng, V, W0, H0):
    """A new fp32 context of the same kind on the factors a step started from."""
    W, H = W0.clone(), H0.clone()
    if seq.kind == "nmfd":
        return E.CudaNmfdEngine(V, W, H, "f32")
    if isinstance(eng, E.CudaSparseNmfEngine):
        return E.CudaSparseNmfEngine(V, W, H)
    return E.CudaNmfEngine(V, W, H, "f32")


class Checker:
    def __init__(self, seq, scale):
        self.seq, self.scale = seq, scale
        self.V = None                             # the current target (dense, device)
        self.worst = 0.0

    def path_prec(self, beta):
        if self.seq.precision in ("f16", "auto"):
            return "f16"
        return "f16" if sc.two_output(beta) else self.seq.precision

    # -- tensor-core steps --------------------------------------------------------------------------------------------------
    def nmf_model(self, W, H, rounding=True):
        return tcm.NmfModel(self.V, W, H, self.path_prec(1), rounding=rounding)

    def nchunks(self, which):
        N, C, R = self.seq.shape
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        tn = tcm.tn(self.seq.precision, R)
        return tcm.plan(C, N, sms, tn)[2] if which == 0 else tcm.plan(N, C, sms, tn)[2]

    def tc_terms(self, W, H, which, beta):
        """(num, den, bar_num, bar_den or None, num64, den64, rtol_num, rtol_den) at the factors (W, H)."""
        if self.seq.kind == "nmfd":
            B, C, L, R, T = self.seq.shape
            ns = tcm.nmfd_splits(*self.seq.shape)[0 if which == 0 else 3]
            num, den, bar = tcm.NmfdModel(self.V, W, H).raw_terms(which, nchunks=ns)
            num64, den64, _ = tcm.NmfdModel(self.V, W, H, rounding=False).raw_terms(which)
            r = tcm.nmfd_rtol64(self.seq.shape, self.V, W, H)
            return num, den, bar, None, num64, den64, r, r
        m = self.nmf_model(W, H)
        num, den, bar, dbar = m.raw_terms(which, beta, nchunks=self.nchunks(which))
        num64, den64, _, _ = self.nmf_model(W, H, rounding=False).raw_terms(which, beta)
        rn, rd = sc.rtol_terms(beta, tcm.RTOL64[self.path_prec(beta)])
        return num, den, bar, dbar, num64, den64, rn, rd

    def tc_update(self, tag, got, W, H, which, st):
        beta, gamma, l1, l2 = st[1:]
        num, den, bar, dbar, num64, den64, rn, rd = self.tc_terms(W, H, which, beta)
        p = (W if which == 0 else H).double()
        kl = beta == 1
        shape = (1, -1) + (1,) * (p.dim() - 2)
        want, mult = fc.ratio64(p, num, den.reshape(shape) if kl else den, gamma, l1, l2, kl)
        want64, _ = fc.ratio64(p, num64, den64.reshape(shape) if kl else den64, gamma, l1, l2, kl)
        rel = bar / num.abs()
        if dbar is not None:
            rel = rel + dbar / den.abs()
        if beta == 2:                             # fp32 Gram, its product with F, num + kappa den, the division
            kap = self.nmf_model(W, H).kappa
            rel = rel + U * (self.seq.shape[2] + 80) * (1 + kap * den.abs() / num.abs())
        elif kl:
            rel = rel + 64 * U                    # the fp32 column sums of the KL denominator
        rel = gamma * rel + fc.ratio_bar(mult, gamma)
        r64 = gamma * (rn + (rd if not kl else 0.0)) + 1e-5
        return tcm.check_terms(tag, got, want, want * rel, want64, r64)

    def tc_loss(self, tag, got, W, H, beta, fold):
        if self.seq.kind == "nmfd":
            model, exact = tcm.NmfdModel(self.V, W, H).loss(), tcm.NmfdModel(self.V, W, H, rounding=False).loss()[0]
            prec = "f16"
        else:
            prec = self.seq.precision if self.seq.precision != "auto" else "f16"
            model = tcm.NmfModel(self.V, W, H, prec).loss(beta, fold=fold)
            exact = tcm.NmfModel(self.V, W, H, prec, rounding=False).loss(beta)[0]
        return tcm.check_loss(tag, got, model, exact, prec, beta)

    # -- one step --------------------------------------------------------------------------------------------------------
    def __call__(self, i, plan, eng, before, out):
        st, seq = plan.step, self.seq
        op = st[0]
        tag = f"{seq.name}{sc.scale_tag(self.scale)}[{i}]{st}"
        W0, H0 = before
        beta = st[2] if op == "raw" else (st[1] if len(st) > 1 else None)
        if op == "rescale":
            return 0.0
        want_prec = self.path_prec(beta) if plan.reported == "tc" else "f32"
        if op != "shard":
            assert eng.precision_for(beta) == want_prec, f"{tag}: path {eng.precision_for(beta)}, expected {want_prec}"
        if plan.path == "f32" and op != "shard":
            e = self.f32_step(tag, eng, st, before, out)
        elif op == "raw":
            num, den, bar, dbar, num64, den64, rn, rd = self.tc_terms(W0, H0, st[1], beta)
            e = tcm.check_terms(tag + "num", out[0], num, bar, num64, rn)
            if dbar is not None:
                e = max(e, tcm.check_terms(tag + "den", out[1], den, dbar, den64, rd))
            else:
                assert torch.allclose(out[1].double().cpu(), den64.reshape(-1).cpu(), rtol=1e-5), tag + " column sums"
        elif op in ("loss", "prefetch"):
            fold = op == "prefetch" and seq.precision == "f16" and seq.kind == "nmf"
            e = self.tc_loss(tag, out, W0, H0, beta, fold)
        elif op in ("update_w", "update_h"):
            which = 0 if op == "update_w" else 1
            e = self.tc_update(tag, eng.W if which == 0 else eng.H, W0, H0, which, st)
        elif op == "iterate":
            e = self.tc_update(tag + "W", eng.W, W0, H0, 0, st)
            e = max(e, self.tc_update(tag + "H", eng.H, eng.W.detach().clone(), H0, 1, st))
        elif op == "shard":
            e = self.shard(tag, plan, eng, before, out)
        else:
            raise AssertionError(op)
        self.worst = max(self.worst, e)
        return e

    def shard(self, tag, plan, eng, before, out):
        W0, H0 = before
        beta, gamma, l1, l2 = plan.step[1:]
        C, R = W0.shape
        if plan.path == "tc":
            num, den, bar, dbar, num64, den64, rn, rd = self.tc_terms(W0, H0, 0, beta)
            e = tcm.check_terms(tag + "partial", out[:C * R].view(C, R), num, bar, num64, rn)
            if dbar is not None:
                e = max(e, tcm.check_terms(tag + "partial-den", out[C * R:].view(C, R), den, dbar, den64, rd))
        else:
            fresh = _fresh_f32(self.seq, eng, self.V_dev, W0, H0)
            try:
                assert torch.equal(out, fresh.w_partial(beta)), tag + ": w_partial differs from a fresh context's"
            finally:
                fresh.close()
            e = 0.0
        # w_apply: the ratio stage of exactly this buffer
        kl = beta == 1
        num = out[:C * R].view(C, R).double()
        den = out[C * R:].double().view(1, R) if kl else out[C * R:].double().view(C, R)
        want, mult = fc.ratio64(W0.double(), num, den, gamma, l1, l2, kl)
        err = float(((eng.W.double() - want).abs() / (fc.ratio_bar(mult, gamma) * want)).max())
        assert err <= 1.0, f"{tag}: w_apply {err:.2f} x the ratio-stage bar"
        return max(e, err)

    def f32_step(self, tag, eng, st, before, out):
        """Bits of the same call on a fresh fp32 context, then the a priori float64 bars of the fp32 kernels
        (tests/f32_cases.py) or of the sparse-target kernels (tests/sparse_cases.py)."""
        W0, H0 = before
        fresh = _fresh_f32(self.seq, eng, self.V_dev, W0, H0)
        try:
            ref = sc.call(fresh, st)
            if st[0] == "raw":
                assert all(torch.equal(a, b) for a, b in zip(out, ref)), tag + ": raw terms differ from a fresh context's"
            elif st[0] in ("loss", "prefetch"):
                assert out == ref, f"{tag}: loss {out!r} != fresh context's {ref!r}"
            else:
                assert torch.equal(eng.W, fresh.W) and torch.equal(eng.H, fresh.H), tag + ": factors differ from a fresh context's"
        finally:
            fresh.close()
        return F32Bars(self, eng).check(tag, st, eng, before, out)


class F32Bars:
    """The float64 bars the fp32 kernels are held to by their own suites, for one step of a sequence."""

    def __init__(self, chk, eng):
        self.chk, self.seq = chk, chk.seq
        self.sparse = isinstance(eng, E.CudaSparseNmfEngine)
        V64 = chk.V.cpu()
        self.V64 = V64
        if self.sparse:
            Vs = chk.V_dev.coalesce()
            self.rows, self.cols = Vs.indices()[0].cpu(), Vs.indices()[1].cpu()
            self.vals = Vs.values().double().cpu()

    def _nmfd_case(self):
        B, C, L, R, T = self.seq.shape
        return (B, C, (L,), R, (T,))

    def terms(self, W, H, which, beta):
        """(num, den, bar_num, bar_den): float64 terms at (W, H) and their relative bars (scalars or per-row tensors)."""
        W, H = W.double().cpu(), H.double().cpu()
        if self.sparse:
            N, C, R = self.seq.shape
            num, den = spc.sp_terms64(which, beta, self.rows, self.cols, self.vals, W, H)
            n = spc.seg_lengths(which, self.rows, self.cols, N, C)
            bn = spc.num_bar(beta, R, n)[:, None]
            if beta == 1:
                bd = fc.gam(N if which == 0 else C) + fc.U
            else:
                pl = _capi.sparse_plan(N, C, R)
                rpb, nb = (pl["rpb_n"], pl["nb_n"]) if which == 0 else (pl["rpb_c"], pl["nb_c"])
                bd = spc.den_bar(R, rpb, nb)
            return num, den, bn, bd
        num, den = sc.terms64(self.seq.kind, self.V64, W, H, which, beta)
        if self.seq.kind == "nmfd":
            case = self._nmfd_case()
            ks, nw, nh = fc.nmfd_terms(case)
            B, C, X, R, K = case
            pl = _capi.nmfd_plan(B, C, list(X), R, list(K))
            n, nch = (nw, pl["wgrad_nsplit"]) if which == 0 else (nh, pl["dgrad_nsplit"])
        else:
            N, C, R = self.seq.shape
            pl = _capi.nmf_plan(N, C, R)
            ks = R
            n, nch = (N, pl["nch_w"]) if which == 0 else (C, pl["nch_h"])
        bn, bd = fc.terms_bar(beta, ks, n, nch)
        return num, den, bn, bd

    def loss(self, W, H, beta):
        W, H = W.double().cpu(), H.double().cpu()
        if self.sparse:
            d = (self.rows, self.cols, self.vals, W, H)
            return spc.sp_loss64(beta, *d), spc.loss_bar(beta, *d)
        ks = fc.nmfd_terms(self._nmfd_case())[0] if self.seq.kind == "nmfd" else self.seq.shape[2]
        S = sc.recon64(self.seq.kind, W, H).reshape(-1)
        return fc.loss_bar(beta, S, self.V64.reshape(-1), ks, tcm.EPS)

    def _rel(self, tag, got, want, bar):
        got, want = got.double().cpu().reshape(want.shape), want.double()
        e = float(((got - want).abs() / (bar * want.abs()).clamp_min(1e-300)).max())
        assert e <= 1.0, f"{tag}: {e:.2f} x the fp32 float64 bar"
        return e

    def update(self, tag, got, W, H, which, st):
        beta, gamma, l1, l2 = st[1:]
        num, den, bn, bd = self.terms(W, H, which, beta)
        p = (W if which == 0 else H).double().cpu()
        kl = beta == 1
        want, mult = fc.ratio64(p, num, den.reshape((1, -1) + (1,) * (p.dim() - 2)) if kl else den, gamma, l1, l2, kl)
        return self._rel(tag, got, want, gamma * (bn + bd) + fc.ratio_bar(mult, gamma))

    def check(self, tag, st, eng, before, out):
        W0, H0 = before
        op = st[0]
        if op == "raw":
            which, beta = st[1:]
            num, den, bn, bd = self.terms(W0, H0, which, beta)
            e = self._rel(tag + "num", out[0], num, bn)
            return max(e, self._rel(tag + "den", out[1], den.reshape(-1) if beta == 1 else den, bd))
        if op in ("loss", "prefetch"):
            want, bar = self.loss(W0, H0, st[1])
            e = abs(out - want) / bar
            assert e <= 1.0, f"{tag}: loss {out!r} vs float64 {want!r}: {e:.2f} x the fp32 bar"
            return e
        if op == "iterate":                     # the H update starts from the new W
            e = self.update(tag + "W", eng.W, W0, H0, 0, st)
            return max(e, self.update(tag + "H", eng.H, eng.W.detach().clone(), H0, 1, st))
        which = 0 if op == "update_w" else 1
        return self.update(tag, eng.W if which == 0 else eng.H, W0, H0, which, st)


def _set_target_fn(seq, targets, chk):
    def set_target(eng, name):
        V = targets[name].cuda()
        chk.V_dev, chk.V = V, V.double()
        if isinstance(eng, E.CudaSparseNmfEngine):          # the dense engine takes over the sparse one's cached context
            ctx = eng._ctx.value
            W, H = eng.W, eng.H
            eng.close()
            eng = E.CudaNmfEngine(V, W, H, "f32")
            assert eng._ctx.value == ctx, "the workspace cache did not hand the sparse context on"
            return eng
        lib = _capi.load()
        _capi.check(lib.nmfb200_nmf_set_target(eng._ctx, ctypes.c_void_p(V.data_ptr()), V.stride(0), _capi.DTYPE_F32,
                                               ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
        eng.V = V
        return eng
    return set_target


def _check_launches(seq, plans, launches):
    """A W update at beta 1 on a valid prefetch launches one kernel fewer (its contraction) than one on clean operand copies
    without a prefetch; every other W update launches at least as many.  Both counts come from this context, whatever its
    ratio stage is (one fused cooperative kernel or two)."""
    uw = [(p, n) for p, n in zip(plans, launches)
          if p.step[0] == "update_w" and p.path == "tc" and p.step[1] == 1 and seq.kind == "nmf"]
    plain = sorted({n for p, n in uw if not p.reuse and not p.refresh})
    if not plain:
        assert not any(p.reuse for p, _ in uw), f"{seq.name}: no W update to compare a prefetched one with"
        return
    assert len(plain) == 1, f"{seq.name}: clean W updates launched {plain} kernels"
    for p, n in uw:
        if p.reuse:
            assert n == plain[0] - 1, f"{seq.name}: a W update on a valid prefetch launched {n} kernels, expected {plain[0] - 1}"
        else:
            assert n >= plain[0], f"{seq.name}: a W update launched {n} kernels: it skipped its contraction"


def _run(seq, scale=0, unbalanced=0):
    targets, W, H = sc.fitted_data(seq, scale, unbalanced)
    chk = Checker(seq, scale)
    V = targets["V"].cuda()
    chk.V_dev = V
    chk.V = (V.to_dense() if V.is_sparse else V).double()
    eng = _make(seq, V, W.cuda(), H.cuda())
    plans, launches = [], []

    def measure(plan, run_step):
        n0 = _capi.launch_count()
        out = run_step()
        launches.append(_capi.launch_count() - n0)
        plans.append(plan)
        return out
    try:
        eng, res = sc.run(seq, eng, chk, _set_target_fn(seq, targets, chk), measure)
    finally:
        eng.close()
    _check_launches(seq, plans, launches)
    _report(seq=seq.name, scale=scale, unbalanced=unbalanced, steps=len(res), worst_err_over_bar=chk.worst)
    return res


TC_SEQS = [s for s in sc.sequences() if s.tc]


@pytest.mark.parametrize("scale", sc.SCALES, ids=sc.scale_tag)
@pytest.mark.parametrize("name", [s.name for s in TC_SEQS if s.name != "target"])
def test_tensor_core_sequence(name, scale):
    _run(sc.by_name(name), scale)


@pytest.mark.parametrize("scale", sc.SCALES, ids=sc.scale_tag)
def test_tensor_core_sequence_with_a_new_dense_target(scale):
    """The "target" sequence: nmfb200_nmf_set_target registers a new fp32 target on a live tensor-core context."""
    _run(sc.by_name("target"), scale)


@pytest.mark.parametrize("name", ["fit-f16", "fit-split", "mixed-f16"])
def test_unbalanced_factors(name):
    """W 2^8 and H 2^-8: the operand exponents differ by 16, the product is unchanged."""
    _run(sc.by_name(name), 0, unbalanced=8)


def test_sparse_then_dense_on_one_context():
    _run(sc.by_name("sparse"), 0)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs in one process")
def test_nmfd_tensor_core_fit_on_two_devices():
    """The NMFD kernels opt into > 48 KB of shared memory per device: a fit on cuda:1 after one on cuda:0 must launch."""
    from oracle import mu_oracle as orc
    from torchnmf_b200 import NMFD
    g = torch.Generator().manual_seed(3)
    V = torch.rand(1, 20, 300, generator=g) + 0.1
    W0 = torch.rand(20, 4, 40, generator=g) + 0.1
    H0 = torch.rand(1, 4, 261, generator=g) + 0.1
    W, H, _, _ = orc.fit(V, W0, H0, beta=1, tol=float("-inf"), max_iter=5, kind="nmfd")
    for dev in ("cuda:0", "cuda:1"):
        m = NMFD(W=W0, H=H0).to(dev)
        m.fit(V.to(dev), 1, float("-inf"), 5, precision="f16")
        assert m.last_fit_precision == "f16"
        for got, want in ((m.W.data.cpu(), W), (m.H.data.cpu(), H)):
            assert torch.allclose(got, want, rtol=1e-3, atol=1e-5 * float(want.abs().max())), dev
