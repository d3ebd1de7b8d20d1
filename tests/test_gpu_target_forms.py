"""One NMF context taken through every target form the C ABI registers, in turn: a dense fp32 target, then a mask, a weight,
a sparse target (beta 1 / 2), a sparse target at any beta, weighted and unweighted observed cells, and a dense bf16 target.

After each set_target* (or set_mask / set_weight), every call the form serves -- raw_terms of W and of H, loss, update_w
and update_h at beta 0.5, 1 and 2 -- gives, bit for bit, what it gives on a fresh context that holds that form alone, and
so does target_minmax wherever the form sets it.  The form-dependent refusals return the same code and message on both:
nothing an earlier form registered (a selector, entry weights, the any-beta flag) leaks into a later one.
"""
import ctypes

import pytest
import torch

from torchnmf_b200 import _capi
from torchnmf_b200.engine import _compressed_forms

pytestmark = pytest.mark.gpu

N, C, R = 96, 80, 8
BETAS = (0.5, 1.0, 2.0)
ERR_INVALID, ERR_STATE = 1, 3          # include/nmf_b200.h


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _last_error():
    return _capi.load().nmfb200_last_error().decode()


def _data():
    g = torch.Generator().manual_seed(11)
    V = torch.rand(N, C, generator=g) + 0.1
    M = (torch.rand(N, C, generator=g) < 0.7).to(torch.uint8)
    Wt = torch.rand(N, C, generator=g) * 2
    Wt[torch.rand(N, C, generator=g) < 0.1] = 0.0
    S = V * (torch.rand(N, C, generator=g) < 0.3)
    obs = M.bool()
    O = torch.sparse_coo_tensor(obs.nonzero().t(), V[obs], (N, C)).coalesce()
    w_obs = Wt[O.indices()[0], O.indices()[1]] + 0.5
    W = torch.rand(C, R, generator=g) + 0.1
    H = torch.rand(N, R, generator=g) + 0.1
    dev = "cuda"
    return dict(V=V.to(dev), M=M.to(dev), Wt=Wt.to(dev), S=S.to_sparse().coalesce().to(dev), O=O.to(dev),
                w_obs=w_obs.to(dev), W=W.to(dev), H=H.to(dev))


class Ctx:
    """An fp32 NMF context and the tensors it borrows."""

    def __init__(self):
        self.lib = _capi.load()
        self.p = ctypes.c_void_p()
        _capi.check(self.lib.nmfb200_nmf_create(ctypes.byref(self.p), torch.cuda.current_device(), N, C, R,
                                                _capi.PREC_F32))
        self.keep = []

    def close(self):
        self.lib.nmfb200_destroy(self.p)


def _dense(ctx, d, dtype=torch.float32):
    V = d["V"].to(dtype).contiguous()
    ctx.keep.append(V)
    _capi.check(ctx.lib.nmfb200_nmf_set_target(ctx.p, _p(V), C, _capi.DTYPES[dtype], _st()))


def _sparse(ctx, d, symbol):
    forms = _compressed_forms(d["S"])
    ctx.keep.append(forms)
    v = forms[2].double()
    pos = v[v > 0]
    kl, eu = float((pos * pos.log()).sum() - v.sum()), float((v * v).sum() * 0.5)
    _capi.check(getattr(ctx.lib, symbol)(ctx.p, forms[2].numel(), *(_p(t) for t in forms), kl, eu, _st()))


def _observed(ctx, d, weighted):
    forms = _compressed_forms(d["O"], d["w_obs"] if weighted else None)
    ctx.keep.append(forms)
    nnz = forms[2].numel()
    if weighted:
        _capi.check(ctx.lib.nmfb200_nmf_set_target_observed_weighted(ctx.p, nnz, *(_p(t) for t in forms), _st()))
    else:
        _capi.check(ctx.lib.nmfb200_nmf_set_target_observed(ctx.p, nnz, *(_p(t) for t in forms), _st()))


def _select(ctx, d, name):
    t = d[name]
    ctx.keep.append(t)
    fn = ctx.lib.nmfb200_set_mask if name == "M" else ctx.lib.nmfb200_set_weight
    _capi.check(fn(ctx.p, _p(t), _st()))


# (name, what it registers on a context that holds the previous form, what registers it on a fresh one, betas it serves,
#  whether it sets target_minmax)
FORMS = [
    ("dense-f32", lambda c, d: _dense(c, d), lambda c, d: _dense(c, d), BETAS, True),
    ("mask", lambda c, d: _select(c, d, "M"), lambda c, d: (_dense(c, d), _select(c, d, "M")), BETAS, True),
    ("weight", lambda c, d: _select(c, d, "Wt"), lambda c, d: (_dense(c, d), _select(c, d, "Wt")), BETAS, True),
    ("sparse", lambda c, d: _sparse(c, d, "nmfb200_nmf_set_target_sparse"), None, (1.0, 2.0), False),
    ("sparse-any-beta", lambda c, d: _sparse(c, d, "nmfb200_nmf_set_target_sparse_any_beta"), None, BETAS, False),
    ("observed-weighted", lambda c, d: _observed(c, d, True), None, BETAS, True),
    ("observed", lambda c, d: _observed(c, d, False), None, BETAS, True),
    ("dense-bf16", lambda c, d: _dense(c, d, torch.bfloat16), None, BETAS, True),
]


def _results(ctx, d, betas, minmax):
    """Every output the form serves, from fresh copies of the same starting factors."""
    lib, out = ctx.lib, []
    for beta in betas:
        for which in (0, 1):
            n = int(lib.nmfb200_raw_terms_numel(ctx.p, which, beta))
            buf = torch.empty(n, dtype=torch.float32, device="cuda")
            _capi.check(lib.nmfb200_raw_terms(ctx.p, _p(d["W"]), _p(d["H"]), which, beta, _p(buf), _st()))
            out.append((f"raw_terms which={which} beta={beta}", buf))
        loss = torch.zeros(1, dtype=torch.float64, device="cuda")
        _capi.check(lib.nmfb200_loss(ctx.p, _p(d["W"]), _p(d["H"]), beta, _p(loss), _st()))
        out.append((f"loss beta={beta}", loss))
        for which, fn in ((0, lib.nmfb200_update_w), (1, lib.nmfb200_update_h)):
            W, H = d["W"].clone(), d["H"].clone()
            _capi.check(fn(ctx.p, _p(W), _p(H), beta, 1.0, 0.0, 0.0, _st()))
            out.append((f"update which={which} beta={beta}", W if which == 0 else H))
    if minmax:
        lo, hi = ctypes.c_float(), ctypes.c_float()
        _capi.check(lib.nmfb200_target_minmax(ctx.p, ctypes.byref(lo), ctypes.byref(hi), _st()))
        out.append(("target_minmax", torch.tensor([lo.value, hi.value])))
    return out


def _refusals(ctx, d, form):
    """(code, message or None) of each form-dependent check; set_mask only where it refuses (it would change the form)."""
    lib = ctx.lib
    W, H = d["W"].clone(), d["H"].clone()
    buf = torch.empty(2 * N * R, dtype=torch.float32, device="cuda")
    probes = {
        "cd_update": lambda: lib.nmfb200_nmf_cd_update(ctx.p, _p(W), _p(H), 0, 0.0, 0.0, _st()),
        "contract_only": lambda: lib.nmfb200_nmf_contract_only(ctx.p, _p(W), _p(H), 0, 1.0, _st()),
        "plca_masked_terms": lambda: lib.nmfb200_plca_masked_terms(ctx.p, _p(W), _p(H), 1, _p(buf), None, _st()),
        "raw_terms beta=0.5": lambda: lib.nmfb200_raw_terms(ctx.p, _p(W), _p(H), 1, 0.5, _p(buf), _st()),
    }
    if form.startswith(("sparse", "observed")):
        probes["set_mask"] = lambda: lib.nmfb200_set_mask(ctx.p, _p(d["M"]), _st())
    got = {}
    for name, call in probes.items():
        rc = int(call())
        got[name] = (rc, _last_error() if rc else None)
    return got


SPARSE_FORMS = ("sparse", "sparse-any-beta", "observed-weighted", "observed")
# the refusals whose code and message the form decides (include/nmf_b200.h)
EXPECTED = {
    "set_mask": {f: (ERR_INVALID, "a mask needs a dense target (set_target or nmfd_set_target)") for f in SPARSE_FORMS},
    "cd_update": {f: (ERR_INVALID, "cd: observed-cell targets are not served") for f in SPARSE_FORMS[2:]},
    "contract_only": {f: (ERR_STATE, "not available for a sparse target") for f in SPARSE_FORMS},
    "plca_masked_terms": {f: (ERR_INVALID, "plca_masked_terms needs a dense target") for f in SPARSE_FORMS},
    "raw_terms beta=0.5": {"sparse": (ERR_INVALID, "sparse targets: beta must be 1 or 2 (densify the target for other beta)")},
}


def test_every_target_form_on_one_context():
    d = _data()
    live = Ctx()
    try:
        for name, on_live, on_fresh, betas, minmax in FORMS:
            on_live(live, d)
            fresh = Ctx()
            try:
                (on_fresh or on_live)(fresh, d)
                got, want = _results(live, d, betas, minmax), _results(fresh, d, betas, minmax)
                for (what, a), (_, b) in zip(got, want):
                    assert torch.equal(a, b), f"{name}: {what} differs from a fresh context's"
                got_r, want_r = _refusals(live, d, name), _refusals(fresh, d, name)
                assert got_r == want_r, f"{name}: refusals {got_r} != a fresh context's {want_r}"
                for probe, forms in EXPECTED.items():
                    if name in forms:
                        assert got_r[probe] == forms[name], f"{name}: {probe} returned {got_r[probe]}"
            finally:
                fresh.close()
    finally:
        live.close()
