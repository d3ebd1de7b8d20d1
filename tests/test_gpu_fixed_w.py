"""Fixed components of W (`fit(V, ..., fixed_W=F)`, `nmfb200_set_fixed_w`) on the GPU.

One W update from the same W and H, with and without `fixed_W`: on the multiplicative and EM paths every free column equals
the plain update's bit for bit and every fixed column its input; coordinate descent, which skips each fixed k inside the
sweep, is held to a float64 skip oracle within test_gpu_cd.py's per-entry bound.  Then whole fits: none fixed is the plain
fit, all fixed is trainable_W=False, a planted separation problem, repeated fits on a cached context, and the ABI refusals.
"""
import ctypes

import pytest
import torch

from test_gpu_cd import U, _planted
from torchnmf_b200 import NMF, NMF2D, NMF3D, NMFD, PLCA, SIPLCA, _capi

pytestmark = pytest.mark.gpu

RANKS = [1, 17, 64, 129]


def _sets(R):
    """First-k, last-k and scattered fixed sets (at least one free component); R = 1: the one component fixed."""
    if R == 1:
        return {"all": [0]}
    k = max(1, R // 2)
    return {"first": list(range(k)), "last": list(range(R - k, R)), "scattered": list(range(0, R - 1, 3))}


def _flags(R, idx):
    F = torch.zeros(R, dtype=torch.bool)
    F[idx] = True
    return F


def _nmf_target(N, C, R, seed, kind="f32"):
    g = torch.Generator().manual_seed(seed)
    V = torch.rand(N, C, generator=g) + 0.05
    W, H = torch.rand(C, R, generator=g) + 0.1, torch.rand(N, R, generator=g) + 0.1
    Vd = V.cuda()
    if kind == "bf16":
        Vd = Vd.bfloat16()
    elif kind == "strided":
        Vd = torch.cat([Vd, torch.ones(N, 5, device="cuda")], 1)[:, :C]
    return Vd, W, H


def _after_one(cls, W, H, V, F=None, module_kw=None, **fit_kw):
    """W after one iteration of fit (the W update comes first, from W and H as given)."""
    m = cls(W=W.clone(), H=H.clone(), **(module_kw or {})).cuda()
    extra = {} if F is None else {"fixed_W": F}
    m.fit(V, tol=float("-inf"), max_iter=1, **fit_kw, **extra)
    return m.W.data.cpu()


def _check_mu(W0, plain, got, F):
    assert torch.equal(got[:, F], W0[:, F]), "a fixed column moved"
    assert torch.equal(got[:, ~F], plain[:, ~F]), float((got[:, ~F] - plain[:, ~F]).abs().max())


# ---- one update, multiplicative ------------------------------------------------------------------------------------------

@pytest.mark.parametrize("R", RANKS)
@pytest.mark.parametrize("precision,beta", [("f32", 1), ("f32", 2), ("f32", 0.5), ("f16", 1), ("f16", 2), ("f16", 0.5),
                                            ("f16_split", 1)])
def test_nmf_mu_update(R, precision, beta):
    if precision != "f32" and R > 128:
        pytest.skip("the tensor-core path takes R <= 128")
    V, W, H = _nmf_target(300, 257, R, seed=R)
    plain = _after_one(NMF, W, H, V, beta=beta, precision=precision)
    for name, idx in _sets(R).items():
        F = _flags(R, idx)
        got = _after_one(NMF, W, H, V, F, beta=beta, precision=precision)
        if bool(F.all()):
            assert torch.equal(got, W)
        else:
            _check_mu(W, plain, got, F)


@pytest.mark.parametrize("kind", ["bf16", "strided"])
@pytest.mark.parametrize("R", [17, 64])
@pytest.mark.parametrize("precision", ["f32", "f16"])
def test_nmf_mu_update_half_and_strided_targets(kind, R, precision):
    V, W, H = _nmf_target(200, 130, R, seed=3 * R, kind=kind)
    plain = _after_one(NMF, W, H, V, beta=1, precision=precision)
    F = _flags(R, _sets(R)["scattered"])
    _check_mu(W, plain, _after_one(NMF, W, H, V, F, beta=1, precision=precision), F)


@pytest.mark.parametrize("beta", [0.5, 1, 2])
@pytest.mark.parametrize("R", [1, 17, 64, 129])
def test_sparse_target_mu_update(beta, R):
    V, W, H = _nmf_target(180, 150, R, seed=R + 11)
    V = torch.where(V > 0.6, V, torch.zeros((), device="cuda")).to_sparse()
    plain = _after_one(NMF, W, H, V, beta=beta)
    for idx in _sets(R).values():
        F = _flags(R, idx)
        got = _after_one(NMF, W, H, V, F, beta=beta)
        if bool(F.all()):
            assert torch.equal(got, W)
        else:
            _check_mu(W, plain, got, F)


@pytest.mark.parametrize("sel", ["mask", "weight", "sparse_mask", "sparse_weight"])
@pytest.mark.parametrize("R", [17, 64])
@pytest.mark.parametrize("beta", [1, 2])
def test_selected_cells_mu_update(sel, R, beta):
    V, W, H = _nmf_target(160, 140, R, seed=R + beta)
    g = torch.Generator().manual_seed(R)
    M = torch.rand(V.shape, generator=g) > 0.3
    kw = {"mask": M} if "mask" in sel else {"weight": M.float() * (torch.rand(V.shape, generator=g) + 0.5)}
    if sel.startswith("sparse"):
        kw = {k: v.to_sparse() for k, v in kw.items()}
    kw = {k: v.cuda() for k, v in kw.items()}
    plain = _after_one(NMF, W, H, V, beta=beta, **kw)
    F = _flags(R, _sets(R)["first"])
    _check_mu(W, plain, _after_one(NMF, W, H, V, F, beta=beta, **kw), F)


def _conv_case(cls, R, seed):
    g = torch.Generator().manual_seed(seed)
    if cls is NMFD:
        return torch.rand(2, 40, 90, generator=g).cuda(), torch.rand(40, R, 8, generator=g) + 0.1, torch.rand(2, R, 83, generator=g) + 0.1
    if cls is NMF2D:
        return (torch.rand(1, 6, 20, 40, generator=g).cuda(), torch.rand(6, R, 3, 4, generator=g) + 0.1,
                torch.rand(1, R, 18, 37, generator=g) + 0.1)
    return (torch.rand(1, 3, 8, 9, 10, generator=g).cuda(), torch.rand(3, R, 2, 2, 3, generator=g) + 0.1,
            torch.rand(1, R, 7, 8, 8, generator=g) + 0.1)


@pytest.mark.parametrize("cls,precision,beta", [(NMFD, "f32", 1), (NMFD, "f32", 2), (NMFD, "auto", 1), (NMFD, "f16", 1),
                                                (NMF2D, "f32", 1), (NMF2D, "f16", 1), (NMF2D, "f32", 0.5),
                                                (NMF3D, "f32", 1), (NMF3D, "f32", 2)])
@pytest.mark.parametrize("R", [1, 17, 64])
def test_convolutive_mu_update(cls, precision, beta, R):
    V, W, H = _conv_case(cls, R, seed=R)
    plain = _after_one(cls, W, H, V, beta=beta, precision=precision)
    for idx in _sets(R).values():
        F = _flags(R, idx)
        got = _after_one(cls, W, H, V, F, beta=beta, precision=precision)
        if bool(F.all()):
            assert torch.equal(got, W)
        else:
            _check_mu(W, plain, got, F)


# ---- one update, coordinate descent ----------------------------------------------------------------------------------------

def _skip_sweep(A, B, X, F, l1, l2):
    """HALS sweep of X (float64, rows x R) with per-row Grams B (rows x R x R) or one Gram (R x R), skipping fixed k."""
    X = X.double().clone()
    Bb = B if B.dim() == 3 else B.expand(X.shape[0], *B.shape)
    for k in range(X.shape[1]):
        if bool(F[k]):
            continue
        hess = Bb[:, k, k] + l2
        step = (A[:, k] - (Bb[:, :, k] * X).sum(1) - l1 - l2 * X[:, k]) / hess
        X[:, k] = torch.where(hess != 0, (X[:, k] + step).clamp_min(0.0), X[:, k])
    return X


@pytest.mark.parametrize("R", RANKS)
@pytest.mark.parametrize("target", ["dense", "sparse", "observed"])
def test_cd_update_against_float64_skip_oracle(R, target):
    if R > 128 and target != "dense":
        R = 100                       # the sparse and observed cd kernels serve R <= 256; keep the oracle small
    N, C, l1, l2 = 400, 300, 0.5, 0.25
    V, W, H = _planted(N, C, R, seed=R + len(target))
    g = torch.Generator().manual_seed(R)
    M = torch.rand(N, C, generator=g) > 0.4 if target == "observed" else torch.ones(N, C, dtype=torch.bool)
    if target == "sparse":
        V = torch.where(V > V.median(), V, torch.zeros(()))
    Vd = V.cuda().to_sparse() if target == "sparse" else V.cuda()
    kw = {"mask": M.to_sparse().cuda()} if target == "observed" else {}
    Mf = M.double()
    A = (Mf * V.double()).t() @ H.double()                              # C x R
    B = torch.einsum("nc,nr,ns->crs", Mf, H.double(), H.double())       # C x R x R
    for idx in _sets(R).values():
        F = _flags(R, idx)
        m = NMF(W=W.clone(), H=H.clone()).cuda()
        m.fit(Vd, 2, float("-inf"), 1, False, 0.75, 2 / 3, solver="cd", fixed_W=F, **kw)
        got = m.W.data.cpu().double()
        X64 = _skip_sweep(A, B, W, F, l1, l2)
        K = N
        diag = torch.diagonal(B, dim1=1, dim2=2)
        bound = 8 * (K + R + 4) * U * (A + torch.einsum("cr,crs->cs", X64.abs(), B)) / (diag + l2)
        assert torch.equal(got[:, F], W.double()[:, F])
        assert ((got - X64).abs() <= bound).all(), float(((got - X64).abs() / bound).max())


# ---- one update, EM ----------------------------------------------------------------------------------------------------------

def _plca_after_one(cls, V, W, H, Z, F=None, **kw):
    """(W as the module holds it before the fit -- normalised -- and W after one EM step)."""
    m = cls(W=W.clone(), H=H.clone(), Z=Z.clone()).cuda()
    W0 = m.W.data.cpu().clone()
    m.fit(V, float("-inf"), 1, **({} if F is None else {"fixed_W": F}), **kw)
    return W0, m.W.data.cpu()


@pytest.mark.parametrize("target", ["dense", "sparse", "masked", "siplca"])
@pytest.mark.parametrize("R", [1, 17, 64, 129])
def test_em_update(target, R):
    g = torch.Generator().manual_seed(R)
    kw = {}
    if target == "siplca":
        cls, V = SIPLCA, torch.rand(2, 30, 70, generator=g).cuda()
        W, H = torch.rand(30, R, 6, generator=g), torch.rand(2, R, 65, generator=g)
    else:
        cls, V = PLCA, torch.rand(150, 120, generator=g).cuda()
        W, H = torch.rand(120, R, generator=g), torch.rand(150, R, generator=g)
        if target == "sparse":
            V = torch.where(V > 0.5, V, torch.zeros((), device="cuda")).to_sparse()
        if target == "masked":
            kw["mask"] = (torch.rand(V.shape, generator=g) > 0.2).cuda()
    Z = torch.rand(R, generator=g) + 0.1
    W0, plain = _plca_after_one(cls, V, W, H, Z, **kw)
    for idx in _sets(R).values():
        F = _flags(R, idx)
        _, got = _plca_after_one(cls, V, W, H, Z, F, **kw)
        if bool(F.all()):
            assert torch.equal(got, W0)
        else:
            _check_mu(W0, plain, got, F)


# ---- whole fits --------------------------------------------------------------------------------------------------------------

def _fit(cls, W, H, V, **kw):
    m = cls(W=W.clone(), H=H.clone(), **kw.pop("module_kw", {})).cuda()
    n = m.fit(V, **kw)
    return n, m.W.data.cpu(), m.H.data.cpu()


@pytest.mark.parametrize("precision,beta,solver", [("auto", 1, "mu"), ("f16_split", 1, "mu"), ("f32", 0.5, "mu"),
                                                   ("f32", 2, "cd")])
def test_none_fixed_is_plain_and_all_fixed_is_frozen_w(precision, beta, solver):
    V, W, H = _nmf_target(500, 300, 32, seed=5)
    kw = dict(beta=beta, tol=1e-5, max_iter=60, precision=precision, solver=solver)
    plain = _fit(NMF, W, H, V, **kw)
    none = _fit(NMF, W, H, V, fixed_W=torch.zeros(32, dtype=torch.bool), **kw)
    frozen = _fit(NMF, W, H, V, module_kw={"trainable_W": False}, **kw)
    allf = _fit(NMF, W, H, V, fixed_W=torch.ones(32, dtype=torch.bool).cuda(), **kw)
    for a, b in ((plain, none), (frozen, allf)):
        assert a[0] == b[0] and torch.equal(a[1], b[1]) and torch.equal(a[2], b[2])
    assert torch.equal(allf[1], W)


def test_plca_none_and_all_fixed():
    g = torch.Generator().manual_seed(2)
    V, W, H, Z = torch.rand(200, 100, generator=g).cuda(), torch.rand(100, 8, generator=g), torch.rand(200, 8, generator=g), \
        torch.rand(8, generator=g)

    def run(F=None, **mk):
        m = PLCA(W=W.clone(), H=H.clone(), Z=Z.clone(), **mk).cuda()
        n, _ = m.fit(V, 1e-6, 40, **({} if F is None else {"fixed_W": F}))
        return n, m.W.data.cpu(), m.H.data.cpu(), m.Z.data.cpu()
    for a, b in ((run(), run(torch.zeros(8, dtype=torch.bool))), (run(trainable_W=False), run(torch.ones(8, dtype=torch.bool)))):
        assert a[0] == b[0] and all(torch.equal(x, y) for x, y in zip(a[1:], b[1:]))


def test_planted_separation_recovers_the_free_part():
    # V = H_k W_k^T (a known source on a fixed dictionary) + H_f W_f^T (the rest); the fit starts from the true W_k and a
    # random W_f.  Stated error: the free part H_f W_f^T within 2 % of its Frobenius norm after 300 cd iterations.
    g = torch.Generator().manual_seed(7)
    N, C, Rk, Rf = 600, 257, 12, 4

    def fac(rows, R):
        X = 0.05 * torch.rand(rows, R, generator=g)
        X[torch.arange(rows), torch.arange(rows) % R] += 1.0 + torch.rand(rows, generator=g)
        return X
    Wk, Wf, Hk, Hf = fac(C, Rk), fac(C, Rf)[torch.randperm(C, generator=g)], fac(N, Rk), fac(N, Rf)[torch.randperm(N, generator=g)]
    V = Hk @ Wk.t() + Hf @ Wf.t()
    W0 = torch.cat([Wk, torch.rand(C, Rf, generator=g) + 0.1], 1)
    F = torch.arange(Rk + Rf) < Rk
    m = NMF(W=W0, H=torch.rand(N, Rk + Rf, generator=g) + 0.1).cuda()
    m.fit(V.cuda(), 2, 0.0, 300, solver="cd", fixed_W=F)
    W, H = m.W.data.cpu(), m.H.data.cpu()
    assert torch.equal(W[:, F], Wk)
    free, want = H[:, ~F] @ W[:, ~F].t(), Hf @ Wf.t()
    err = float((free - want).norm() / want.norm())
    assert err < 2e-2, err


def test_cached_context_repeats_and_then_fits_plain():
    V, W, H = _nmf_target(400, 256, 64, seed=9)
    F = _flags(64, list(range(0, 64, 5)))
    kw = dict(beta=1, tol=float("-inf"), max_iter=25, precision="f16")
    a = _fit(NMF, W, H, V, fixed_W=F, **kw)
    b = _fit(NMF, W, H, V, fixed_W=F, **kw)
    assert torch.equal(a[1], b[1]) and torch.equal(a[2], b[2])
    assert torch.equal(a[1][:, F], W[:, F])
    plain1 = _fit(NMF, W, H, V, **kw)
    from torchnmf_b200 import engine
    engine.release_workspaces()
    plain2 = _fit(NMF, W, H, V, **kw)                  # on a fresh context
    assert torch.equal(plain1[1], plain2[1]) and torch.equal(plain1[2], plain2[2])


# ---- the C ABI ---------------------------------------------------------------------------------------------------------------

def test_abi_refusals_and_peer_report():
    lib = _capi.load()
    dev = torch.cuda.current_device()
    fixed = torch.ones(16, dtype=torch.uint8, device="cuda")
    fp = ctypes.c_void_p(fixed.data_ptr())
    ctx = ctypes.c_void_p()
    assert lib.nmfb200_nmf_create(ctypes.byref(ctx), dev, 256, 256, 16, _capi.PREC_F16) == 0
    try:
        assert lib.nmfb200_set_fixed_w(ctx, fp, None) == 3                      # NMFB200_ERR_STATE: no target yet
        V = torch.rand(256, 256, device="cuda")
        assert lib.nmfb200_nmf_set_target(ctx, ctypes.c_void_p(V.data_ptr()), 256, 0, None) == 0
        peer = lib.nmfb200_nmf_peer_supported(ctx, 1.0)
        assert lib.nmfb200_set_fixed_w(ctx, fp, None) == 0
        assert lib.nmfb200_nmf_peer_supported(ctx, 1.0) == 0
        assert lib.nmfb200_set_fixed_w(ctx, None, None) == 0
        assert lib.nmfb200_nmf_peer_supported(ctx, 1.0) == peer
        torch.cuda.synchronize()
    finally:
        lib.nmfb200_destroy(ctx)
    for create in (lambda c: lib.nmfb200_nmf_batched_create(ctypes.byref(c), dev, 2, 64, 64, 16),
                   lambda c: lib.nmfb200_plca_sparse_create(ctypes.byref(c), dev, 64, 64, 16, 100)):
        c = ctypes.c_void_p()
        assert create(c) == 0
        try:
            assert lib.nmfb200_set_fixed_w(c, fp, None) == 1                    # NMFB200_ERR_INVALID
        finally:
            lib.nmfb200_destroy(c)
