"""Coordinate descent at beta 2 on the observed cells, on the GPU (`NMF.fit(V, beta=2, solver="cd", mask=M)` with a sparse
mask or weight; include/nmf_b200.h: nmfb200_nmf_observed_cd_*).

* One update against the float64 oracle (tests/observed_cd_oracle.py) at every rank branch and segment length, within a bound
  derived per entry from the kernel's summation orders (csrc/observed_cd.cu).
* Whole fits against the oracle, bit-for-bit repeatability across runs, selectors and target forms, and the dense solver.
* The loss trace, a planted completion problem, the ABI's refusals and the memory of a large fit.
"""
import ctypes

import pytest
import torch

import observed_cd_oracle as ocd

pytestmark = pytest.mark.gpu

U = 2.0 ** -24                     # fp32 unit roundoff


def _segments(N, C, density, seed):
    """A mask (N, C) of `density` whose row 0 and column 0 are fully observed (segments longer than 1024 when N, C > 1024),
    row 1 and column 1 empty, every other segment short."""
    g = torch.Generator().manual_seed(seed)
    M = torch.rand(N, C, generator=g) < density
    M[0, :] = True
    M[:, 0] = True
    M[1, :] = False
    M[:, 1] = False
    return M


def _planted_factors(rows, R, gen):
    X = 0.05 * torch.rand(rows, R, generator=gen)
    X[torch.arange(rows), torch.arange(rows) % R] += 1.0 + torch.rand(rows, generator=gen)
    return X


def _engine(O, W, H, weights=None):
    from torchnmf_b200.engine import CudaObservedNmfEngine
    return CudaObservedNmfEngine(O.cuda(), W, H, weights=None if weights is None else weights.cuda())


def _observed(V, M, Wt=None):
    """(O, weights) of the cells M: the coalesced observed-cell tensor and its entries' weights (Wt at those cells)."""
    idx = M.nonzero().t()
    O = torch.sparse_coo_tensor(idx, V[M].float(), V.shape).coalesce()
    return O, (None if Wt is None else Wt[M].float().contiguous())


def _bound(V, Mw, W, H, which, X64, l1, l2):
    """Per-entry bound on |fp32 update - float64 update| (rows x R).  A column step's numerator sums K_s + R + 4 rounded
    terms (the residual's R-term dot and its group corrections, then K_s products), each within u of the magnitudes
    a_s = sum w |v| |f_k| and b_s = sum w (|x_s| . |f_j|) |f_k|; it is divided by hess = sum w f_k^2 + l2.  An earlier
    column's error e_i enters column k through G[i,k] / hess (the in-group correction and the residual update alike):
    e_k = 4 (K_s + R + 4) u (a_s + b_s + l1 + l2 |x|) / hess + sum_{i<k} |G[i,k]| e_i / hess, plus u |x| for the store."""
    n, c = Mw.nonzero(as_tuple=True)
    v, w = V[n, c].double(), Mw[n, c].double()
    seg, oth = (c, n) if which == 0 else (n, c)
    F = (H if which == 0 else W).double()
    Fo = F[oth].abs()
    rows, R = X64.shape
    K = torch.zeros(rows, dtype=torch.float64).index_add_(0, seg, torch.ones_like(w))
    xf = (X64.abs()[seg] * Fo).sum(1)
    e = torch.zeros(rows, R, dtype=torch.float64)
    for k in range(R):
        a = torch.zeros(rows, dtype=torch.float64).index_add_(0, seg, w * v.abs() * Fo[:, k])
        b = torch.zeros(rows, dtype=torch.float64).index_add_(0, seg, w * xf * Fo[:, k])
        hess = torch.zeros(rows, dtype=torch.float64).index_add_(0, seg, w * Fo[:, k] * Fo[:, k]) + l2
        hs = torch.where(hess > 0, hess, torch.ones_like(hess))
        Gk = torch.zeros(rows, R, dtype=torch.float64).index_add_(0, seg, (w * Fo[:, k])[:, None] * Fo) if k else None
        prop = (Gk[:, :k] * e[:, :k]).sum(1) if k else 0.0
        e[:, k] = torch.where(hess > 0, (4 * (K + R + 4) * U * (a + b + l1 + l2 * X64[:, k].abs()) + prop) / hs, 0.0)
    return e + U * X64.abs()


@pytest.mark.parametrize("R", [1, 17, 31, 32, 33, 64, 100, 256])
@pytest.mark.parametrize("which", [0, 1])
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("l1,l2", [(0.0, 0.0), (0.3, 0.2)])
def test_one_update_matches_float64(R, which, weighted, l1, l2):
    N, C = 1100, 1060
    gen = torch.Generator().manual_seed(R * 4 + which * 2 + weighted)
    M = _segments(N, C, 0.005, seed=R)
    W, H = _planted_factors(C, R, gen), _planted_factors(N, R, gen)
    V = (_planted_factors(N, R, gen) @ _planted_factors(C, R, gen).t() + 0.01 * torch.rand(N, C, generator=gen)).float()
    Wt = (0.25 + 2 * torch.rand(N, C, generator=gen)) if weighted else None
    Mw = M.double() * (Wt.float().double() if weighted else 1.0)
    X64 = ocd.update(V.double(), Mw, W.double(), H.double(), which, l1, l2)
    bound = _bound(V.double(), Mw, W, H, which, X64, l1, l2)
    O, wts = _observed(V, M, Wt)
    Wd, Hd = W.cuda(), H.cuda()
    eng = _engine(O, Wd, Hd, wts)
    try:
        eng.cd_update(which, l1, l2)
    finally:
        eng.close()
    got = (Wd if which == 0 else Hd).cpu().double()
    X0 = (W if which == 0 else H).double()
    assert torch.isfinite(got).all()
    empty = 1                                          # row / column 1 observes nothing
    if l2 == 0:
        assert torch.equal(got[empty], X0[empty])
    err = (got - X64).abs()
    assert (err <= bound).all(), float((err / bound.clamp_min(1e-300)).max())


def _completion(N, C, R, density, seed, noise=0.01):
    """A planted completion problem: V = H* W*^T + noise, the observed cells M (each row and column observed), fp32 starting
    factors."""
    gen = torch.Generator().manual_seed(seed)
    V = _planted_factors(N, R, gen) @ _planted_factors(C, R, gen).t() + noise * torch.rand(N, C, generator=gen)
    M = torch.rand(N, C, generator=gen) < density
    M[torch.arange(N), torch.arange(N) % C] = True
    return V.float(), M, torch.rand(C, R, generator=gen) + 0.1, torch.rand(N, R, generator=gen) + 0.1


def _fit_tolerance(X):
    return 2e-4 * float(X.abs().max())


def _fit(V, sel, W0, H0, **kw):
    from torchnmf_b200 import NMF
    m = NMF(W=W0, H=H0, trainable_W=kw.pop("trainable_W", True), trainable_H=kw.pop("trainable_H", True))
    if kw.pop("cuda", True):
        m = m.cuda()
    if kw.pop("double", False):
        m = m.double()
    n = m.fit(V, 2, kw.pop("tol", 1e-4), kw.pop("max_iter", 60), False, kw.pop("alpha", 0.1), kw.pop("l1_ratio", 0.3),
              solver=kw.pop("solver", "cd"), **sel, **kw)
    return n, m.W.data, m.H.data


@pytest.mark.parametrize("seed", [0, 1])
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("alpha,l1_ratio", [(0.0, 0.0), (1.0, 0.5)])
def test_whole_fit_matches_float64(seed, weighted, alpha, l1_ratio):
    V, M, W0, H0 = _completion(400, 300, 12, 0.3, seed=100 + seed)
    gen = torch.Generator().manual_seed(seed)
    Wt = (0.5 + torch.rand(V.shape, generator=gen)) * M
    sel = {"weight": Wt.to_sparse().cuda()} if weighted else {"mask": M.to_sparse().cuda()}
    n, W, H = _fit(V.cuda(), sel, W0, H0, tol=1e-3, max_iter=200, alpha=alpha, l1_ratio=l1_ratio)
    Mw = Wt.double() if weighted else M.double()
    W64, H64, n_ref, _ = ocd.fit(V.double(), Mw, W0.double(), H0.double(), 1e-3, 200, alpha * l1_ratio,
                                 alpha * (1 - l1_ratio))
    assert n == n_ref
    for got, want in ((W.cpu().double(), W64), (H.cpu().double(), H64)):
        assert (got - want).abs().max() <= _fit_tolerance(want)


@pytest.mark.parametrize("R", [20, 48])
def test_bit_exact_runs_selectors_targets_and_modules(R):
    V, M, W0, H0 = _completion(500, 333, R, 0.2, seed=7)
    V = V.bfloat16().float()                                        # exact in bf16
    Vc, Ms = V.cuda(), {"mask": M.to_sparse().cuda()}
    n, W, H = _fit(Vc, Ms, W0, H0)
    n2, W2, H2 = _fit(Vc, Ms, W0, H0)                               # two runs
    assert n == n2 and torch.equal(W, W2) and torch.equal(H, H2)
    unit = torch.sparse_coo_tensor(M.nonzero().t(), torch.ones(int(M.sum())), M.shape).cuda()
    nu, Wu, Hu = _fit(Vc, {"weight": unit}, W0, H0)                 # a unit weight on the mask's cells
    assert nu == n and torch.equal(Wu, W) and torch.equal(Hu, H)
    Vs = torch.full((500, 340), float("nan"), device="cuda")
    Vs[:, :333] = Vc
    for target in (Vc.bfloat16(), Vs[:, :333], Vc.double(), (Vc * M.cuda()).to_sparse()):
        nt, Wt, Ht = _fit(target, Ms, W0, H0)
        assert nt == n and torch.equal(Wt, W) and torch.equal(Ht, H)
    nh, Wh, Hh = _fit(V, {"mask": M.to_sparse()}, W0, H0, cuda=False)   # a host module is written back
    assert nh == n and Wh.device.type == "cpu" and torch.equal(Wh, W.cpu()) and torch.equal(Hh, H.cpu())
    n64, W64, H64 = _fit(Vc, Ms, W0, H0, double=True)
    assert n64 == n and W64.dtype == torch.float64 and torch.equal(W64, W.double()) and torch.equal(H64, H.double())
    for frozen in ("W", "H"):
        _, Wz, Hz = _fit(Vc, Ms, W0, H0, trainable_W=frozen != "W", trainable_H=frozen != "H")
        assert torch.equal((Wz if frozen == "W" else Hz).cpu(), W0 if frozen == "W" else H0)


def test_fully_observed_mask_agrees_with_the_dense_solver():
    # The two solvers differ only in their fp32 summation orders.  At alpha = 0 the objective is flat along W D, H D^-1 (D a
    # positive diagonal), and neither solver fixes that scale, so rounding can move a component's scale between W and H: the
    # reconstruction H W^T is what the fits pin down, within the whole-fit tolerance of its largest entry.
    V, _, W0, H0 = _completion(600, 500, 16, 1.0, seed=200)
    Vc = V.cuda()
    full = torch.ones(V.shape, dtype=torch.bool).to_sparse().cuda()
    n, W, H = _fit(Vc, {}, W0, H0, tol=1e-3, max_iter=200, alpha=0.0)
    nm, Wm, Hm = _fit(Vc, {"mask": full}, W0, H0, tol=1e-3, max_iter=200, alpha=0.0)
    assert nm == n
    X, Xm = H @ W.t(), Hm @ Wm.t()
    assert (Xm - X).abs().max() <= _fit_tolerance(X)


@pytest.mark.parametrize("R", [32, 80])
def test_loss_never_rises_between_checks(R):
    # alpha = 0: the reported loss is the objective, which no sweep raises in exact arithmetic; fp32 slack 1e-6 relative
    V, M, W0, H0 = _completion(3000, 2000, R, 0.05, seed=9, noise=0.2)
    O, _ = _observed(V, M)
    Wd, Hd = W0.cuda(), H0.cuda()
    eng = _engine(O, Wd, Hd)
    try:
        losses = [eng.loss(2)]
        for _ in range(20):
            eng.cd_iterate(10, 0.0, 0.0)
            losses.append(eng.loss(2))
    finally:
        eng.close()
    for a, b in zip(losses, losses[1:]):
        assert b <= a * (1 + 1e-6), (a, b)


def test_cd_beats_mu_on_a_planted_completion_problem():
    # 30 CD iterations against 200 MU iterations: lower observed loss and lower error on held-out cells.  Not a timing.
    gen = torch.Generator().manual_seed(3)
    N, C, R = 3000, 2000, 10
    V = (torch.rand(N, R, generator=gen) @ torch.rand(R, C, generator=gen)).cuda()
    M = (torch.rand(N, C, generator=gen) < 0.05).cuda()
    held = (~M) & (torch.rand(N, C, generator=gen) < 0.05).cuda()
    W0, H0 = torch.rand(C, R, generator=gen), torch.rand(N, R, generator=gen)
    out = {}
    for solver, iters in (("cd", 30), ("mu", 200)):
        from torchnmf_b200 import NMF
        m = NMF(W=W0, H=H0).cuda()
        m.fit(V, 2, float("-inf"), iters, solver=solver, mask=M.to_sparse())
        E = V - m.H.data @ m.W.data.t()
        out[solver] = (float((E[M] ** 2).sum()), float((E[held] ** 2).mean()))
    assert out["cd"][0] < out["mu"][0] and out["cd"][1] < out["mu"][1], out


def test_abi_refusals():
    from torchnmf_b200 import _capi
    lib = _capi.load()
    dev = torch.cuda.current_device()
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    N, C, R = 70, 50, 8
    V = torch.rand(N, C, device="cuda")
    W, H = torch.rand(C, R, device="cuda"), torch.rand(N, R, device="cuda")
    p = lambda t: ctypes.c_void_p(t.data_ptr())        # noqa: E731
    ctxs = []

    def nmf_ctx():
        c = ctypes.c_void_p()
        assert lib.nmfb200_nmf_create(ctypes.byref(c), dev, N, C, R, _capi.PREC_F32) == 0
        ctxs.append(c)
        return c

    def both(c, Wt=W, Ht=H):
        return (lib.nmfb200_nmf_observed_cd_update(c, p(Wt), p(Ht), 0, 0.0, 0.0, st),
                lib.nmfb200_nmf_observed_cd_iterate(c, p(Wt), p(Ht), 0.0, 0.0, 1, st))

    M = V > 0.5
    O, _ = _observed(V.cpu(), M.cpu())
    O = O.cuda()
    eng = _engine(O, W.clone(), H.clone())
    try:
        assert both(nmf_ctx()) == (3, 3)                                      # NMFB200_ERR_STATE before set_target
        c = nmf_ctx()
        assert lib.nmfb200_nmf_set_target(c, p(V), C, _capi.DTYPE_F32, st) == 0
        assert both(c) == (1, 1)                                              # NMFB200_ERR_INVALID: dense
        assert lib.nmfb200_set_mask(c, p(M.to(torch.uint8)), st) == 0
        assert both(c) == (1, 1)                                              # masked
        c = nmf_ctx()
        assert lib.nmfb200_nmf_set_target(c, p(V), C, _capi.DTYPE_F32, st) == 0
        assert lib.nmfb200_set_weight(c, p(torch.ones(N, C, device="cuda")), st) == 0
        assert both(c) == (1, 1)                                              # weighted
        from torchnmf_b200.engine import CudaSparseNmfEngine
        sp = CudaSparseNmfEngine(O, W.clone(), H.clone())
        try:
            assert both(sp._ctx) == (1, 1)                                    # sparse
        finally:
            sp.close()
        c = ctypes.c_void_p()
        vd, kd = (ctypes.c_int64 * 1)(20), (ctypes.c_int64 * 1)(4)
        assert lib.nmfb200_nmfnd_create(ctypes.byref(c), dev, 2, 6, 1, vd, 3, kd, _capi.PREC_F32) == 0
        ctxs.append(c)
        assert lib.nmfb200_nmfd_set_target(c, p(torch.rand(2, 6, 20, device="cuda")), _capi.DTYPE_F32, st) == 0
        assert both(c, torch.rand(6, 3, 4, device="cuda"), torch.rand(2, 3, 17, device="cuda")) == (1, 1)   # NMFD
        c = ctypes.c_void_p()
        assert lib.nmfb200_nmf_batched_create(ctypes.byref(c), dev, 2, N, C, R) == 0
        ctxs.append(c)
        assert lib.nmfb200_nmf_batched_set_target(c, p(V), C, 0, _capi.DTYPE_F32, st) == 0
        assert both(c, torch.rand(2, C, R, device="cuda"), torch.rand(2, N, R, device="cuda")) == (1, 1)    # batched
        # the observed context: served here, bad arguments refused, and the dense cd call keeps its refusal
        assert both(eng._ctx, eng.W, eng.H) == (0, 0)
        assert lib.nmfb200_nmf_observed_cd_update(eng._ctx, p(eng.W), p(eng.H), 2, 0.0, 0.0, st) == 1
        assert lib.nmfb200_nmf_observed_cd_iterate(eng._ctx, p(eng.W), p(eng.H), 0.0, 0.0, -1, st) == 1
        assert lib.nmfb200_nmf_observed_cd_update(eng._ctx, None, p(eng.H), 0, 0.0, 0.0, st) == 1
        assert lib.nmfb200_nmf_cd_update(eng._ctx, p(eng.W), p(eng.H), 0, 0.0, 0.0, st) == 1
        assert lib.nmfb200_last_error() == b"cd: observed-cell targets are not served"
        assert lib.nmfb200_nmf_cd_iterate(eng._ctx, p(eng.W), p(eng.H), 0.0, 0.0, 1, st) == 1
        assert lib.nmfb200_last_error() == b"cd: observed-cell targets are not served"
    finally:
        eng.close()
        for c in ctxs:
            lib.nmfb200_destroy(c)


def test_large_fit_memory_stays_that_of_the_mu_fit_plus_observed_floats():
    # 262144 x 131072 with 0.01 % observed (3.4 M cells), R = 64: the residual workspace is one float per observed cell, and
    # nothing else of the fit grows with N x C.  torch's peak covers the host-side staging (the observed set); the device's
    # free memory covers the library's own buffers.
    from torchnmf_b200 import NMF
    N, C, R = 262144, 131072, 64
    g = torch.Generator(device="cuda").manual_seed(0)
    nnz0 = int(N * C * 1e-4)
    lin = torch.randint(0, N * C, (nnz0,), generator=g, device="cuda").unique()
    nnz = lin.numel()
    V = torch.sparse_coo_tensor(torch.stack([lin // C, lin % C]), torch.rand(nnz, generator=g, device="cuda"), (N, C))
    V = V.coalesce()
    mask = torch.sparse_coo_tensor(V.indices(), torch.ones(nnz, dtype=torch.bool, device="cuda"), (N, C))
    W0 = torch.rand(C, R, generator=g, device="cuda") + 0.1
    H0 = torch.rand(N, R, generator=g, device="cuda") + 0.1
    peaks, used = {}, {}
    for solver in ("mu", "cd"):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        free0 = torch.cuda.mem_get_info()[0]
        base = torch.cuda.memory_allocated()
        m = NMF(W=W0.clone(), H=H0.clone())
        m.fit(V, 2, float("-inf"), 2, solver=solver, mask=mask)
        torch.cuda.synchronize()
        peaks[solver] = torch.cuda.max_memory_allocated() - base
        used[solver] = free0 - torch.cuda.mem_get_info()[0]
        assert torch.isfinite(m.W.data).all() and torch.isfinite(m.H.data).all()
        del m
    assert peaks["cd"] <= peaks["mu"] + 4 * nnz, peaks
    assert used["cd"] <= used["mu"] + 4 * nnz + (64 << 20), used     # the workspace, within the allocators' rounding
