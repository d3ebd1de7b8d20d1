"""Coordinate descent at beta 2 on the GPU (`NMF.fit(V, beta=2, solver="cd")`, include/nmf_b200.h: nmfb200_nmf_cd_*).

* The numerator the sweep reads equals nmfb200_raw_terms(which, 2.0)'s bit for bit, at every tile plan and V dtype.
* One update and whole fits against the float64 oracle (tests/cd_oracle.py), within tolerances derived below.
* Determinism, half-precision targets, frozen factors, staged modules, sparse targets, the loss trace, and the refusals.
"""
import ctypes
import math

import pytest
import torch

import cd_oracle as cdo
from f32_cases import NMF_CHUNKED, NMF_EDGE

pytestmark = pytest.mark.gpu

U = 2.0 ** -24                     # fp32 unit roundoff


def _engine(V, W, H):
    from torchnmf_b200.engine import CudaNmfEngine
    return CudaNmfEngine(V, W, H, "f32")


def _disjoint(rows, R, gen):
    """A (rows x R) factor whose component k is 1 on a power-of-two number of the rows r with r % R == k and 0 elsewhere: its
    Gram matrix is diagonal with powers of two on the diagonal (0 for a component with no row), exactly in any order."""
    X = torch.zeros(rows, R)
    for k in range(min(R, rows)):
        idx = torch.arange(k, rows, R)
        idx = idx[torch.randperm(idx.numel(), generator=gen)[:1 << int(math.log2(idx.numel()))]]
        X[idx, k] = 1.0
    return X


def _target(N, C, dtype, strided, gen):
    V = torch.rand(N, C + (5 if strided else 0), generator=gen)
    V = V.to(dtype).cuda()
    return V[:, :C] if strided else V


# ---- A: the numerator, bit for bit -----------------------------------------------------------------------------------------

NUM_SHAPES = NMF_EDGE + NMF_CHUNKED[:4]


@pytest.mark.parametrize("N,C,R", NUM_SHAPES)
@pytest.mark.parametrize("kind", ["f32", "f16", "bf16", "strided"])
@pytest.mark.parametrize("which", [0, 1])
def test_numerator_equals_raw_terms_bit_for_bit(N, C, R, kind, which):
    # With the updated factor X = 0, l1 = l2 = 0 and the other factor of disjoint supports (B diagonal, powers of two), every
    # column step is X[c,k] = A[c,k] / B[k,k] exactly (the dot over X is exactly 0): A = X B recovers the sweep's A bit for
    # bit, to be compared with nmfb200_raw_terms' numerator from the same factors.
    gen = torch.Generator().manual_seed(N * 7 + C * 3 + R)
    dtype = {"f16": torch.float16, "bf16": torch.bfloat16}.get(kind, torch.float32)
    V = _target(N, C, dtype, kind == "strided", gen)
    if which == 0:
        W, H = torch.zeros(C, R).cuda(), _disjoint(N, R, gen).cuda()
    else:
        W, H = _disjoint(C, R, gen).cuda(), torch.zeros(N, R).cuda()
    eng = _engine(V, W, H)
    try:
        A_ref = eng.raw_terms(which, 2.0)[0].clone()
        other = H if which == 0 else W
        b = (other * other).sum(0)
        eng.cd_update(which, 0.0, 0.0)
        X = W if which == 0 else H
        assert torch.equal(X * b, A_ref)
    finally:
        eng.close()


# ---- one update and whole fits against float64 -------------------------------------------------------------------------

def _planted(N, C, R, seed, noise=0.01):
    """A well-conditioned problem: factors with one strong entry per row (component row % R) over a weak background, so the
    Gram matrices are diagonally dominant; V = H* W*^T plus a little noise.  Returns V and fp32 starting factors."""
    gen = torch.Generator().manual_seed(seed)

    def fac(rows):
        X = 0.05 * torch.rand(rows, R, generator=gen)
        X[torch.arange(rows), torch.arange(rows) % R] += 1.0 + torch.rand(rows, generator=gen)
        return X
    V = fac(N) @ fac(C).t() + noise * torch.rand(N, C, generator=gen)
    return V, torch.rand(C, R, generator=gen) + 0.1, torch.rand(N, R, generator=gen) + 0.1


@pytest.mark.parametrize("N,C,R", [(300, 200, 16), (1000, 700, 64), (129, 2112, 17)])
@pytest.mark.parametrize("which", [0, 1])
@pytest.mark.parametrize("l1,l2", [(0.0, 0.0), (0.5, 0.25)])
def test_one_update_matches_float64(N, C, R, which, l1, l2):
    # Tolerance: A and B are fp32 sums of K = N (W) or C (H) non-negative products, each within K u of its value; the dot
    # sum_j X B[j,k] of R non-negative products within R u.  A column step divides a - dot - l1 - l2 x by B[k,k] + l2, so its
    # error is at most (K + R + 4) u (A + |X| B) / (B[k,k] + l2), plus what the earlier columns' errors carry in through
    # B[j,k] / B[k,k] -- about 0.03 each on these diagonally dominant problems, a factor of a few over R columns; x 8.
    V, W, H = _planted(N, C, R, seed=N + R + which)
    Vd, Wd, Hd = V.cuda(), W.cuda(), H.cuda()
    X64 = cdo.update(V, W, H, which, l1, l2)
    A, B = cdo.terms(V, W, H, which)
    K = N if which == 0 else C
    bound = 8 * (K + R + 4) * U * (A + X64.abs() @ B.abs()) / (torch.diagonal(B) + l2)
    eng = _engine(Vd, Wd, Hd)
    try:
        eng.cd_update(which, l1, l2)
    finally:
        eng.close()
    got = (Wd if which == 0 else Hd).cpu().double()
    assert ((got - X64).abs() <= bound).all(), float(((got - X64).abs() / bound).max())


def _fit_tolerance(X):
    return 2e-4 * float(X.abs().max())


@pytest.mark.parametrize("seed", [0, 1, 2])
@pytest.mark.parametrize("alpha,l1_ratio", [(0.0, 0.0), (1.0, 0.5)])
def test_whole_fit_matches_float64(seed, alpha, l1_ratio):
    # Whole fits converge to the same fixed point; fp32 rounding moves it by a few units of 1e-6 relative on these
    # well-conditioned problems, so the factors agree to 2e-4 of their largest entry, and the stop rule (tol 1e-3, losses
    # far apart between checks) takes the same iteration.
    from torchnmf_b200 import NMF
    V, W0, H0 = _planted(400, 300, 12, seed=100 + seed)
    m = NMF(W=W0, H=H0).cuda()
    n = m.fit(V.cuda(), 2, 1e-3, 200, False, alpha, l1_ratio, solver="cd")
    assert m.last_fit_precision == "f32"
    W, H, n_ref, _ = cdo.fit(V.double(), W0.double(), H0.double(), 1e-3, 200, alpha * l1_ratio, alpha * (1 - l1_ratio))
    assert n == n_ref
    for got, want in ((m.W.data.cpu().double(), W), (m.H.data.cpu().double(), H)):
        assert (got - want).abs().max() <= _fit_tolerance(want)


def _fit(V, W0, H0, **kw):
    from torchnmf_b200 import NMF
    m = NMF(W=W0, H=H0, trainable_W=kw.pop("trainable_W", True), trainable_H=kw.pop("trainable_H", True))
    if kw.pop("cuda", True):
        m = m.cuda()
    if kw.pop("double", False):
        m = m.double()
    n = m.fit(V, 2, kw.pop("tol", 1e-4), kw.pop("max_iter", 60), False, kw.pop("alpha", 0.1), kw.pop("l1_ratio", 0.3),
              solver="cd", **kw)
    return n, m.W.data, m.H.data


def test_bit_exact_runs_targets_and_modules():
    V, W0, H0 = _planted(500, 333, 20, seed=7)
    V = V.bfloat16().float()                                        # exact in bf16
    Vc = V.cuda()
    n, W, H = _fit(Vc, W0, H0)
    # two runs of the same fit are bit-identical
    n2, W2, H2 = _fit(Vc, W0, H0)
    assert n == n2 and torch.equal(W, W2) and torch.equal(H, H2)
    # a bf16 V gives the bits of V.float(); so does fp16 of an fp16-exact V
    nb, Wb, Hb = _fit(Vc.bfloat16(), W0, H0)
    assert nb == n and torch.equal(Wb, W) and torch.equal(Hb, H)
    V16 = Vc.half().float()
    nf, Wf, Hf = _fit(V16, W0, H0)
    nh, Wh, Hh = _fit(V16.half(), W0, H0)
    assert nh == nf and torch.equal(Wh, Wf) and torch.equal(Hh, Hf)
    # a row-strided fp32 view gives the bits of the contiguous target
    Vs = torch.zeros(500, 340, device="cuda")
    Vs[:, :333] = Vc
    ns, Ws, Hs = _fit(Vs[:, :333], W0, H0)
    assert ns == n and torch.equal(Ws, W) and torch.equal(Hs, H)
    # a float64 target is staged: the bits of its fp32 copy
    nd, Wd, Hd = _fit(Vc.double(), W0, H0)
    assert nd == n and torch.equal(Wd, W) and torch.equal(Hd, H)
    # host modules and float64 modules are written back
    nhst, Whst, Hhst = _fit(V, W0, H0, cuda=False)
    assert nhst == n and Whst.device.type == "cpu" and torch.equal(Whst, W.cpu()) and torch.equal(Hhst, H.cpu())
    n64, W64, H64 = _fit(Vc, W0, H0, double=True)
    assert n64 == n and W64.dtype == torch.float64 and torch.equal(W64, W.double()) and torch.equal(H64, H.double())
    # a frozen factor stays bit-identical
    for frozen in ("W", "H"):
        _, Wz, Hz = _fit(Vc, W0, H0, trainable_W=frozen != "W", trainable_H=frozen != "H")
        assert torch.equal((Wz if frozen == "W" else Hz).cpu(), W0 if frozen == "W" else H0)


@pytest.mark.parametrize("seed", [0, 1])
def test_sparse_target_matches_its_dense_fit(seed):
    # the numerator's sums run in stored order instead of the dense tiles': the fits agree within the whole-fit tolerance
    gen = torch.Generator().manual_seed(seed)
    V, W0, H0 = _planted(600, 500, 16, seed=200 + seed)
    V = V * (torch.rand(V.shape, generator=gen) < 0.3)
    n, W, H = _fit(V.cuda(), W0, H0, tol=1e-3, max_iter=200, alpha=0.0)
    ns, Ws, Hs = _fit(V.to_sparse().cuda(), W0, H0, tol=1e-3, max_iter=200, alpha=0.0)
    assert ns == n
    assert (Ws - W).abs().max() <= _fit_tolerance(W) and (Hs - H).abs().max() <= _fit_tolerance(H)


def test_loss_never_rises_between_checks():
    # alpha = 0: the reported loss is the objective, which no sweep raises in exact arithmetic; fp32 slack 1e-6 relative
    V, W0, H0 = _planted(2000, 1500, 32, seed=9, noise=0.2)
    Vd, Wd, Hd = V.cuda(), W0.cuda(), H0.cuda()
    eng = _engine(Vd, Wd, Hd)
    try:
        losses = [eng.loss(2)]
        for _ in range(20):
            eng.cd_iterate(10, 0.0, 0.0)
            losses.append(eng.loss(2))
    finally:
        eng.close()
    for a, b in zip(losses, losses[1:]):
        assert b <= a * (1 + 1e-6), (a, b)


def test_cd_beats_mu_on_a_planted_low_rank_target():
    # a coarse check that the solver does its job, not a timing
    from torchnmf_b200 import NMF
    gen = torch.Generator().manual_seed(3)
    R = 20
    V = (torch.rand(1500, R, generator=gen) @ torch.rand(R, 1000, generator=gen)).cuda()
    W0, H0 = torch.rand(1000, R, generator=gen), torch.rand(1500, R, generator=gen)
    out = {}
    for solver, iters in (("cd", 50), ("mu", 200)):
        m = NMF(W=W0, H=H0).cuda()
        m.fit(V, 2, float("-inf"), iters, precision="f32", solver=solver)
        out[solver] = float(((V - m.H.data @ m.W.data.t()) ** 2).sum())
    assert out["cd"] < out["mu"], out


# ---- the ABI's refusals -----------------------------------------------------------------------------------------------------

def test_abi_refusals():
    from torchnmf_b200 import _capi
    from torchnmf_b200.engine import CudaObservedNmfEngine
    lib = _capi.load()
    dev = torch.cuda.current_device()
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    N, C, R = 70, 50, 8
    V = torch.rand(N, C, device="cuda")
    W, H = torch.rand(C, R, device="cuda"), torch.rand(N, R, device="cuda")
    p = lambda t: ctypes.c_void_p(t.data_ptr())        # noqa: E731
    ctxs = []

    def nmf_ctx(r=R, target=True):
        c = ctypes.c_void_p()
        assert lib.nmfb200_nmf_create(ctypes.byref(c), dev, N, C, r, _capi.PREC_F32) == 0
        ctxs.append(c)
        if target:
            assert lib.nmfb200_nmf_set_target(c, p(V), C, _capi.DTYPE_F32, st) == 0
        return c

    def both(c, Wt=W, Ht=H):
        return (lib.nmfb200_nmf_cd_update(c, p(Wt), p(Ht), 0, 0.0, 0.0, st),
                lib.nmfb200_nmf_cd_iterate(c, p(Wt), p(Ht), 0.0, 0.0, 1, st))

    try:
        assert both(nmf_ctx(target=False)) == (3, 3)                          # NMFB200_ERR_STATE before set_target
        c = nmf_ctx()
        assert both(c) == (0, 0)
        assert lib.nmfb200_set_mask(c, p(torch.ones(N, C, dtype=torch.uint8, device="cuda")), st) == 0
        assert both(c) == (1, 1)                                              # NMFB200_ERR_INVALID: a mask
        c = nmf_ctx()
        assert lib.nmfb200_set_weight(c, p(torch.ones(N, C, device="cuda")), st) == 0
        assert both(c) == (1, 1)                                              # a weight
        W257, H257 = torch.rand(C, 257, device="cuda"), torch.rand(N, 257, device="cuda")
        assert both(nmf_ctx(r=257), W257, H257) == (1, 1)                     # R > 256
        c = ctypes.c_void_p()
        vd, kd = (ctypes.c_int64 * 1)(20), (ctypes.c_int64 * 1)(4)
        assert lib.nmfb200_nmfnd_create(ctypes.byref(c), dev, 2, 6, 1, vd, 3, kd, _capi.PREC_F32) == 0
        ctxs.append(c)
        Vn = torch.rand(2, 6, 20, device="cuda")
        assert lib.nmfb200_nmfd_set_target(c, p(Vn), _capi.DTYPE_F32, st) == 0
        assert both(c, torch.rand(6, 3, 4, device="cuda"), torch.rand(2, 3, 17, device="cuda")) == (1, 1)   # NMFD
        c = ctypes.c_void_p()
        assert lib.nmfb200_nmf_batched_create(ctypes.byref(c), dev, 2, N, C, R) == 0
        ctxs.append(c)
        assert lib.nmfb200_nmf_batched_set_target(c, p(V), C, 0, _capi.DTYPE_F32, st) == 0
        assert both(c, torch.rand(2, C, R, device="cuda"), torch.rand(2, N, R, device="cuda")) == (1, 1)    # batched
        O = (V * (V > 0.5)).to_sparse().coalesce()
        eng = CudaObservedNmfEngine(O, W.clone(), H.clone())
        try:
            assert both(eng._ctx) == (1, 1)                                   # observed cells
        finally:
            eng.close()
    finally:
        for c in ctxs:
            lib.nmfb200_destroy(c)
