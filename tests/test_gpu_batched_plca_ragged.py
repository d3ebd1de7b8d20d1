"""BatchedPLCA.fit(V, ..., lengths=L) on the H100 (nmfb200_plca_iterate / nmfb200_plca_loss on a ragged NMF batch): the EM
step term by term against the float64 model with the padding of H, Hz and the raw H numerators left untouched, the losses
and whole fits bit for bit against each problem's P = 1 fit (stopping at different counts, under permutation), full lengths
against the uniform batch, the reference fixtures, staged targets and modules, launch counts and a large batch."""
import ctypes

import pytest
import torch

from batched_plca_oracle import em_step, kl_loss, raw_terms, _rank
from test_batched_plca import _worst
from test_batched_plca_ragged import CASES, golden_case
from torchnmf_b200 import BatchedPLCA, _capi
from torchnmf_b200 import engine as _engine

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
SENT_H, SENT_HZ, SENT_WORK = 7.0, 9.0, -5.0


def _problems(lengths, N, C, R, seed=0, pad=float("nan")):
    """V (P, N, C) of multiples of 2^-8 below 2 -- every sum of a problem's target is exact in fp32, so its norm does not
    depend on torch's reduction order -- NaN past each length; W, H, Z normalised per problem over the real rows, H's padding
    a sentinel."""
    P = len(lengths)
    g = torch.Generator().manual_seed(seed)
    V = torch.randint(13, 512, (P, N, C), generator=g).float() / 256
    W = torch.rand(P, C, R, generator=g) + 0.1
    H = torch.rand(P, N, R, generator=g) + 0.1
    Z = torch.rand(P, R, generator=g) + 0.1
    for p, n in enumerate(lengths):
        V[p, n:] = pad
        H[p, :n] = H[p, :n] / H[p, :n].sum(0)
        H[p, n:] = SENT_H
    return V, W / W.sum(1, keepdim=True), H, Z / Z.sum(1, keepdim=True)


def _norms(V, lengths):
    return torch.stack([V[p, :n].sum() for p, n in enumerate(lengths)])


def _normalised_target(V, lengths):
    norm = _norms(V, lengths)
    return V / norm.view(-1, 1, 1), norm


def _em_once(R, flags, alpha, lengths, N=40, C=24, inactive=1, seed=0):
    """One plca_iterate step of a ragged engine on the GPU, and the float64 model's step of each problem on its real rows."""
    P = len(lengths)
    V, W, H, Z = _problems(lengths, N, C, R, seed)
    Vn, norm = _normalised_target(V, lengths)
    g = torch.Generator().manual_seed(seed + 1)
    alphas = []
    for t in (W, H, Z):
        if alpha == "none":
            alphas.append(None)
        elif alpha == "scalar":
            alphas.append(torch.full(t.shape, 1.3))
        else:
            alphas.append(0.8 + 0.6 * torch.rand(t.shape, generator=g))
    if alphas[1] is not None:
        for p, n in enumerate(lengths):
            alphas[1][p, n:] = float("nan")              # the padding of H_alpha is never read
    Wd, Hd, Zd = (t.to(DEV).contiguous() for t in (W, H, Z))
    Hz = (Hd * _rank(Zd, Hd)).contiguous()
    for p, n in enumerate(lengths):
        Hz[p, n:] = SENT_HZ
    eng = _engine.CudaBatchedNmfEngine(Vn.to(DEV).contiguous(), Wd, Hz, lengths=lengths)
    try:
        act = torch.ones(P, dtype=torch.bool)
        act[inactive] = False
        eng.set_active(act)
        eng._plca_work = torch.full((int(eng._lib.nmfb200_plca_work_numel(eng._ctx)),), SENT_WORK, device=DEV)
        before = {k: t.clone() for k, t in (("W", Wd), ("H", Hd), ("Z", Zd), ("Hz", Hz))}
        eng.plca_iterate(1, Hd, Zd, bool(flags & 1), bool(flags & 2), bool(flags & 4),
                         *[a.to(DEV).contiguous() if a is not None else None for a in alphas])
        loss = eng.plca_losses(norm.float().to(DEV))
        torch.cuda.synchronize()
        wn = P * C * R
        dHz = eng._plca_work[wn:wn + P * N * R].view(P, N, R).cpu()
        got = {"W": Wd.cpu(), "H": Hd.cpu(), "Z": Zd.cpu(), "Hz": Hz.cpu(), "loss": loss, "dHz": dHz}
    finally:
        eng.close()
    want = {k: before[k].cpu().double() for k in ("W", "H", "Z", "Hz")}
    want["loss"] = torch.zeros(P, dtype=torch.float64)
    for p, n in enumerate(lengths):
        if p == inactive:
            continue
        W64, H64, Z64 = W[p:p + 1].double(), H[p:p + 1, :n].double(), Z[p:p + 1].double()
        dW, dHz = raw_terms(Vn[p:p + 1, :n].double(), W64, H64 * _rank(Z64, H64))
        sl = [None if a is None else a[p:p + 1].double() for a in alphas]
        if sl[1] is not None:
            sl[1] = sl[1][:, :n]
        Wn, Hn, Zn = em_step(W64, H64, Z64, dW, dHz, bool(flags & 1), bool(flags & 2), bool(flags & 4), *sl)
        want["W"][p], want["H"][p, :n], want["Z"][p] = Wn[0], Hn[0], Zn[0]
        want["Hz"][p, :n] = (Hn * _rank(Zn, Hn))[0]
        want["loss"][p] = kl_loss(Vn[p:p + 1, :n].double(), Wn, Hn * _rank(Zn, Hn), norm[p:p + 1].double())[0]
    return got, want


def _check(got, want, lengths, inactive=1, rtol=2e-4):
    for k in ("W", "H", "Z", "Hz"):
        g, w = got[k].double(), want[k]
        assert torch.allclose(g, w, rtol=rtol, atol=1e-6 * float(w.abs().max())), (k, _worst(g, w))
    for p, n in enumerate(lengths):
        assert bool((got["H"][p, n:] == SENT_H).all()) and bool((got["Hz"][p, n:] == SENT_HZ).all())
        assert bool((got["dHz"][p, n:] == SENT_WORK).all())             # the raw H numerators' padding rows
        if p != inactive:
            assert bool((got["dHz"][p, :n] != SENT_WORK).all())


LENGTHS = [40, 1, 23, 17]


@pytest.mark.parametrize("flags", range(8))
@pytest.mark.parametrize("alpha", ["none", "scalar", "tensor"])
def test_em_step_flags_and_alphas(flags, alpha):
    got, want = _em_once(7, flags, alpha, LENGTHS)
    _check(got, want, LENGTHS)


@pytest.mark.parametrize("R", [1, 7, 16, 256])
def test_em_step_ranks(R):
    got, want = _em_once(R, 7, "tensor" if R == 7 else "none", LENGTHS, inactive=2)
    _check(got, want, LENGTHS, inactive=2)
    act = torch.tensor([True, True, False, True])
    assert torch.allclose(got["loss"][act], want["loss"][act], rtol=1e-4, atol=1e-6)


def test_losses_bit_for_bit_against_single_problems():
    lengths = [40, 1, 23, 17, 64]
    V, W, H, Z = _problems(lengths, 64, 24, 5, seed=2)
    Vn, norm = _normalised_target(V, lengths)
    Hz = H * _rank(Z, H)
    eng = _engine.CudaBatchedNmfEngine(Vn.to(DEV).contiguous(), W.to(DEV), Hz.to(DEV).contiguous(), lengths=lengths)
    try:
        loss = eng.plca_losses(norm.float().to(DEV))
    finally:
        eng.close()
    for p, n in enumerate(lengths):
        one = _engine.CudaBatchedNmfEngine(Vn[p:p + 1, :n].to(DEV).contiguous(), W[p:p + 1].to(DEV).contiguous(),
                                           Hz[p:p + 1, :n].to(DEV).contiguous())
        try:
            l1 = one.plca_losses(norm[p:p + 1].float().to(DEV))
        finally:
            one.close()
        assert torch.equal(l1[0], loss[p]), p


def _module(W, H, Z, device=DEV):
    """A module holding exactly these factors: the constructor's normalisation is undone by copying them back."""
    m = BatchedPLCA(W=W, H=H, Z=Z)
    for k, t in (("W", W), ("H", H), ("Z", Z)):
        getattr(m, k).data.copy_(t)
    return m.to(device)


def _fit(V, W, H, Z, device=DEV, **kw):
    m = _module(W, H, Z, device)
    n, norm = m.fit(V, **kw)
    return m, n, norm


def _single(V, W, H, Z, p, n, **kw):
    """The P = 1 fit without lengths on V[p:p+1, :L_p] from W[p:p+1], H[p:p+1, :L_p], Z[p:p+1]."""
    return _fit(V[p:p + 1, :n], W[p:p + 1], H[p:p + 1, :n], Z[p:p + 1], **kw)


def _assert_problem(m, n, norm, p, L, m1, n1, norm1):
    assert int(n1[0]) == int(n[p]) and torch.equal(norm1[0], norm[p]), p
    assert torch.equal(m1.W.data[0], m.W.data[p]) and torch.equal(m1.Z.data[0], m.Z.data[p]), p
    assert torch.equal(m1.H.data[0], m.H.data[p, :L]), p


def test_fits_bit_for_bit_against_single_fits_and_permutation():
    lengths = [64, 1, 37, 12, 50, 64]
    V, W, H, Z = _problems(lengths, 64, 32, 4, seed=3)
    Vd = V.to(DEV)
    for tol in torch.logspace(-4, -0.5, 22).tolist():   # the first tolerance at which the problems stop at different counts
        m, n, norm = _fit(Vd, W, H, Z, tol=tol, max_iter=60, lengths=lengths)
        if len(set(n.tolist())) > 1:
            break
    assert len(set(n.tolist())) > 1 and int(n.min()) < 59
    for p, L in enumerate(lengths):
        assert bool((m.H.data[p, L:] == SENT_H).all())
        m1, n1, norm1 = _single(Vd, W, H, Z, p, L, tol=tol, max_iter=60)
        _assert_problem(m, n, norm, p, L, m1, n1, norm1)
    perm = [3, 0, 5, 2, 1, 4]
    mp, n_p, norm_p = _fit(Vd[perm].contiguous(), W[perm], H[perm], Z[perm], tol=tol, max_iter=60,
                           lengths=[lengths[p] for p in perm])
    for i, p in enumerate(perm):
        assert int(n_p[i]) == int(n[p]) and torch.equal(norm_p[i], norm[p])
        for k in ("W", "H", "Z"):
            assert torch.equal(getattr(mp, k).data[i], getattr(m, k).data[p])


@pytest.mark.parametrize("frozen", ["Z", "W", "WZ"])
def test_frozen_factors_bit_for_bit(frozen):
    lengths = [30, 1, 17]
    V, W, H, Z = _problems(lengths, 30, 16, 3, seed=4)
    kw = dict(trainable_W="W" not in frozen, trainable_Z="Z" not in frozen)

    def fit(Vx, Wx, Hx, Zx, **fkw):
        m = BatchedPLCA(W=Wx, H=Hx, Z=Zx, **kw)
        for k, t in (("W", Wx), ("H", Hx), ("Z", Zx)):
            getattr(m, k).data.copy_(t)
        m = m.to(DEV)
        n, norm = m.fit(Vx, **fkw)
        return m, n, norm
    m, n, norm = fit(V.to(DEV), W, H, Z, tol=-1.0, max_iter=20, H_alpha=1.1, lengths=lengths)
    for p, L in enumerate(lengths):
        m1, n1, norm1 = fit(V[p:p + 1, :L].to(DEV), W[p:p + 1], H[p:p + 1, :L], Z[p:p + 1], tol=-1.0, max_iter=20,
                            H_alpha=1.1)
        _assert_problem(m, n, norm, p, L, m1, n1, norm1)


def test_full_lengths_equal_uniform_batch():
    V, W, H, Z = _problems([48] * 4, 48, 20, 5, seed=5)
    Vd = V.to(DEV)
    a, na, norma = _fit(Vd, W, H, Z, tol=1e-4, max_iter=60)
    b, nb, normb = _fit(Vd, W, H, Z, tol=1e-4, max_iter=60, lengths=[48] * 4)
    assert na.tolist() == nb.tolist() and torch.equal(norma, normb)
    for k in ("W", "H", "Z"):
        assert torch.equal(getattr(a, k).data, getattr(b, k).data)


@pytest.mark.parametrize("name", CASES)
def test_against_reference_fixtures(name):
    c = golden_case(name)
    lengths = c["lengths"].tolist()
    m = BatchedPLCA(W=c["W0"], H=c["H0"], Z=c["Z0"], trainable_W=bool(c["trainable_W"]),
                    trainable_Z=bool(c["trainable_Z"])).to(DEV)
    W_alpha = c["W_alpha"].reshape(-1, 1, 1) if isinstance(c["W_alpha"], torch.Tensor) else c["W_alpha"]
    n, norm = m.fit(c["V"].to(DEV), tol=c["tol"], max_iter=int(c["max_iter"]), W_alpha=W_alpha, H_alpha=c["H_alpha"],
                    Z_alpha=c["Z_alpha"], lengths=lengths)
    assert n.tolist() == c["n_iter"].tolist()
    assert torch.allclose(norm.double().cpu(), c["norm"], rtol=1e-6)
    for k in ("W", "H", "Z"):
        got, want = getattr(m, k).data.cpu(), c[k]
        assert torch.allclose(got, want, rtol=1e-3, atol=1e-5 * float(want.abs().max())), (k, _worst(got, want))


def test_staging_dtypes_and_host_modules():
    lengths = [32, 1, 20, 9]
    V, W, H, Z = _problems(lengths, 32, 16, 4, seed=6)
    ref, nr, normr = _fit(V.to(DEV), W, H, Z, tol=-1.0, max_iter=20, lengths=lengths)
    # lengths as a CUDA tensor
    t, nt, normt = _fit(V.to(DEV), W, H, Z, tol=-1.0, max_iter=20, lengths=torch.tensor(lengths, device=DEV))
    assert nt.tolist() == nr.tolist() and torch.equal(normt, normr)
    for k in ("W", "H", "Z"):
        assert torch.equal(getattr(t, k).data, getattr(ref, k).data)
    # half and double targets: each problem as its P = 1 fit of the same dtype
    for dt in (torch.bfloat16, torch.float16, torch.float64):
        Vt = V.to(dt).to(DEV)
        m, n, norm = _fit(Vt, W, H, Z, tol=-1.0, max_iter=20, lengths=lengths)
        assert norm.dtype == dt
        for p, L in enumerate(lengths):
            m1, n1, norm1 = _single(Vt, W, H, Z, p, L, tol=-1.0, max_iter=20)
            _assert_problem(m, n, norm, p, L, m1, n1, norm1)
    # a host module and a float64 module: staged, written back on the real rows only
    for host in (_module(W, H, Z, device="cpu"), _module(W, H, Z, device="cpu").double()):
        nh, _ = host.fit(V.to(DEV), tol=-1.0, max_iter=20, lengths=lengths)
        assert host.W.device.type == "cpu" and nh.tolist() == nr.tolist()
        assert torch.equal(host.W.data.float(), ref.W.data.cpu()) and torch.equal(host.Z.data.float(), ref.Z.data.cpu())
        for p, L in enumerate(lengths):
            assert torch.equal(host.H.data[p, :L].float(), ref.H.data[p, :L].cpu())
            assert bool((host.H.data[p, L:] == SENT_H).all())


def test_launch_count_independent_of_batch():
    counts = {}
    for P in (1, 64):
        g = torch.Generator().manual_seed(7)
        lengths = torch.randint(1, 49, (P,), generator=g).tolist()
        V, W, H, Z = _problems(lengths, 48, 20, 8, seed=7)
        Vn, _ = _normalised_target(V, lengths)
        Wd, Hd, Zd = (t.to(DEV).contiguous() for t in (W, H, Z))
        Hz = (Hd * Zd.unsqueeze(1)).contiguous()
        eng = _engine.CudaBatchedNmfEngine(Vn.to(DEV).contiguous(), Wd, Hz, lengths=lengths)
        try:
            eng.plca_iterate(1, Hd, Zd, True, True, True)
            c0 = _capi.launch_count()
            eng.plca_iterate(10, Hd, Zd, True, True, True, torch.full_like(Wd, 1.2), None, None)
            counts[P] = _capi.launch_count() - c0
        finally:
            eng.close()
    assert counts[1] == counts[64] and counts[1] % 10 == 0


def test_large_ragged_batch():
    P, N, C, R = 4096, 512, 64, 16
    g = torch.Generator().manual_seed(11)
    lengths = torch.randint(1, N + 1, (P,), generator=g)
    lengths[0], lengths[1] = 1, N
    V = (torch.randint(13, 512, (P, N, C), generator=g).float() / 256).to(DEV)
    m = BatchedPLCA((P, N, C), rank=R).to(DEV)
    W0, H0, Z0 = m.W.data.clone(), m.H.data.clone(), m.Z.data.clone()
    n, norm = m.fit(V, tol=1e-4, max_iter=30, lengths=lengths)
    assert bool(torch.isfinite(m.W.data).all()) and bool(torch.isfinite(m.Z.data).all())
    L = lengths.tolist()
    for p in (0, 1, 2345, P - 1):
        s = _module(W0[p:p + 1], H0[p:p + 1, :L[p]], Z0[p:p + 1])
        n1, norm1 = s.fit(V[p:p + 1, :L[p]], tol=1e-4, max_iter=30)
        _assert_problem(m, n, norm, p, L[p], s, n1, norm1)
        assert torch.equal(m.H.data[p, L[p]:], H0[p, L[p]:])


def test_capi_serves_a_ragged_nmf_context():
    lib = _capi.load()
    P, N, C, R = 3, 20, 12, 4
    lengths = [20, 1, 9]
    lens = (ctypes.c_int64 * P)(*lengths)
    ctx = ctypes.c_void_p()
    assert lib.nmfb200_nmf_batched_create_ragged(ctypes.byref(ctx), torch.cuda.current_device(), P, N, C, R, lens) == 0
    try:
        V, W, H, Z = _problems(lengths, N, C, R, seed=8)
        Vn = _normalised_target(V, lengths)[0].to(DEV).contiguous()
        W, H, Z = W.to(DEV).contiguous(), H.to(DEV).contiguous(), Z.to(DEV).contiguous()
        Hz = (H * Z.unsqueeze(1)).contiguous()
        stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        assert lib.nmfb200_nmf_batched_set_target(ctx, ctypes.c_void_p(Vn.data_ptr()), C, N * C, _capi.DTYPES[Vn.dtype],
                                                  stream) == 0
        work = torch.empty(int(lib.nmfb200_plca_work_numel(ctx)), device=DEV)
        assert lib.nmfb200_plca_iterate(ctx, ctypes.c_void_p(W.data_ptr()), ctypes.c_void_p(H.data_ptr()),
                                        ctypes.c_void_p(Z.data_ptr()), ctypes.c_void_p(Hz.data_ptr()),
                                        ctypes.c_void_p(work.data_ptr()), 7, None, None, None, 2, stream) == 0
        norm = torch.ones(P, device=DEV)
        loss = torch.zeros(P, dtype=torch.float64, device=DEV)
        assert lib.nmfb200_plca_loss(ctx, ctypes.c_void_p(W.data_ptr()), ctypes.c_void_p(Hz.data_ptr()),
                                     ctypes.c_void_p(norm.data_ptr()), ctypes.c_void_p(loss.data_ptr()), stream) == 0
        torch.cuda.synchronize()
        assert bool(torch.isfinite(loss).all()) and bool((loss > 0).all())
    finally:
        lib.nmfb200_destroy(ctx)
