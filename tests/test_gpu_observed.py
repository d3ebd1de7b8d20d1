"""Fits on the observed cells of a sparse mask (`NMF.fit(V, ..., mask=M)` with a sparse COO `M`,
nmfb200_nmf_set_target_observed) on the GPU.

The observed-cell gathers are checked term by term against float64 (tests/masked_oracle.py in double precision on the
densified mask): the raw numerators and denominators of both updates and the loss, at every rank-per-lane branch and its
edges and at every beta branch.  Then whole fits: against the dense-mask fit, against the unmodified reference's BetaMu
fixtures, bit for bit across input forms, repeat calls, the cached workspace, the densified path above rank 256 and the
sharded protocol over gloo, and one fit past 2^31 cells.
"""
import ctypes
import os
import socket
import sys

import pytest
import torch

import masked_oracle as mo
from test_masked import CASES
from test_observed import OBS, sparse_target

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
DEV = torch.device("cuda", 0)
BETAS = (0, 0.5, 1, 1.5, 2, 3)
RANKS = (1, 31, 32, 33, 64, 65, 128, 129, 256)


def _observed(V, M):
    from torchnmf_b200.nmf import _observed_cells
    return _observed_cells(V, M if M.is_sparse else M.to_sparse(), DEV)


def _engine(V, M, W, H):
    from torchnmf_b200 import engine
    return engine.CudaObservedNmfEngine(_observed(V, M), W, H)


def _inputs(N, C, R, beta, density, seed=0):
    """V, W, H and a mask of the given density with rows 3 and 7 and columns 2 and 5 empty, row 1 and column 4 full."""
    g = torch.Generator().manual_seed(seed)
    V = torch.rand(N, C, generator=g)
    if beta <= 0:
        V = V.clamp_min(2 ** -7)
    W = torch.rand(C, R, generator=g) + 0.1
    H = torch.rand(N, R, generator=g) + 0.1
    M = torch.rand(N, C, generator=g) < density
    M[1] = True
    M[:, 4] = True
    M[[3, 7]] = False
    M[:, [2, 5]] = False
    return V, W, H, M


@pytest.mark.parametrize("density", [0.01, 0.6])
@pytest.mark.parametrize("beta", BETAS)
@pytest.mark.parametrize("R", RANKS)
def test_terms_and_loss_against_float64(R, beta, density):
    N, C = 150, 90
    V, W, H, M = _inputs(N, C, R, beta, density, seed=R)
    V64, W64, H64 = V.double(), W.double(), H.double()
    Wd, Hd = W.to(DEV), H.to(DEV)
    eng = _engine(V, M, Wd, Hd)
    try:
        assert eng.precision_for(beta) == "f32"
        for which in (0, 1):
            num, den = eng.raw_terms(which, beta)
            want = mo.masked_terms(V64, W64, H64, M, beta, which)
            f = W if which == 0 else H
            assert num.shape == f.shape and den.shape == f.shape
            for got, w in ((num, want[0]), (den, want[1])):
                got = got.double().cpu()
                assert torch.allclose(got, w, rtol=2e-4, atol=1e-6 * float(w.abs().max())), \
                    (R, beta, which, float((got - w).abs().max()))
        loss = float(mo.masked_loss(H64 @ W64.t(), V64, M, beta))
        got = eng.loss(beta)
        assert abs(got - loss) <= 1e-4 * abs(loss) + 1e-6, (got, loss)
        assert eng.minmax() == (float(V[M].min()), float(V[M].max()))
    finally:
        eng.close()
    assert torch.equal(Wd.cpu(), W) and torch.equal(Hd.cpu(), H)


def test_context_calls_of_an_observed_target():
    from torchnmf_b200 import _capi, engine
    lib = _capi.load()
    V, W, H, M = _inputs(40, 30, 8, 1, 0.3)
    Wd, Hd = W.to(DEV), H.to(DEV)
    eng = _engine(V, M, Wd, Hd)
    try:
        for beta in BETAS:
            assert lib.nmfb200_raw_terms_numel(eng._ctx, 0, float(beta)) == 2 * W.numel()
            assert lib.nmfb200_raw_terms_numel(eng._ctx, 1, float(beta)) == 2 * H.numel()
            assert lib.nmfb200_precision_for_beta(eng._ctx, float(beta)) == _capi.PREC_F32
            assert lib.nmfb200_nmf_peer_supported(eng._ctx, float(beta)) == 0
        stream = ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)
        assert lib.nmfb200_nmf_contract_only(eng._ctx, Wd.data_ptr(), Hd.data_ptr(), 0, 1.0, stream) == 3   # ERR_STATE
        Md = M.to(DEV)
        assert lib.nmfb200_set_mask(eng._ctx, Md.data_ptr(), stream) == 1                                  # ERR_INVALID
        loss = torch.zeros(1, dtype=torch.float64, device=DEV)
        assert lib.nmfb200_nmf_loss_prefetch_w(eng._ctx, Wd.data_ptr(), Hd.data_ptr(), 0.5, loss.data_ptr(), stream) == 0
        assert float(loss) == eng.loss(0.5)
    finally:
        eng.close()
    empty = torch.zeros(40, 30, dtype=torch.bool)
    eng = _engine(V, empty, Wd, Hd)
    try:
        assert eng.minmax() == (float("inf"), float("-inf"))
    finally:
        eng.close()
    W3, H3 = torch.rand(30, 300, device=DEV), torch.rand(40, 300, device=DEV)
    with pytest.raises(_capi.NmfB200Error, match="rank > 256"):
        engine.CudaObservedNmfEngine(_observed(V, M), W3, H3)
    engine.release_workspaces()


# ---- whole fits ----------------------------------------------------------------------------------------------------------
def _fit(V, W, H, M, beta, max_iter=20, trainable_W=True, **kw):
    from torchnmf_b200 import NMF
    m = NMF(W=W, H=H, trainable_W=trainable_W).to(DEV)
    n = m.fit(V, beta, float("-inf"), max_iter, mask=M, **kw)
    return m.W.data.cpu(), m.H.data.cpu(), n, m


@pytest.mark.parametrize("case", ["b0", "b0.5", "b1", "b2", "b1_alpha", "b0.5_frozenW"])
def test_sparse_mask_fit_matches_the_dense_mask_fit(case):
    beta = float(case.split("_")[0][1:])
    kw = {"alpha": 0.1, "l1_ratio": 0.5} if "alpha" in case else {}
    tw = "frozenW" not in case
    V, W, H, M = _inputs(300, 200, 32, beta, 0.3)
    Vd, Md = V.to(DEV), M.to(DEV)
    Wa, Ha, na, ma = _fit(Vd, W, H, Md.to_sparse(), beta, trainable_W=tw, **kw)
    Wb, Hb, nb, _ = _fit(Vd, W, H, Md, beta, trainable_W=tw, **kw)
    assert na == nb and ma.last_fit_precision == "f32"
    for a, b in ((Wa, Wb), (Ha, Hb)):
        assert torch.allclose(a, b, rtol=1e-4, atol=1e-6 * float(b.abs().max())), float((a - b).abs().max())
    if not tw:
        assert torch.equal(Wa, W)


@pytest.mark.parametrize("name", sorted(n for n, c in CASES.items() if c["kind"] == "nmf"))
def test_fit_matches_reference_masked(name):
    c = CASES[name]
    from torchnmf_b200 import NMF
    m = NMF(W=c["W0"], H=c["H0"], trainable_W=bool(c["trainable_W"])).to(DEV)
    n_iter = m.fit(c["V"].to(DEV), c["beta"], c["tol"], c["max_iter"], False, c["alpha"], c["l1_ratio"],
                   mask=c["M"].to(DEV).to_sparse())
    assert n_iter == c["n_iter"]
    for got, want in ((m.W.data.cpu(), c["W"]), (m.H.data.cpu(), c["H"])):
        assert torch.allclose(got, want, rtol=1e-3, atol=1e-5 * float(want.abs().max())), float((got - want).abs().max())


@pytest.mark.parametrize("name", sorted(OBS))
def test_fit_matches_reference_observed(name):
    c = OBS[name]
    from torchnmf_b200 import NMF
    m = NMF(W=c["W0"], H=c["H0"], trainable_W=bool(c["trainable_W"])).to(DEV)
    n_iter = m.fit(sparse_target(c).to(DEV), c["beta"], c["tol"], c["max_iter"], False, c["alpha"], c["l1_ratio"],
                   mask=c["M"].to_sparse().to(DEV))
    assert n_iter == c["n_iter"] and m.last_fit_precision == "f32"
    for got, want in ((m.W.data.cpu(), c["W"]), (m.H.data.cpu(), c["H"])):
        assert torch.allclose(got, want, rtol=1e-3, atol=1e-5 * float(want.abs().max())), float((got - want).abs().max())


def test_every_input_form_of_one_observed_set_gives_the_same_bits():
    V, W, H, M = _inputs(257, 129, 40, 0.5, 0.2)
    V = V.bfloat16().float()                                      # exact in bf16 too
    Md = M.to(DEV)
    Ms = Md.to_sparse()
    idx = Ms.indices()
    miss = (~Md).nonzero().t()[:, :100]
    dup = torch.sparse_coo_tensor(torch.cat([idx.flip(1), idx[:, :50], miss], 1),
                                  torch.cat([torch.ones(idx.shape[1] + 50, dtype=torch.bool, device=DEV),
                                             torch.zeros(100, dtype=torch.bool, device=DEV)]), M.shape)
    big = torch.full((V.shape[0], V.shape[1] + 11), float("nan"), device=DEV)
    big[:, 3:3 + V.shape[1]] = V.to(DEV)
    Vsp = (V * M + (V + 1) * (~M & (torch.rand(V.shape) < 0.3))).to_sparse().to(DEV)   # stored entries outside M as well
    forms = [(V.to(DEV), Ms), (V.to(DEV).bfloat16(), Ms), (big[:, 3:3 + V.shape[1]], Ms), (Vsp, Ms),
             (V.masked_fill(~M, float("nan")).to(DEV), Ms), (V.to(DEV), dup), (V.to(DEV), Ms)]
    out = [_fit(Vf, W, H, Mf, 0.5)[:2] for Vf, Mf in forms]
    for Wg, Hg in out[1:]:
        assert torch.equal(Wg, out[0][0]) and torch.equal(Hg, out[0][1])


def test_cached_workspace_after_an_observed_fit_gives_the_unmasked_bits():
    from torchnmf_b200 import engine
    V, W, H, M = _inputs(200, 150, 24, 1, 0.3)
    Vd = V.to(DEV)
    engine.release_workspaces()
    first = _fit(Vd, W, H, None, 1, precision="f32")[:2]
    _fit(Vd, W, H, M.to(DEV).to_sparse(), 1)                    # the same cached "f32" context, observed cells set
    again = _fit(Vd, W, H, None, 1, precision="f32")[:2]
    assert torch.equal(first[0], again[0]) and torch.equal(first[1], again[1])


def test_rank_above_256_is_the_dense_mask_fit_bit_for_bit():
    V, W, H, M = _inputs(120, 90, 300, 0.5, 0.4)
    Vn = V.masked_fill(~M, float("nan")).to(DEV)
    a = _fit(Vn, W, H, M.to(DEV).to_sparse(), 0.5, max_iter=10)
    b = _fit(V.masked_fill(~M, 0.0).to(DEV), W, H, M.to(DEV), 0.5, max_iter=10)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    c = _fit(V.to(DEV).to_sparse(), W, H, M.to_sparse(), 0.5, max_iter=10)
    assert torch.equal(a[0], c[0]) and torch.equal(a[1], c[1])


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def test_repeat_fits_and_a_one_rank_gloo_group_give_the_unsharded_bits():
    import torch.distributed as dist
    V, W, H, M = _inputs(180, 120, 48, 1.5, 0.25)
    Vd, Ms = V.to(DEV), M.to(DEV).to_sparse()
    runs = [_fit(Vd, W, H, Ms, 1.5) for _ in range(2)]
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{_free_port()}", rank=0, world_size=1)
    try:
        sharded = _fit(Vd, W, H, Ms, 1.5, group=dist.group.WORLD)
    finally:
        dist.destroy_process_group()
    assert sharded[2] == runs[0][2]
    assert torch.equal(sharded[0], runs[0][0]) and torch.equal(sharded[1], runs[0][1])


def _worker(rank, world, port, out_dir):
    for p in (ROOT, os.path.join(ROOT, "pytorch-nmf_b200"), HERE):
        if p not in sys.path:
            sys.path.insert(0, p)
    import torch.distributed as dist
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    import test_gpu_observed as tg
    V, W, H, M = tg._inputs(301, 170, 40, 1, 0.2)
    n = V.shape[0]
    lo, hi = [0, (2 * n) // 3, n][rank], [0, (2 * n) // 3, n][rank + 1]
    Wg, Hg, n_iter, _ = tg._fit(V[lo:hi].to_sparse().to(tg.DEV), W, H[lo:hi], M[lo:hi].to_sparse().to(tg.DEV), 1,
                                group=dist.group.WORLD)
    torch.save({"W": Wg, "H": Hg, "n_iter": n_iter}, os.path.join(out_dir, f"rank{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


def test_two_gloo_processes_on_one_gpu_match_the_unsharded_fit(tmp_path):
    import torch.multiprocessing as mp
    mp.spawn(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    V, W, H, M = _inputs(301, 170, 40, 1, 0.2)
    Ws, Hs, n_single, _ = _fit(V.to(DEV), W, H, M.to(DEV).to_sparse(), 1)
    parts = [torch.load(os.path.join(tmp_path, f"rank{r}.pt")) for r in range(2)]
    assert all(p["n_iter"] == n_single for p in parts)
    assert torch.equal(parts[0]["W"], parts[1]["W"])
    assert torch.allclose(parts[0]["W"], Ws, rtol=1e-4, atol=1e-6 * float(Ws.max()))
    assert torch.allclose(torch.cat([p["H"] for p in parts]), Hs, rtol=1e-4, atol=1e-6 * float(Hs.max()))


# ---- past 2^31 cells ---------------------------------------------------------------------------------------------------------
def _sample_terms(O, F, G, seg, which, beta):
    """float64 terms of the segments `seg` (rows of H for which = 1, of W for which = 0) from the gathered factors."""
    rows, cols = O.indices()
    own, other = (cols, rows) if which == 0 else (rows, cols)
    sel = torch.isin(own, seg)
    pos = torch.searchsorted(seg, own[sel])
    fo = G[other[sel]].double()
    x = (F[own[sel]].double() * fo).sum(1)
    v = O.values()[sel].double()
    eps = 1.1920928955078125e-07
    a = {2: torch.ones_like(x), 1: 1 / (x + eps)}.get(beta, (x + eps) ** (beta - 2))
    b = {2: x, 1: torch.ones_like(x)}.get(beta, (x + eps) ** (beta - 1))
    num = torch.zeros(seg.numel(), F.shape[1], dtype=torch.float64, device=F.device).index_add_(0, pos, (v * a)[:, None] * fo)
    den = torch.zeros_like(num).index_add_(0, pos, b[:, None] * fo)
    return num, den


def test_fit_past_2_31_cells_on_little_memory():
    from torchnmf_b200 import NMF, engine
    N, C, R, nnz = 262144, 131072, 16, 1 << 20
    assert N * C > 2 ** 31
    g = torch.Generator(device=DEV).manual_seed(0)
    lin = torch.randint(0, N * C, (nnz,), device=DEV, generator=g)
    idx = torch.stack([lin // C, lin % C])
    W = torch.rand(C, R, device=DEV, generator=g) + 0.1
    H = torch.rand(N, R, device=DEV, generator=g) + 0.1
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(DEV)
    base = torch.cuda.memory_allocated(DEV)
    V = torch.sparse_coo_tensor(idx, torch.rand(nnz, device=DEV, generator=g), (N, C))
    M = torch.sparse_coo_tensor(idx, torch.ones(nnz, dtype=torch.bool, device=DEV), (N, C))
    O = _observed(V, M)
    eng = engine.CudaObservedNmfEngine(O, W.clone(), H.clone())
    try:
        for beta in (1, 0.5):
            for which, F, G in ((1, H, W), (0, W, H)):
                seg = torch.unique(O.indices()[1 - which])[:: 997][:64].contiguous()     # a sample of non-empty rows / columns
                num, den = eng.raw_terms(which, beta)
                wn, wd = _sample_terms(O, F, G, seg, which, beta)
                for got, want in ((num[seg], wn), (den[seg], wd)):
                    assert torch.allclose(got.double(), want, rtol=2e-4, atol=1e-6 * float(want.abs().max()))
        loss0 = eng.loss(1)
    finally:
        eng.close()
    m = NMF(W=W, H=H).to(DEV)
    assert m.fit(V, 1, float("-inf"), 20, mask=M) == 20
    eng = engine.CudaObservedNmfEngine(O, m.W.data, m.H.data)
    try:
        assert eng.loss(1) < loss0
    finally:
        eng.close()
    assert torch.cuda.max_memory_allocated(DEV) - base < 1 << 30
    engine.release_workspaces()
