"""Fits with per-cell weights (`fit(V, ..., weight=Wt)`, nmfb200_set_weight, nmfb200_nmf_set_target_observed_weighted) on
the GPU.

The weighted fp32 kernels are checked term by term against float64 (tests/weighted_oracle.py in double precision): the raw
numerators and denominators of both updates and the loss, for NMF off the 64-tile edges at ranks 1 to 300 and fp32, fp16,
bf16 and row-strided targets, for NMFD, NMF2D and NMF3D, and for the observed-cell gathers of a sparse weight at every
rank-floats-per-lane branch.  Then bit identities: a weight of M.float() against the mask M, a sparse weight of ones
against the sparse mask, a uniform power-of-two weight against an all-true mask; whole fits against the unmodified
reference's BetaMu fixtures (tests/golden/reference_weighted.npz); non-finite values at zero-weight cells; the reuse of a
cached workspace; the rank-300 densified sparse weight; and the sharded protocol over gloo.
"""
import os
import socket
import sys

import pytest
import torch

import weighted_oracle as wo
from test_weighted import CASES

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
DEV = torch.device("cuda", 0)
BETAS = (0, 0.5, 1, 1.5, 2)


def _engine_cls(kind):
    from torchnmf_b200 import engine
    return engine.CudaNmfEngine if kind == "nmf" else engine.CudaNmfdEngine


def _inputs(vshape, wshape, hshape, beta, seed=0, zero=0.3):
    """V, W, H and real-valued weights in [0.25, 4), 0 at a share `zero` of the cells."""
    g = torch.Generator().manual_seed(seed)
    V = torch.rand(*vshape, generator=g)
    if beta <= 0:
        V = V.clamp_min(2 ** -7)
    W = torch.rand(*wshape, generator=g) + 0.1
    H = torch.rand(*hshape, generator=g) + 0.1
    Wt = 0.25 + 3.75 * torch.rand(*vshape, generator=g)
    Wt = Wt.masked_fill(torch.rand(*vshape, generator=g) < zero, 0.0)
    return V, W, H, Wt


def _want(kind, V, W, H, Wt, beta):
    V64, W64, H64, Wt64 = V.double(), W.double(), H.double(), Wt.double()
    terms = [wo.weighted_terms(V64, W64, H64, Wt64, beta, which, kind) for which in (0, 1)]
    loss = float(wo.weighted_loss(wo.KINDS[kind][0](H64, W64), V64, Wt64, beta))
    return terms, loss


def _close(got, want, what):
    got = got.double().cpu()
    assert torch.allclose(got, want, rtol=2e-4, atol=1e-6 * float(want.abs().max())), (what, float((got - want).abs().max()))


def _check_engine(eng, W, H, terms, loss, beta, what):
    for which in (0, 1):
        num, den = eng.raw_terms(which, beta)
        f = W if which == 0 else H
        assert num.shape == f.shape and den.shape == f.shape
        _close(num, terms[which][0], (what, which, "num"))
        _close(den, terms[which][1], (what, which, "den"))
    got = eng.loss(beta)
    assert abs(got - loss) <= 1e-4 * abs(loss) + 1e-6, (what, got, loss)


def _check_terms(kind, V, W, H, Wt, beta, Vdev=None):
    terms, loss = _want(kind, V, W, H, Wt, beta)
    Wd, Hd = W.to(DEV), H.to(DEV)
    eng = _engine_cls(kind)(Vdev if Vdev is not None else V.to(DEV), Wd, Hd, "f32")
    try:
        eng.set_weight(Wt.to(DEV))
        assert eng.precision_for(beta) == "f32"
        _check_engine(eng, W, H, terms, loss, beta, (kind, beta))
    finally:
        eng.close()
    assert torch.equal(Wd.cpu(), W) and torch.equal(Hd.cpu(), H)


@pytest.mark.parametrize("beta", BETAS)
@pytest.mark.parametrize("R", [1, 16, 64, 200, 300])
@pytest.mark.parametrize("N,C", [(70, 130), (129, 65)])
def test_nmf_weighted_terms_against_float64(N, C, R, beta):
    V, W, H, Wt = _inputs((N, C), (C, R), (N, R), beta, seed=R)
    _check_terms("nmf", V, W, H, Wt, beta)


@pytest.mark.parametrize("beta", BETAS)
@pytest.mark.parametrize("vdtype", ["float16", "bfloat16", "strided"])
def test_nmf_weighted_terms_half_and_strided_targets(vdtype, beta):
    N, C, R = 97, 83, 16
    V, W, H, Wt = _inputs((N, C), (C, R), (N, R), beta, seed=3)
    if vdtype == "strided":
        big = torch.full((N, C + 13), float("nan"), device=DEV)
        big[:, 5:5 + C] = V.to(DEV)
        Vdev = big[:, 5:5 + C]
    else:
        Vdev = V.to(getattr(torch, vdtype)).to(DEV)
        V = Vdev.float().cpu()
    _check_terms("nmf", V, W, H, Wt, beta, Vdev)


ND_SHAPES = {           # name: (kind, V shape, kernel size, R)
    "nmfd": ("nmfd", (2, 21, 61), (5,), 4),
    "nmfd_wide": ("nmfd", (3, 70, 150), (9,), 40),
    "nmf2d": ("nmf2d", (2, 5, 12, 20), (2, 3), 3),
    "nmf3d": ("nmf3d", (1, 3, 6, 7, 16), (2, 2, 3), 3),
}


def _nd_inputs(shape, beta, seed=None):
    kind, vs, ks, R = ND_SHAPES[shape]
    B, C, X = vs[0], vs[1], vs[2:]
    return (kind,) + _inputs(vs, (C, R, *ks), (B, R, *(x - k + 1 for x, k in zip(X, ks))), beta,
                             seed=R if seed is None else seed)


@pytest.mark.parametrize("beta", BETAS)
@pytest.mark.parametrize("shape", sorted(ND_SHAPES))
def test_nmfnd_weighted_terms_against_float64(shape, beta):
    kind, V, W, H, Wt = _nd_inputs(shape, beta)
    _check_terms(kind, V, W, H, Wt, beta)


@pytest.mark.parametrize("beta", BETAS)
@pytest.mark.parametrize("R", [1, 40, 100, 256])          # 1, 2, 4 and 8 rank floats per lane
def test_observed_weighted_gathers_against_float64(R, beta):
    from torchnmf_b200 import engine
    N, C = 150, 90
    V, W, H, Wt = _inputs((N, C), (C, R), (N, R), beta, seed=R, zero=0.9)
    terms, loss = _want("nmf", V, W, H, Wt, beta)
    idx = (Wt > 0).nonzero().t()
    O = torch.sparse_coo_tensor(idx, V[idx[0], idx[1]], (N, C)).coalesce().to(DEV)
    Wd, Hd = W.to(DEV), H.to(DEV)
    eng = engine.CudaObservedNmfEngine(O, Wd, Hd, weights=Wt[idx[0], idx[1]].to(DEV))
    try:
        _check_engine(eng, W, H, terms, loss, beta, ("observed", R, beta))
    finally:
        eng.close()


# ---- bit identities --------------------------------------------------------------------------------------------------
def _terms_and_loss(eng, beta):
    out = [t.clone() for which in (0, 1) for t in eng.raw_terms(which, beta)]
    return out, float(eng.loss_tensor(beta).item())


def _fit(cls_kind, W0, H0, V, beta, iters=20, **kw):
    from torchnmf_b200 import NMF, NMF2D, NMFD
    cls = {"nmf": NMF, "nmfd": NMFD, "nmf2d": NMF2D}[cls_kind]
    m = cls(W=W0.to(DEV), H=H0.to(DEV))
    n = m.fit(V.to(DEV) if not V.is_sparse else V, beta, float("-inf"), iters, **kw)
    return m.W.data.cpu(), m.H.data.cpu(), n


def _nmf_case(R, beta, seed=0):
    return ("nmf",) + _inputs((150, 130), (130, R), (150, R), beta, seed=seed)


@pytest.mark.parametrize("beta", BETAS)
@pytest.mark.parametrize("case", ["nmf64", "nmf300", "nmfd", "nmf2d"])
def test_zero_one_weight_gives_the_bits_of_the_mask(case, beta):
    if case.startswith("nmf") and case[3:].isdigit():
        kind, V, W, H, Wt = _nmf_case(int(case[3:]), beta)
    else:
        kind, V, W, H, Wt = _nd_inputs(case, beta)
    M = Wt > 0
    Vd = V.to(DEV)
    out = []
    for sel in ("mask", "weight"):
        eng = _engine_cls(kind)(Vd, W.to(DEV), H.to(DEV), "f32")
        try:
            if sel == "mask":
                eng.set_mask(M.to(DEV))
            else:
                eng.set_weight(M.float().to(DEV))
            out.append(_terms_and_loss(eng, beta))
            eng.update_w(beta, 1.0, 0.0, 0.0)
            eng.update_h(beta, 1.0, 0.0, 0.0)
            out.append((eng.W.cpu(), eng.H.cpu()))
        finally:
            eng.close()
    (tm, lm), fm, (tw, lw), fw = out
    assert all(torch.equal(a, b) for a, b in zip(tm, tw)) and lm == lw
    assert torch.equal(fm[0], fw[0]) and torch.equal(fm[1], fw[1])
    a = _fit(kind, W, H, V, beta, mask=M.to(DEV))
    b = _fit(kind, W, H, V, beta, weight=M.float().to(DEV))
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and a[2] == b[2]


@pytest.mark.parametrize("beta", [0.5, 1, 2])
@pytest.mark.parametrize("R", [24, 300])
def test_sparse_ones_weight_gives_the_bits_of_the_sparse_mask(R, beta):
    _, V, W, H, Wt = _nmf_case(R, beta, seed=5)
    M = (Wt > 0).to_sparse()
    ones = torch.sparse_coo_tensor(M.indices(), torch.ones(M._nnz()), M.shape)
    a = _fit("nmf", W, H, V, beta, mask=M)
    b = _fit("nmf", W, H, V, beta, weight=ones)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


@pytest.mark.parametrize("beta", [0.5, 1, 2])
@pytest.mark.parametrize("k", [2, 4])
def test_uniform_power_of_two_weight_scales_terms_and_loss_exactly(k, beta):
    """w = 2^k: every term and the loss's sum scale by 2^k exactly; the updates keep the all-true mask's bits where the
    ratio stage's eps is absorbed (terms >= 4 here)."""
    N, C, R = 300, 200, 8
    g = torch.Generator().manual_seed(7)
    V = 1 + 4 * torch.rand(N, C, generator=g)
    W = torch.rand(C, R, generator=g) + 0.5
    H = torch.rand(N, R, generator=g) + 0.5
    Vd = V.to(DEV)
    res = []
    for sel in ("mask", "weight"):
        eng = _engine_cls("nmf")(Vd, W.to(DEV), H.to(DEV), "f32")
        try:
            if sel == "mask":
                eng.set_mask(torch.ones(N, C, dtype=torch.bool, device=DEV))
            else:
                eng.set_weight(torch.full((N, C), 2.0 ** k, device=DEV))
            terms, loss = _terms_and_loss(eng, beta)
            assert min(float(t.min()) for t in terms) >= 4
            eng.iterate(3, beta, 1.0, 0.0, 0.0)
            res.append((terms, loss, eng.W.cpu(), eng.H.cpu()))
        finally:
            eng.close()
    (tm, lm, Wm, Hm), (tw, lw, Ww, Hw) = res
    assert all(torch.equal(a * 2.0 ** k, b) for a, b in zip(tm, tw))
    assert lw == lm * 2.0 ** k
    assert torch.equal(Wm, Ww) and torch.equal(Hm, Hw)


@pytest.mark.parametrize("name", sorted(CASES))
def test_fit_with_weight_matches_reference_betamu(name):
    c = CASES[name]
    from torchnmf_b200 import NMF, NMF2D, NMF3D, NMFD
    cls = {"nmf": NMF, "nmfd": NMFD, "nmf2d": NMF2D, "nmf3d": NMF3D}[c["kind"]]
    m = cls(W=c["W0"].to(DEV), H=c["H0"].to(DEV), trainable_W=bool(c["trainable_W"]))
    n = m.fit(c["V"].to(DEV), c["beta"], c["tol"], c["max_iter"], False, c["alpha"], c["l1_ratio"], weight=c["Wt"].to(DEV))
    assert n == c["n_iter"]
    assert m.last_fit_precision == "f32"
    for got, want in ((m.W.data.cpu(), c["W"]), (m.H.data.cpu(), c["H"])):
        assert torch.allclose(got, want, rtol=1e-3, atol=1e-5 * float(want.abs().max())), (got - want).abs().max()
    if c["kind"] == "nmf":          # the same cells as a sparse weight, on the observed-cell gathers
        ms = NMF(W=c["W0"].to(DEV), H=c["H0"].to(DEV), trainable_W=bool(c["trainable_W"]))
        ms.fit(c["V"].to(DEV), c["beta"], c["tol"], c["max_iter"], False, c["alpha"], c["l1_ratio"],
               weight=c["Wt"].to_sparse())
        for got, want in ((ms.W.data.cpu(), c["W"]), (ms.H.data.cpu(), c["H"])):
            assert torch.allclose(got, want, rtol=1e-3, atol=1e-5 * float(want.abs().max()))


@pytest.mark.parametrize("kind", ["nmf", "nmfd"])
@pytest.mark.parametrize("beta", [0.5, 1, 2])
def test_non_finite_zero_weight_cells_give_the_bits_of_zeros(kind, beta):
    if kind == "nmf":
        _, V, W, H, Wt = _nmf_case(24, beta)
    else:
        kind, V, W, H, Wt = _nd_inputs("nmfd", beta)
    out = []
    for fill in (0.0, float("nan"), float("inf"), -1.0):
        out.append(_fit(kind, W, H, V.masked_fill(Wt == 0, fill), beta, weight=Wt.to(DEV)))
    for a in out[1:]:
        assert torch.equal(a[0], out[0][0]) and torch.equal(a[1], out[0][1])


def test_cached_workspace_after_a_weighted_fit_gives_the_unweighted_bits():
    from torchnmf_b200 import engine
    engine.release_workspaces()
    _, V, W, H, Wt = _nmf_case(32, 1)
    fresh = _fit("nmf", W, H, V, 1, precision="f32")
    _fit("nmf", W, H, V, 1, weight=Wt.to(DEV))
    again = _fit("nmf", W, H, V, 1, precision="f32")
    assert torch.equal(fresh[0], again[0]) and torch.equal(fresh[1], again[1])
    engine.release_workspaces()


@pytest.mark.parametrize("beta", [0.5, 1])
def test_rank_300_sparse_weight_equals_the_dense_weight_fit(beta):
    _, V, W, H, Wt = _nmf_case(300, beta, seed=9)
    a = _fit("nmf", W, H, V, beta, weight=Wt.to(DEV))
    b = _fit("nmf", W, H, V, beta, weight=Wt.to_sparse())
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float64])
def test_staged_weight_dtypes_give_the_fp32_bits(dtype):
    _, V, W, H, _ = _nmf_case(16, 1.5)
    Wt = torch.randint(0, 4, V.shape, generator=torch.Generator().manual_seed(1)).float()
    a = _fit("nmf", W, H, V, 1.5, weight=Wt.to(DEV))
    b = _fit("nmf", W, H, V, 1.5, weight=Wt.to(dtype).to(DEV))
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


# ---- the sharded protocol over gloo -------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, kind, sparse, zero_shard, out_dir):
    for p in (ROOT, os.path.join(ROOT, "pytorch-nmf_b200"), HERE):
        if p not in sys.path:
            sys.path.insert(0, p)
    import torch.distributed as dist
    import test_gpu_weighted as tw
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    kind_, V, W, H, Wt = tw._case(kind, zero_shard)
    n = V.shape[0]
    bounds = [0, (2 * n) // 3, n] if world == 2 else [0, n]
    lo, hi = bounds[rank], bounds[rank + 1]
    w = Wt[lo:hi].to_sparse() if sparse else Wt[lo:hi].to(tw.DEV)
    res = tw._fit(kind_, W, H[lo:hi], V[lo:hi], 1, group=dist.group.WORLD, weight=w)
    torch.save({"W": res[0], "H": res[1]}, os.path.join(out_dir, f"rank{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


def _case(kind, zero_shard=False):
    """zero_shard: the second rank's shard (the last third of the rows / batch elements) of weight 0 everywhere."""
    kind_, V, W, H, Wt = _nmf_case(24, 1, seed=11) if kind == "nmf" else _nd_inputs("nmfd_wide", 1, seed=11)
    if zero_shard:
        Wt[(2 * V.shape[0]) // 3:] = 0.0
    return kind_, V, W, H, Wt


@pytest.mark.parametrize("world,zero_shard", [(1, False), (2, False), (2, True)])
@pytest.mark.parametrize("kind,sparse", [("nmf", False), ("nmf", True), ("nmfd", False)])
def test_sharded_weighted_fit(tmp_path, kind, sparse, world, zero_shard):
    """zero_shard: one rank's shard is zero everywhere (sparse: stores nothing), which is valid input."""
    import torch.multiprocessing as mp
    mp.spawn(_worker, args=(world, _free_port(), kind, sparse, zero_shard, str(tmp_path)), nprocs=world, join=True)
    kind_, V, W, H, Wt = _case(kind, zero_shard)
    ref = _fit(kind_, W, H, V, 1, weight=Wt.to_sparse() if sparse else Wt.to(DEV))
    parts = [torch.load(os.path.join(tmp_path, f"rank{r}.pt")) for r in range(world)]
    Hs = torch.cat([p["H"] for p in parts])
    if world == 1:
        assert torch.equal(parts[0]["W"], ref[0]) and torch.equal(Hs, ref[1])
    else:
        assert torch.equal(parts[0]["W"], parts[1]["W"])
        assert torch.allclose(parts[0]["W"], ref[0], rtol=1e-4, atol=1e-7)
        assert torch.allclose(Hs, ref[1], rtol=1e-4, atol=1e-7)
