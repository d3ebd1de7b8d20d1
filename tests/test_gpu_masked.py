"""Fits on the observed cells of the target only (`fit(V, ..., mask=M)`, nmfb200_set_mask) on the GPU.

The masked fp32 kernels are checked term by term against float64 (tests/masked_oracle.py in double precision): the raw
numerators and denominators of both updates and the loss, for NMF off the 64-tile edges at ranks 1 to 300 and fp32, fp16,
bf16 and row-strided targets, and for NMFD, NMF2D and NMF3D.  Then whole fits: against the unmodified reference's BetaMu
fixtures (tests/golden/reference_masked.npz), an all-true mask against the unmasked fit, the reuse of a cached workspace,
repeat calls, and the sharded protocol over gloo.
"""
import os
import socket
import sys

import pytest
import torch

import masked_oracle as mo
from test_masked import CASES

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
DEV = torch.device("cuda", 0)
BETAS = (0, 0.5, 1, 1.5, 2)


def _engine_cls(kind):
    from torchnmf_b200 import engine
    return engine.CudaNmfEngine if kind == "nmf" else engine.CudaNmfdEngine


def _inputs(vshape, wshape, hshape, beta, seed=0, missing=0.3):
    g = torch.Generator().manual_seed(seed)
    V = torch.rand(*vshape, generator=g)
    if beta <= 0:
        V = V.clamp_min(2 ** -7)
    W = torch.rand(*wshape, generator=g) + 0.1
    H = torch.rand(*hshape, generator=g) + 0.1
    M = torch.rand(*vshape, generator=g) >= missing
    return V, W, H, M


def _want(kind, V, W, H, M, beta):
    """float64 raw terms of both updates and the loss."""
    V64, W64, H64 = V.double(), W.double(), H.double()
    terms = [mo.masked_terms(V64, W64, H64, M, beta, which, kind) for which in (0, 1)]
    loss = float(mo.masked_loss(mo.KINDS[kind][0](H64, W64), V64, M, beta))
    return terms, loss


def _check_terms(kind, V, W, H, M, beta, Vdev=None):
    """Vdev: the target as the engine reads it (another dtype or a strided view of V's values)."""
    terms, loss = _want(kind, V, W, H, M, beta)
    Wd, Hd = W.to(DEV), H.to(DEV)
    eng = _engine_cls(kind)(Vdev if Vdev is not None else V.to(DEV), Wd, Hd, "f32")
    try:
        eng.set_mask(M.to(DEV))
        assert eng.precision_for(beta) == "f32"
        for which in (0, 1):
            num, den = eng.raw_terms(which, beta)
            f = W if which == 0 else H
            assert num.shape == f.shape and den.shape == f.shape
            for got, want in ((num, terms[which][0]), (den, terms[which][1])):
                got = got.double().cpu()
                assert torch.allclose(got, want, rtol=2e-4, atol=1e-6 * float(want.abs().max())), \
                    (kind, beta, which, float((got - want).abs().max()))
        got = eng.loss(beta)
        assert abs(got - loss) <= 1e-4 * abs(loss) + 1e-6, (got, loss)
    finally:
        eng.close()
    assert torch.equal(Wd.cpu(), W) and torch.equal(Hd.cpu(), H)              # raw terms leave the factors alone


@pytest.mark.parametrize("beta", BETAS)
@pytest.mark.parametrize("R", [1, 16, 64, 200, 300])
@pytest.mark.parametrize("N,C", [(70, 130), (129, 65)])
def test_nmf_masked_terms_against_float64(N, C, R, beta):
    V, W, H, M = _inputs((N, C), (C, R), (N, R), beta, seed=R)
    _check_terms("nmf", V, W, H, M, beta)


@pytest.mark.parametrize("beta", BETAS)
@pytest.mark.parametrize("vdtype", ["float16", "bfloat16", "strided"])
def test_nmf_masked_terms_half_and_strided_targets(vdtype, beta):
    N, C, R = 97, 83, 16
    V, W, H, M = _inputs((N, C), (C, R), (N, R), beta, seed=3)
    if vdtype == "strided":
        big = torch.full((N, C + 13), float("nan"), device=DEV)
        big[:, 5:5 + C] = V.to(DEV)
        Vdev = big[:, 5:5 + C]
    else:
        Vdev = V.to(getattr(torch, vdtype)).to(DEV)
        V = Vdev.float().cpu()
    _check_terms("nmf", V, W, H, M, beta, Vdev)


ND_SHAPES = {           # name: (kind, V shape, kernel size, R)
    "nmfd": ("nmfd", (2, 21, 61), (5,), 4),
    "nmfd_wide": ("nmfd", (3, 70, 150), (9,), 40),
    "nmf2d": ("nmf2d", (2, 5, 12, 20), (2, 3), 3),
    "nmf3d": ("nmf3d", (1, 3, 6, 7, 16), (2, 2, 3), 3),
}


@pytest.mark.parametrize("beta", BETAS)
@pytest.mark.parametrize("shape", sorted(ND_SHAPES))
def test_nmfnd_masked_terms_against_float64(shape, beta):
    kind, vs, ks, R = ND_SHAPES[shape]
    B, C, X = vs[0], vs[1], vs[2:]
    V, W, H, M = _inputs(vs, (C, R, *ks), (B, R, *(x - k + 1 for x, k in zip(X, ks))), beta, seed=R)
    _check_terms(kind, V, W, H, M, beta)


@pytest.mark.parametrize("kind", ["nmf", "nmfd"])
@pytest.mark.parametrize("beta", [0.5, 1, 2])
def test_non_finite_missing_cells_give_the_bits_of_zeros(kind, beta):
    if kind == "nmf":
        V, W, H, M = _inputs((150, 90), (90, 24), (150, 24), beta)
    else:
        V, W, H, M = _inputs((2, 21, 61), (21, 4, 5), (2, 4, 57), beta)
    out = []
    for fill in (0.0, float("nan"), float("inf"), -1.0):
        Wd, Hd = W.to(DEV), H.to(DEV)
        eng = _engine_cls(kind)(V.masked_fill(~M, fill).to(DEV), Wd, Hd, "f32")
        try:
            eng.set_mask(M.to(DEV))
            res = [t.cpu() for which in (0, 1) for t in eng.raw_terms(which, beta)]
            res.append(torch.tensor(eng.loss(beta), dtype=torch.float64))
            assert eng.minmax() == (float(V[M].min()), float(V[M].max()))
            eng.update_w(beta, 1.0, 0.0, 0.0)
            eng.update_h(beta, 1.0, 0.0, 0.0)
            res += [Wd.cpu(), Hd.cpu()]
        finally:
            eng.close()
        out.append(res)
    for res in out[1:]:
        assert all(torch.equal(a, b) for a, b in zip(res, out[0]))


def _module(c, device=DEV):
    from torchnmf_b200 import NMF, NMF2D, NMF3D, NMFD
    cls = {"nmf": NMF, "nmfd": NMFD, "nmf2d": NMF2D, "nmf3d": NMF3D}[c["kind"]]
    return cls(W=c["W0"], H=c["H0"], trainable_W=bool(c["trainable_W"])).to(device)


def _fit(c, **kw):
    m = _module(c)
    n = m.fit(c["V"].to(DEV), c["beta"], c["tol"], c["max_iter"], False, c["alpha"], c["l1_ratio"], mask=c["M"].to(DEV),
              **kw)
    return m, n


@pytest.mark.parametrize("name", sorted(CASES))
def test_fit_matches_reference_betamu(name):
    c = CASES[name]
    m, n_iter = _fit(c)
    assert n_iter == c["n_iter"]
    assert m.last_fit_precision == "f32"
    for got, want in ((m.W.data.cpu(), c["W"]), (m.H.data.cpu(), c["H"])):
        assert torch.allclose(got, want, rtol=1e-3, atol=1e-5 * float(want.abs().max())), \
            float((got - want).abs().max())


def test_fit_on_host_buffers_and_auto_precision():
    c = CASES["nmf_rand30_b1"]
    m = _module(c, "cpu")
    n = m.fit(c["V"], 1, c["tol"], c["max_iter"], mask=c["M"])             # CPU module: staged through the device
    assert n == c["n_iter"] and m.last_fit_precision == "f32" and m.W.device.type == "cpu"
    assert torch.allclose(m.W.data, c["W"], rtol=1e-3, atol=1e-5 * float(c["W"].max()))


@pytest.mark.parametrize("beta", [1, 0.5, 2])
@pytest.mark.parametrize("kind", ["nmf", "nmfd"])
def test_all_true_mask_is_the_unmasked_fit(kind, beta):
    from torchnmf_b200 import NMF, NMFD
    if kind == "nmf":
        V, W, H, _ = _inputs((300, 200), (200, 32), (300, 32), beta)
        cls = NMF
    else:
        V, W, H, _ = _inputs((2, 21, 61), (21, 4, 5), (2, 4, 57), beta)
        cls = NMFD
    out = []
    for mask in (None, torch.ones(V.shape, dtype=torch.bool, device=DEV)):
        m = cls(W=W, H=H).to(DEV)
        kw = {} if mask is None else {"mask": mask}
        m.fit(V.to(DEV), beta, float("-inf"), 20, precision="f32", **kw)
        out.append((m.W.data.cpu(), m.H.data.cpu()))
    for a, b in zip(out[0], out[1]):
        assert torch.allclose(b, a, rtol=1e-5, atol=1e-6 * float(a.abs().max())), float((b - a).abs().max())


@pytest.mark.parametrize("kind", ["nmf", "nmfd"])
def test_cached_workspace_after_a_masked_fit_gives_the_unmasked_bits(kind):
    from torchnmf_b200 import engine
    c = CASES["nmf_rand30_b1" if kind == "nmf" else "nmfd_rand30_b1"]
    V = torch.nan_to_num(c["V"], nan=0.5).to(DEV)

    def unmasked():
        m = _module(c)
        m.fit(V, 1, float("-inf"), 20, precision="f32")
        return m.W.data.cpu(), m.H.data.cpu()

    engine.release_workspaces()
    first = unmasked()
    _fit(c, precision="f32")                    # the same cached "f32" context, with a mask set
    again = unmasked()
    assert torch.equal(first[0], again[0]) and torch.equal(first[1], again[1])


def test_repeat_fits_and_a_poisoned_workspace_give_the_same_bits():
    from torchnmf_b200 import engine
    for name in ("nmf_rowcol_b0.5", "nmfd_rand30_b0.5"):
        c = CASES[name]
        runs = []
        for poison in (False, False, True):
            if poison:
                engine.release_workspaces()
                junk = torch.full((64 << 20,), float("nan"), device=DEV)      # 256 MB of NaN, handed back to the driver
                del junk
                torch.cuda.synchronize()
                torch.cuda.empty_cache()
            m, _ = _fit(c)
            runs.append((m.W.data.cpu(), m.H.data.cpu()))
        for W, H in runs[1:]:
            assert torch.equal(W, runs[0][0]) and torch.equal(H, runs[0][1])


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def test_one_rank_gloo_group_is_the_unsharded_fit():
    import torch.distributed as dist
    c = CASES["nmf_rand30_b0.5"]
    single, n_single = _fit(c)
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{_free_port()}", rank=0, world_size=1)
    try:
        sharded, n_sharded = _fit(c, group=dist.group.WORLD)
    finally:
        dist.destroy_process_group()
    assert n_sharded == n_single
    assert torch.equal(sharded.W.data, single.W.data) and torch.equal(sharded.H.data, single.H.data)


def _worker(rank, world, port, name, out_dir):
    for p in (ROOT, os.path.join(ROOT, "pytorch-nmf_b200"), HERE):
        if p not in sys.path:
            sys.path.insert(0, p)
    import torch.distributed as dist
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    import test_gpu_masked as tg
    c = tg.CASES[name]
    n = c["V"].shape[0]
    lo, hi = [0, (2 * n) // 3, n][rank], [0, (2 * n) // 3, n][rank + 1]
    shard = dict(c, V=c["V"][lo:hi], M=c["M"][lo:hi], H0=c["H0"][lo:hi])
    m, n_iter = tg._fit(shard, group=dist.group.WORLD)
    torch.save({"W": m.W.data.cpu(), "H": m.H.data.cpu(), "n_iter": n_iter}, os.path.join(out_dir, f"rank{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("name", ["nmf_rand30_b1", "nmfd_rand30_b2"])
def test_two_gloo_processes_on_one_gpu_match_the_unsharded_fit(tmp_path, name):
    import torch.multiprocessing as mp
    mp.spawn(_worker, args=(2, _free_port(), name, str(tmp_path)), nprocs=2, join=True)
    single, n_single = _fit(CASES[name])
    parts = [torch.load(os.path.join(tmp_path, f"rank{r}.pt")) for r in range(2)]
    assert all(p["n_iter"] == n_single for p in parts)
    assert torch.equal(parts[0]["W"], parts[1]["W"])
    W = single.W.data.cpu()
    assert torch.allclose(parts[0]["W"], W, rtol=1e-4, atol=1e-6 * float(W.max()))
    H = single.H.data.cpu()
    assert torch.allclose(torch.cat([p["H"] for p in parts]), H, rtol=1e-4, atol=1e-6 * float(H.max()))
