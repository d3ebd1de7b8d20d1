"""Batch-sharded NMFD / NMF2D / NMF3D fits on the H100: V and H split along the batch axis, W replicated, one all-reduce of
the W terms (nmfb200_raw_terms(which = 0)) before the ratio stage (nmfb200_w_apply).

(a) A one-rank group is the unsharded fit bit for bit: the partial folds the split slabs (and the tensor-core path's
    centring term) in the order the ratio stage does, the one-rank all-reduce is the identity, and the ratio stage on one
    pre-summed slab without a centring term sees the same numerator.
(b) Two processes sharing one GPU over gloo, (c) two GPUs over NCCL: uneven shards match the unsharded fit of the whole
    batch, and the W replicas stay bit-identical.
(d) The C ABI: the partial is the W raw terms, the pair is one W update, and the refusals."""
import ctypes
import os
import socket
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

# name -> (model, V shape, W shape, precision); B = 5 everywhere, so the two-rank shards are 3 + 2 batch elements
CASES = {
    "nmfd_f16": ("NMFD", (5, 48, 260), (48, 16, 9), "f16"),
    "nmfd_f32": ("NMFD", (5, 48, 260), (48, 16, 9), "f32"),
    "nmf2d_f16": ("NMF2D", (5, 24, 10, 96), (24, 8, 3, 7), "f16"),
    "nmf3d_f32": ("NMF3D", (5, 8, 5, 6, 40), (8, 4, 2, 2, 5), "f32"),
}
BOUNDS = [0, 3, 5]


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close()
    return p


def _case(name):
    model, vs, ws, prec = CASES[name]
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    V = torch.rand(vs, generator=g) + 0.05
    W0 = torch.rand(ws, generator=g) + 0.1
    H0 = torch.rand((vs[0], ws[1]) + tuple(x - k + 1 for x, k in zip(vs[2:], ws[2:])), generator=g) + 0.1
    return model, V, W0, H0, prec


def _fit(name, beta, lo, hi, max_iter, tol, group=None):
    import torchnmf_b200
    model, V, W0, H0, prec = _case(name)
    m = getattr(torchnmf_b200, model)(W=W0, H=H0[lo:hi]).cuda()
    n = m.fit(V[lo:hi].cuda(), beta, tol, max_iter, precision=prec, group=group)
    return m, n


def _uses_tc(name, beta):
    return CASES[name][3] == "f16" and beta == 1


# ---- (a) one-rank group ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("beta", [1, 0.5])
@pytest.mark.parametrize("name", list(CASES))
def test_one_rank_group_is_the_unsharded_fit(name, beta):
    ref, n_ref = _fit(name, beta, 0, 5, 30, 1e-4)
    dist.init_process_group("gloo", store=dist.HashStore(), rank=0, world_size=1)
    try:
        m, n = _fit(name, beta, 0, 5, 30, 1e-4, group=dist.group.WORLD)
    finally:
        dist.destroy_process_group()
    assert m.last_fit_precision == ref.last_fit_precision == ("f16" if _uses_tc(name, beta) else "f32")
    assert m.last_w_update_path == "nccl"
    assert n == n_ref
    assert torch.equal(m.W.data, ref.W.data)
    assert torch.equal(m.H.data, ref.H.data)


# ---- (b) two processes on one GPU over gloo, (c) two GPUs over NCCL ------------------------------------------------------------
def _worker(rank, world, port, backend, name, beta, out_dir):
    for p in (ROOT, os.path.join(ROOT, "pytorch-nmf_b200")):
        if p not in sys.path:
            sys.path.insert(0, p)
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    dev = rank if backend == "nccl" else 0
    torch.cuda.set_device(dev)
    if backend == "nccl":
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", dev))
    else:
        dist.init_process_group("gloo", rank=rank, world_size=world)
    m, n = _fit(name, beta, BOUNDS[rank], BOUNDS[rank + 1], 40, 1e-5, group=dist.group.WORLD)
    torch.save({"W": m.W.data.cpu(), "H": m.H.data.cpu(), "n": n, "path": m.last_w_update_path,
                "precision": m.last_fit_precision}, os.path.join(out_dir, f"r{rank}.pt"))
    dist.barrier(); dist.destroy_process_group()


def _two_ranks_match_unsharded(tmp_path, backend, name, beta):
    mp.spawn(_worker, args=(2, _free_port(), backend, name, beta, str(tmp_path)), nprocs=2, join=True)
    ref, n_ref = _fit(name, beta, 0, 5, 40, 1e-5)
    parts = [torch.load(os.path.join(tmp_path, f"r{r}.pt")) for r in range(2)]
    assert parts[0]["n"] == parts[1]["n"] == n_ref
    assert parts[0]["path"] == parts[1]["path"] == "nccl"
    assert parts[0]["precision"] == parts[1]["precision"] == ref.last_fit_precision
    assert torch.equal(parts[0]["W"], parts[1]["W"])                     # replicas stay bit-identical
    H = torch.cat([p["H"] for p in parts])
    for got, want in ((parts[0]["W"], ref.W.data.cpu()), (H, ref.H.data.cpu())):
        if _uses_tc(name, beta):         # fp16 operands, each rank centred and scaled on its own shard: the north-star bar
            ok = torch.allclose(got, want, rtol=1e-3, atol=1e-5 * float(want.abs().max()))
        else:
            ok = torch.allclose(got, want, rtol=1e-4, atol=1e-6 * float(want.abs().max()))
        assert ok, (got - want).abs().max().item()


TWO_RANK_CASES = [("nmfd_f32", 1), ("nmfd_f32", 0.5), ("nmfd_f16", 1), ("nmf2d_f16", 1)]


@pytest.mark.parametrize("name,beta", TWO_RANK_CASES)
def test_two_processes_one_gpu_gloo(tmp_path, name, beta):
    _two_ranks_match_unsharded(tmp_path, "gloo", name, beta)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("name,beta", TWO_RANK_CASES)
def test_two_gpus_nccl(tmp_path, name, beta):
    _two_ranks_match_unsharded(tmp_path, "nccl", name, beta)


# ---- (d) the C ABI -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,beta,l1,l2", [("nmfd_f16", 1, 0.0, 0.0), ("nmfd_f32", 0.5, 0.0, 0.0),
                                             ("nmf2d_f16", 1, 0.05, 0.05), ("nmf3d_f32", 2, 0.05, 0.05)])
def test_w_partial_is_w_raw_terms_and_w_apply_is_update_w(name, beta, l1, l2):
    from torchnmf_b200.engine import CudaNmfdEngine
    from torchnmf_b200.nmf import _gamma
    _, V, W0, H0, prec = _case(name)
    V = V.cuda()
    a, b = (CudaNmfdEngine(V, W0.cuda(), H0.cuda(), prec) for _ in range(2))
    try:
        lib = a._lib
        assert a.precision_for(beta) == ("f16" if _uses_tc(name, beta) else "f32")
        for _ in range(3):           # later rounds start from a ratio stage's tensor-core state: w_apply must leave it right
            num, den = a.raw_terms(0, beta)
            part = a.w_partial(beta)
            assert part.numel() == num.numel() + den.numel()
            assert torch.equal(part, torch.cat([num.reshape(-1), den.reshape(-1)]))
            a.w_apply(part, beta, _gamma(beta), l1, l2)
            b.update_w(beta, _gamma(beta), l1, l2)
            assert torch.equal(a.W, b.W)
            a.update_h(beta, _gamma(beta), l1, l2)
            b.update_h(beta, _gamma(beta), l1, l2)
            assert torch.equal(a.H, b.H)
        assert a.loss(beta) == b.loss(beta)
    finally:
        a.close()
        b.close()


def test_raw_terms_and_w_apply_refusals():
    from torchnmf_b200 import _capi
    lib = _capi.load()
    vp, st = ctypes.c_void_p, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    ERR_INVALID, ERR_STATE = 1, 3
    W, H = torch.rand(8, 4, 5, device="cuda"), torch.rand(2, 4, 36, device="cuda")
    V = torch.rand(2, 8, 40, device="cuda")
    buf = torch.empty(2 * W.numel(), device="cuda")
    w, h, v, p = vp(W.data_ptr()), vp(H.data_ptr()), vp(V.data_ptr()), vp(buf.data_ptr())
    assert lib.nmfb200_raw_terms_numel(None, 0, 1.0) == -1
    assert lib.nmfb200_raw_terms(None, w, h, 0, 1.0, p, st) == ERR_INVALID
    assert lib.nmfb200_w_apply(None, w, p, 1.0, 1.0, 0.0, 0.0, st) == ERR_INVALID

    nmf = vp()
    _capi.check(lib.nmfb200_nmf_create(ctypes.byref(nmf), 0, 64, 32, 4, _capi.PREC_F32))
    try:        # an NMF context takes the same calls: W terms of C * R (+ R at beta 1), and no ratio stage before a target
        assert lib.nmfb200_raw_terms_numel(nmf, 0, 1.0) == 32 * 4 + 4
        assert lib.nmfb200_w_apply(nmf, w, p, 1.0, 1.0, 0.0, 0.0, st) == ERR_STATE
    finally:
        lib.nmfb200_destroy(nmf)

    ctx = vp()
    _capi.check(lib.nmfb200_nmfnd_create(ctypes.byref(ctx), 0, 2, 8, 1, (ctypes.c_int64 * 1)(40), 4,
                                         (ctypes.c_int64 * 1)(5), _capi.PREC_F32))
    try:
        assert lib.nmfb200_raw_terms_numel(ctx, 0, 1.0) == W.numel() + 4
        assert lib.nmfb200_raw_terms_numel(ctx, 0, 0.5) == 2 * W.numel()
        assert lib.nmfb200_raw_terms(ctx, w, h, 0, 1.0, p, st) == ERR_STATE          # before set_target
        assert lib.nmfb200_w_apply(ctx, w, p, 1.0, 1.0, 0.0, 0.0, st) == ERR_STATE
        _capi.check(lib.nmfb200_nmfd_set_target(ctx, v, _capi.DTYPE_F32, st))
        assert lib.nmfb200_raw_terms(ctx, None, h, 0, 1.0, p, st) == ERR_INVALID
        assert lib.nmfb200_raw_terms(ctx, w, None, 0, 1.0, p, st) == ERR_INVALID
        assert lib.nmfb200_raw_terms(ctx, w, h, 0, 1.0, None, st) == ERR_INVALID
        assert lib.nmfb200_w_apply(ctx, None, p, 1.0, 1.0, 0.0, 0.0, st) == ERR_INVALID
        assert lib.nmfb200_w_apply(ctx, w, None, 1.0, 1.0, 0.0, 0.0, st) == ERR_INVALID
        assert lib.nmfb200_raw_terms(ctx, w, h, 0, 1.0, p, st) == 0
        assert lib.nmfb200_w_apply(ctx, w, p, 1.0, 1.0, 0.0, 0.0, st) == 0
        torch.cuda.synchronize()
        assert torch.isfinite(W).all() and (W > 0).all()
    finally:
        lib.nmfb200_destroy(ctx)
