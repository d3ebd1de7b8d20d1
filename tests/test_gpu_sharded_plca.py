"""Sharded PLCA / SIPLCA / SIPLCA2 / SIPLCA3 fits on the H100: PLCA's rows (dense or sparse COO V) or the clips of the
shift-invariant models split over the ranks, W and Z replicated, one all-reduce of [dW | dZ] per EM step around the
single fit's own kernels (the fp32 or tensor-core raw terms, the sliding kernels, the sparse gathers).

(a) A one-rank group is the unsharded fit bit for bit: n_iter, norm, W, H, Z and last_fit_precision.
(b) Two processes sharing one GPU over gloo, (c) two GPUs over NCCL: uneven shards give the same n_iter and norm on every
    rank as the unsharded fit of the whole target, bit-identical W and Z replicas, and W, H, Z within rtol 1e-4 of it
    (1e-3 at "f16", where each rank's tensor-core operands are its own shard's).
Every fit runs at a tol at which the unsharded fit stops at an interior check, and the divergence its stop rule sees at
every check must be the unsharded fit's (bit for bit with one rank): that checks the loss all-reduce.  The spawned ranks
have a deadline and a short collective timeout, so a desynchronised pair fails the test instead of holding the GPU."""
import datetime
import os
import socket
import sys

import pytest
import torch
import torch.distributed as dist

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
if HERE not in sys.path:
    sys.path.insert(0, HERE)

from sharded_plca_checks import interior_tol, recorded_losses, spawn  # noqa: E402

# name -> (model, V shape, W shape, precision, density of a sparse V (None: dense), (W_alpha, H_alpha, Z_alpha), shard bounds
# along axis 0).  Above rank 256 every row stores more entries than the rank, so the fit is not degenerate.  The alphas are
# close to 1, so that the loss still falls over several checks and the stop rule meets an interior check.
CASES = {
    "plca_f32": ("PLCA", (300, 257), (257, 24), "f32", None, (1., 1., 1.), [0, 180, 300]),
    "plca_f16": ("PLCA", (300, 257), (257, 24), "f16", None, (1., 1., 1.), [0, 180, 300]),
    "sparse_r64": ("PLCA", (400, 300), (300, 64), "f32", 0.1, (1.0001, 1.00002, 1.0002), [0, 250, 400]),
    "sparse_r300": ("PLCA", (1200, 1024), (1024, 300), "f32", 0.5, (1., 1., 1.), [0, 700, 1200]),
    "siplca_f32": ("SIPLCA", (5, 48, 200), (48, 16, 9), "f32", None, (1.0001, 1.00002, 1.0002), [0, 3, 5]),
    "siplca_f16": ("SIPLCA", (5, 48, 200), (48, 16, 9), "f16", None, (1., 1., 1.), [0, 3, 5]),
    "siplca2_f16": ("SIPLCA2", (5, 24, 10, 96), (24, 8, 3, 7), "f16", None, (1., 1., 1.), [0, 3, 5]),
    "siplca3_f32": ("SIPLCA3", (5, 8, 5, 6, 40), (8, 4, 2, 2, 5), "f32", None, (1., 1., 1.), [0, 3, 5]),
}
MAX_ITER = 100


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close()
    return p


def _case(name):
    """V with dyadic values (its sums are exact in fp32, so the shards' norms add up to the whole target's bit for bit) and
    W, H, Z normalised over the whole target."""
    from torchnmf_b200.plca import get_norm
    model, vs, ws = CASES[name][:3]
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    V = torch.randint(0, 64, vs, generator=g).float() / 16
    if CASES[name][4] is not None:
        V = V * (torch.rand(vs, generator=g) < CASES[name][4])
        V[:, 0] += 0.5                                   # every row stores an entry
    hs = (vs[0], ws[1]) + tuple(x - k + 1 for x, k in zip(vs[2:], ws[2:]))
    W, H, Z = torch.rand(ws, generator=g) + 0.1, torch.rand(hs, generator=g) + 0.1, torch.rand(ws[1], generator=g) + 0.1
    return V, W / get_norm(W), H / get_norm(H), Z / Z.sum()


def _fit(name, lo, hi, tol, group=None):
    """The fit of rows (clips) lo:hi: (module, n_iter, norm, the divergence at every check)."""
    import torchnmf_b200
    model, _, _, prec, density, alphas, _ = CASES[name]
    V, W, H, Z = _case(name)
    m = getattr(torchnmf_b200, model)(W=W, H=H[lo:hi], Z=Z).cuda()
    for p, x in ((m.W, W), (m.H, H[lo:hi]), (m.Z, Z)):
        p.data.copy_(x)                                  # the whole target's normalisation, not the shard's
    Vs = V[lo:hi].cuda()
    with recorded_losses() as losses:
        n, norm = m.fit(Vs if density is None else Vs.to_sparse(), tol, MAX_ITER, False, *alphas, precision=prec,
                        group=group)
    return m, n, norm, losses


def _stop_tol(name):
    """A tol at which the unsharded fit stops at an interior check (sharded_plca_checks.interior_tol)."""
    return interior_tol(_fit(name, 0, CASES[name][1][0], float("-inf"))[3])


# ---- (a) one-rank group ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(CASES))
def test_one_rank_group_is_the_unsharded_fit(name):
    whole, tol = CASES[name][1][0], _stop_tol(name)
    ref, n_ref, norm_ref, losses_ref = _fit(name, 0, whole, tol)
    dist.init_process_group("gloo", store=dist.HashStore(), rank=0, world_size=1)
    try:
        m, n, norm, losses = _fit(name, 0, whole, tol, group=dist.group.WORLD)
    finally:
        dist.destroy_process_group()
    assert m.last_fit_precision == ref.last_fit_precision == CASES[name][3]
    assert 9 <= n_ref < MAX_ITER - 1 and n == n_ref
    assert losses == losses_ref
    assert norm.dtype == norm_ref.dtype and torch.equal(norm, norm_ref)
    for nm in ("W", "H", "Z"):
        assert torch.equal(getattr(m, nm).data, getattr(ref, nm).data), nm


# ---- (b) two processes on one GPU over gloo, (c) two GPUs over NCCL ------------------------------------------------------------
def _worker(rank, world, port, backend, tols, out_dir):
    for p in (ROOT, os.path.join(ROOT, "pytorch-nmf_b200")):
        if p not in sys.path:
            sys.path.insert(0, p)
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    dev = rank if backend == "nccl" else 0
    torch.cuda.set_device(dev)
    timeout = datetime.timedelta(seconds=60)
    if backend == "nccl":
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", dev), timeout=timeout)
    else:
        dist.init_process_group("gloo", rank=rank, world_size=world, timeout=timeout)
    out = {}
    for name in CASES:
        bounds = CASES[name][6]
        m, n, norm, losses = _fit(name, bounds[rank], bounds[rank + 1], tols[name], group=dist.group.WORLD)
        out[name] = {"W": m.W.data.cpu(), "H": m.H.data.cpu(), "Z": m.Z.data.cpu(), "n": n, "norm": norm.cpu(),
                     "precision": m.last_fit_precision, "losses": losses}
    torch.save(out, os.path.join(out_dir, f"r{rank}.pt"))
    dist.barrier(); dist.destroy_process_group()


def _two_ranks_match_unsharded(tmp_path, backend):
    tols = {name: _stop_tol(name) for name in CASES}
    spawn(_worker, (2, _free_port(), backend, tols, str(tmp_path)), timeout=300)
    parts = [torch.load(os.path.join(tmp_path, f"r{r}.pt")) for r in range(2)]
    for name in CASES:
        ref, n_ref, norm_ref, losses_ref = _fit(name, 0, CASES[name][1][0], tols[name])
        a, b = parts[0][name], parts[1][name]
        assert 9 <= n_ref < MAX_ITER - 1, (name, n_ref)                                 # an interior stop
        assert a["n"] == b["n"] == n_ref, (name, a["n"], b["n"], n_ref)
        rtol = 1e-3 if CASES[name][3] == "f16" else 1e-4
        # the stop rule's divergences are the whole target's, the same bits on both ranks
        assert a["losses"] == b["losses"] and len(a["losses"]) == len(losses_ref), name
        assert torch.allclose(torch.tensor(a["losses"]), torch.tensor(losses_ref), rtol=rtol, atol=0), \
            (name, a["losses"], losses_ref)
        assert torch.equal(a["norm"], norm_ref.cpu()) and torch.equal(b["norm"], norm_ref.cpu()), name
        assert a["precision"] == b["precision"] == ref.last_fit_precision, name
        assert torch.equal(a["W"], b["W"]) and torch.equal(a["Z"], b["Z"]), name      # replicas stay bit-identical
        H = torch.cat([a["H"], b["H"]])
        for nm, got, want in (("W", a["W"], ref.W.data.cpu()), ("H", H, ref.H.data.cpu()), ("Z", a["Z"], ref.Z.data.cpu())):
            ok = torch.allclose(got, want, rtol=rtol, atol=1e-6 * float(want.abs().max()))
            assert ok, (name, nm, (got - want).abs().max().item(), float(want.abs().max()))


def test_two_processes_one_gpu_gloo(tmp_path):
    _two_ranks_match_unsharded(tmp_path, "gloo")


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpus_nccl(tmp_path):
    _two_ranks_match_unsharded(tmp_path, "nccl")
