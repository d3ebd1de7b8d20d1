"""World-size-2 gloo test of the batch-sharded NMFD fit protocol on CPU.

Each rank owns a shard of V and H along the batch axis and a replica of W; `ShardedEngine` inserts one sum-all-reduce per
W update and one scalar all-reduce per loss evaluation.  The result must equal the unsharded fit (reduction order
differs, so a tight rtol rather than bit equality), and ranks whose sizes past the batch axis differ must be refused."""
import os
import socket
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (ROOT, os.path.join(ROOT, "pytorch-nmf_b200"), HERE):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from oracle import mu_oracle as orc  # noqa: E402
from oracle_engine import OracleNmfdEngine  # noqa: E402

B, C, L, R, T = 5, 6, 30, 3, 4
BOUNDS = [0, 3, B]          # uneven shards: 3 + 2 batch elements


class ShardableOracleNmfdEngine(OracleNmfdEngine):
    """The oracle NMFD engine plus the batch-sharded W update, in the buffer layout of nmfb200_raw_terms(which = 0)."""

    def w_partial(self, beta):
        num, den = self.raw_terms(0, beta)
        return torch.cat([num.reshape(-1), den.reshape(-1)]).contiguous()

    def w_apply(self, reduced, beta, gamma, l1, l2):
        n = self.W.numel()
        num = reduced[:n].view(self.W.shape)
        den = reduced[n:].view(1, -1, 1) if beta == 1 else reduced[n:].view(self.W.shape)
        self.W.copy_(orc._ratio_update(self.W, num, den, gamma, l1, l2, beta == 1))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _inputs():
    torch.manual_seed(0)
    V = torch.rand(B, C, L)
    torch.manual_seed(1)
    return V, torch.rand(C, R, T) + 0.1, torch.rand(B, R, L - T + 1) + 0.1


def _fit_worker(rank, world, port, beta, alpha, out_dir):
    torch.set_num_threads(1)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from torchnmf_b200 import NMFD
    V, W0, H0 = _inputs()
    lo, hi = BOUNDS[rank], BOUNDS[rank + 1]
    m = NMFD(W=W0, H=H0[lo:hi])
    m._engine_factory = ShardableOracleNmfdEngine
    n_iter = m.fit(V[lo:hi], beta, 1e-3, 40, False, alpha, 0.5, group=dist.group.WORLD)
    torch.save({"W": m.W.data, "H": m.H.data, "n_iter": n_iter, "path": m.last_w_update_path},
               os.path.join(out_dir, f"rank{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("beta,alpha", [(1, 0), (0.5, 0), (2, 0), (1, 0.1)])
def test_batch_sharded_nmfd_equals_single(tmp_path, beta, alpha):
    world = 2
    mp.spawn(_fit_worker, args=(world, _free_port(), beta, alpha, str(tmp_path)), nprocs=world, join=True)
    from torchnmf_b200 import NMFD
    V, W0, H0 = _inputs()
    ref = NMFD(W=W0, H=H0)
    ref._engine_factory = ShardableOracleNmfdEngine
    n_ref = ref.fit(V, beta, 1e-3, 40, False, alpha, 0.5)
    parts = [torch.load(os.path.join(tmp_path, f"rank{r}.pt")) for r in range(world)]
    assert all(p["n_iter"] == n_ref for p in parts)          # identical stop decision on every rank
    assert all(p["path"] == "nccl" for p in parts)            # the all-reduce W update (no peer-memory path for NMFD)
    assert torch.equal(parts[0]["W"], parts[1]["W"])          # W replicas stay bit-identical
    H = torch.cat([p["H"] for p in parts])
    assert torch.allclose(parts[0]["W"], ref.W.data, rtol=1e-4, atol=1e-7)
    assert torch.allclose(H, ref.H.data, rtol=1e-4, atol=1e-7)


def _mismatch_worker(rank, world, port, what, out_dir):
    torch.set_num_threads(1)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from torchnmf_b200 import NMFD
    c, t = C, T
    if rank == 1:
        c, t = (C + 1, T) if what == "C" else (C, T + 2)
    V = torch.rand(2, c, L)
    m = NMFD(W=torch.rand(c, R, t), H=torch.rand(2, R, L - t + 1))
    m._engine_factory = ShardableOracleNmfdEngine
    try:
        m.fit(V, 1, 1e-3, 5, group=dist.group.WORLD)
        err = None
    except ValueError as e:
        err = str(e)
    torch.save({"err": err}, os.path.join(out_dir, f"rank{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("what,named", [("C", "C from 6 to 7"), ("T", "kernel_size[0] from 4 to 6")])
def test_batch_sharded_nmfd_refuses_different_sizes(tmp_path, what, named):
    world = 2
    mp.spawn(_mismatch_worker, args=(world, _free_port(), what, str(tmp_path)), nprocs=world, join=True)
    errs = [torch.load(os.path.join(tmp_path, f"rank{r}.pt"))["err"] for r in range(world)]
    for err in errs:                                          # every rank raises, so none waits in a collective
        assert err is not None and named in err, err
    assert "C=6" in errs[0] and f"C={7 if what == 'C' else 6}" in errs[1]
