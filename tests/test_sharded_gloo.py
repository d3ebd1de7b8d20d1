"""World-size-2 gloo test of the row-sharded fit protocol on CPU.

Each rank owns a row shard of V and H and a replica of W; `ShardedEngine` inserts one sum-all-reduce
per W update and one scalar all-reduce per loss evaluation.  The result must equal the unsharded fit
(reduction order differs, so a tight rtol rather than bit equality)."""
import os
import socket
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, beta, alpha, out_dir):
    for p in (ROOT, os.path.join(ROOT, "pytorch-nmf_b200"), HERE):
        if p not in sys.path:
            sys.path.insert(0, p)
    torch.set_num_threads(1)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from torchnmf_b200 import NMF
    from oracle_engine import OracleNmfEngine
    torch.manual_seed(0)
    N, C, R = 64, 30, 5
    V = torch.rand(N, C) + (0.01 if beta <= 0 else 0.0)
    torch.manual_seed(1)
    W0 = torch.randn(C, R).abs()
    H0 = torch.randn(N, R).abs()
    # uneven shard on purpose: rank 0 gets 40 rows, rank 1 gets 24
    bounds = [0, 40, N]
    lo, hi = bounds[rank], bounds[rank + 1]
    m = NMF(W=W0, H=H0[lo:hi])
    m._engine_factory = OracleNmfEngine
    n_iter = m.fit(V[lo:hi], beta, 1e-3, 40, False, alpha, 0.5, group=dist.group.WORLD)
    torch.save({"W": m.W.data, "H": m.H.data, "n_iter": n_iter, "lo": lo, "hi": hi},
               os.path.join(out_dir, f"rank{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("beta,alpha", [(1, 0), (0.5, 0.1), (2, 0)])
def test_sharded_fit_equals_single(tmp_path, beta, alpha):
    world = 2
    port = _free_port()
    mp.spawn(_worker, args=(world, port, beta, alpha, str(tmp_path)), nprocs=world, join=True)
    sys.path.insert(0, HERE)
    from torchnmf_b200 import NMF
    from oracle_engine import OracleNmfEngine
    torch.manual_seed(0)
    N, C, R = 64, 30, 5
    V = torch.rand(N, C) + (0.01 if beta <= 0 else 0.0)
    torch.manual_seed(1)
    W0 = torch.randn(C, R).abs()
    H0 = torch.randn(N, R).abs()
    ref = NMF(W=W0, H=H0)
    ref._engine_factory = OracleNmfEngine
    n_ref = ref.fit(V, beta, 1e-3, 40, False, alpha, 0.5)
    parts = [torch.load(os.path.join(tmp_path, f"rank{r}.pt")) for r in range(world)]
    assert all(p["n_iter"] == n_ref for p in parts)          # identical stop decision on every rank
    assert torch.equal(parts[0]["W"], parts[1]["W"])          # W replicas stay bit-identical
    H = torch.cat([p["H"] for p in parts])
    assert torch.allclose(parts[0]["W"], ref.W.data, rtol=1e-4, atol=1e-7)
    assert torch.allclose(H, ref.H.data, rtol=1e-4, atol=1e-7)
