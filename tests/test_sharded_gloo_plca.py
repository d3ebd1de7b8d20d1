"""World-size-2 gloo test of the sharded PLCA / SIPLCA fits on CPU, through the float64 oracle engines of
tests/test_plca.py and tests/test_sparse_plca.py (SIPLCA2: the SIPLCA one over the oracle's two-axis contractions).

PLCA shards the rows of V and H (dense or sparse COO V), SIPLCA / SIPLCA2 the batch axis; W and Z are replicated.  Each
EM step sums [dW | dZ] over the ranks in one all-reduce, H's column sums in one more where the update divides by them
(W and Z frozen, H_alpha != 1), and the loss every 10th iteration.  The result must equal the unsharded fit of the whole
target (a different summation order: a tight rtol, not bit equality), with the same n_iter and norm on every rank and
bit-identical replicas of W and Z.  Each fit runs at a tol at which the unsharded fit stops at an interior check, and the
divergence the stop rule sees at every check must be the unsharded fit's: that checks the loss all-reduce, which a
rank stopping on its own shard's loss would fail.  A one-rank group is the unsharded fit bit for bit.  Checks that fail on one rank
only are agreed first, so every rank raises and none waits in a collective; every spawn has a timeout."""
import datetime
import os
import socket
import sys

import pytest
import torch
import torch.distributed as dist

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (ROOT, os.path.join(ROOT, "pytorch-nmf_b200"), HERE):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from oracle import mu_oracle as orc  # noqa: E402
from sharded_plca_checks import interior_tol, recorded_losses, spawn  # noqa: E402
from test_plca import PlcaOracleEngine, SiplcaOracleEngine  # noqa: E402
from test_sparse_plca import OracleSparsePlcaEngine  # noqa: E402
from torchnmf_b200 import PLCA, SIPLCA, SIPLCA2, BatchedPLCA  # noqa: E402
from torchnmf_b200.plca import get_norm  # noqa: E402


class Siplca2OracleEngine(SiplcaOracleEngine):
    """SiplcaOracleEngine over two shifted axes: the oracle's NMF2D reconstruction and contractions."""
    _recon = staticmethod(orc.nmfnd_reconstruct)
    _grad_w = staticmethod(lambda G, H, W: orc.nmfnd_grad_w(G, H, W.shape[2:]))
    _grad_h = staticmethod(lambda G, W, H: orc.nmfnd_grad_h(G, W, H.shape[2:]))


# model -> (class, V shape, W shape, shard bounds along axis 0, oracle engine).  Ranks large enough for the loss to fall
# over many checks, so that the stop rule has interior checks to choose from.
MODELS = {
    "plca_dense": (PLCA, (64, 40), (40, 12), [0, 40, 64], PlcaOracleEngine),
    "plca_sparse": (PLCA, (64, 40), (40, 12), [0, 40, 64], OracleSparsePlcaEngine),
    "siplca": (SIPLCA, (5, 12, 40), (12, 6, 5), [0, 3, 5], SiplcaOracleEngine),
    "siplca2": (SIPLCA2, (5, 6, 10, 14), (6, 5, 2, 3), [0, 3, 5], Siplca2OracleEngine),
}
# prior -> (trainable_W, trainable_Z, W_alpha, H_alpha, Z_alpha)
PRIORS = {
    "plain": (True, True, 1., 1., 1.),
    "alphas": (True, True, 1.001, 1.0002, 1.002),
    "frozen_z": (True, False, 1., 1., 1.),
    "frozen_wz": (False, False, 1., 1., 1.),
}
# the dense fits stage V through fp32, so their modules are fp32; the sparse fit runs in the factors' dtype
DTYPE = {model: torch.float64 if model == "plca_sparse" else torch.float32 for model in MODELS}
MAX_ITER = 60


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _inputs(model):
    """V with dyadic values (every partial sum is exact, so the shards' norms add up to the whole target's bit for bit),
    and W, H, Z normalised in float64 over the whole target."""
    cls, vs, ws, _, _ = MODELS[model]
    g = torch.Generator().manual_seed(sum(map(ord, model)))
    V = torch.randint(0, 64, vs, generator=g).double() / 16
    if model == "plca_sparse":
        V = V * (torch.rand(vs, generator=g) < 0.3)
        V[:, 0] += 0.5                                   # every row stores an entry
        V = V.to_sparse()
    hs = (vs[0], ws[1]) + tuple(x - k + 1 for x, k in zip(vs[2:], ws[2:]))
    W, H, Z = torch.rand(ws, generator=g) + 0.1, torch.rand(hs, generator=g) + 0.1, torch.rand(ws[1], generator=g) + 0.1
    W, H, Z = W.double(), H.double(), Z.double()
    return V, W / get_norm(W), H / get_norm(H), Z / Z.sum()


def _rows(V, lo, hi):
    return V.to_dense()[lo:hi].to_sparse() if V.is_sparse else V[lo:hi]


def _fit(model, prior, tol, lo=None, hi=None, group=None):
    """The fit of rows (clips) lo:hi on the oracle engine: (module, n_iter, norm, the divergence at every check)."""
    cls, vs, _, _, engine = MODELS[model]
    lo, hi = (0, vs[0]) if lo is None else (lo, hi)
    tw, tz, wa, ha, za = PRIORS[prior]
    V, W, H, Z = _inputs(model)
    m = cls(W=W, H=H[lo:hi], Z=Z, trainable_W=tw, trainable_Z=tz).to(DTYPE[model])
    for p, x in ((m.W, W), (m.H, H[lo:hi]), (m.Z, Z)):
        p.data.copy_(x)                                  # the whole target's normalisation, not the shard's
    m._engine_factory = engine
    with recorded_losses() as losses:
        n_iter, norm = m.fit(_rows(V, lo, hi), tol, MAX_ITER, False, wa, ha, za, group=group)
    return m, n_iter, norm, losses


def _stop_tol(model, prior):
    """A tol at which the unsharded fit stops at an interior check (sharded_plca_checks.interior_tol)."""
    return interior_tol(_fit(model, prior, float("-inf"))[3])


def _init(rank, world, port):
    torch.set_num_threads(1)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=60))


def _fit_worker(rank, world, port, model, tols, out_dir):
    _init(rank, world, port)
    bounds = MODELS[model][3]
    out = {}
    for prior in PRIORS:
        m, n_iter, norm, losses = _fit(model, prior, tols[prior], bounds[rank], bounds[rank + 1], group=dist.group.WORLD)
        out[prior] = {"W": m.W.data, "H": m.H.data, "Z": m.Z.data, "n_iter": n_iter, "norm": norm, "losses": losses}
    torch.save(out, os.path.join(out_dir, f"rank{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("model", list(MODELS))
def test_two_ranks_equal_the_unsharded_fit(tmp_path, model):
    tols = {prior: _stop_tol(model, prior) for prior in PRIORS}
    spawn(_fit_worker, (2, _free_port(), model, tols, str(tmp_path)))
    parts = [torch.load(os.path.join(tmp_path, f"rank{r}.pt")) for r in range(2)]
    for prior in PRIORS:
        ref, n_ref, norm_ref, losses_ref = _fit(model, prior, tols[prior])
        assert 9 <= n_ref < MAX_ITER - 1, (prior, n_ref)                                  # an interior stop
        a, b = parts[0][prior], parts[1][prior]
        assert a["n_iter"] == b["n_iter"] == n_ref, (prior, a["n_iter"], b["n_iter"], n_ref)
        # the stop rule's divergences are the whole target's, the same bits on both ranks
        assert a["losses"] == b["losses"] and len(a["losses"]) == len(losses_ref), prior
        assert torch.allclose(torch.tensor(a["losses"]), torch.tensor(losses_ref), rtol=1e-5, atol=0), \
            (prior, a["losses"], losses_ref)
        assert a["norm"].dtype == norm_ref.dtype and torch.equal(a["norm"], norm_ref) and torch.equal(b["norm"], norm_ref)
        assert torch.equal(a["W"], b["W"]) and torch.equal(a["Z"], b["Z"]), prior        # replicas stay bit-identical
        H = torch.cat([a["H"], b["H"]])
        for nm, got, want in (("W", a["W"], ref.W.data), ("H", H, ref.H.data), ("Z", a["Z"], ref.Z.data)):
            assert torch.allclose(got, want, rtol=1e-4, atol=1e-9 * float(want.abs().max())), \
                (prior, nm, float((got - want).abs().max()))
        if not PRIORS[prior][0]:
            assert torch.equal(a["W"], ref.W.data)                                        # a frozen W stays as given


@pytest.fixture
def one_rank_group():
    dist.init_process_group("gloo", store=dist.HashStore(), rank=0, world_size=1)
    try:
        yield dist.group.WORLD
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("prior", list(PRIORS))
@pytest.mark.parametrize("model", list(MODELS))
def test_one_rank_group_is_the_unsharded_fit(one_rank_group, model, prior):
    tol = _stop_tol(model, prior)
    ref, n_ref, norm_ref, losses_ref = _fit(model, prior, tol)
    m, n_iter, norm, losses = _fit(model, prior, tol, group=one_rank_group)
    assert n_iter == n_ref and norm.dtype == norm_ref.dtype and torch.equal(norm, norm_ref)
    assert losses == losses_ref
    assert m.last_fit_precision == ref.last_fit_precision == "oracle"
    for nm in ("W", "H", "Z"):
        assert torch.equal(getattr(m, nm).data, getattr(ref, nm).data), nm


def test_refusals_before_any_collective(one_rank_group):
    V, W, H, Z = _inputs("plca_dense")
    m = PLCA(W=W, H=H, Z=Z)
    m._engine_factory = PlcaOracleEngine
    with pytest.raises(ValueError, match="mask with group"):
        m.fit(V.float(), mask=torch.ones(V.shape, dtype=torch.bool), group=one_rank_group)
    with pytest.raises(TypeError):
        BatchedPLCA((2, 8, 6), 3).fit(torch.rand(2, 8, 6), group=one_rank_group)


# ---- checks that fail on one rank only: every rank raises ---------------------------------------------------------------------
def _scenario(name, rank):
    """(module, V shard) of rank `rank` in a refusal scenario: rank 1 holds the fault, except for 'zero_mass', where every
    shard stores only zeros."""
    V, W, H, Z = _inputs("plca_dense")
    lo, hi = (0, 40) if rank == 0 else (40, 64)
    cls, Vr = PLCA, V[lo:hi].clone()
    Hr, Wr = H[lo:hi], W
    if name == "negative" and rank == 1:
        Vr[3, 2] = -1.
    elif name == "shape" and rank == 1:
        Vr = V[lo - 1:hi]                                # one row more than its H
    elif name == "sizes" and rank == 1:
        Vr, Wr = torch.cat([Vr, Vr[:, :1]], 1), torch.cat([W, W[:1]], 0)     # C = 41 against rank 0's 40
    elif name == "sizes_siplca":
        V, W, H, Z = _inputs("siplca")
        cls, Vr, Hr, Wr = SIPLCA, V[:2], H[:2], W
        if rank == 1:
            Wr, Hr = torch.rand(12, 6, 7) + 0.1, H[:2, :, :34]                # T = 7 against rank 0's 5
    elif name == "no_rows" and rank == 1:
        Vr, Hr = V[64:], H[64:]                          # a shard of zero rows
    if name in ("empty", "zero_mass") or name.startswith("sparse_"):
        Vr = Vr.to_sparse()
        if name == "empty" and rank == 1:
            Vr = torch.sparse_coo_tensor(torch.zeros(2, 0, dtype=torch.long), torch.zeros(0, dtype=V.dtype), Vr.shape)
        if name == "zero_mass":
            Vr = torch.sparse_coo_tensor(Vr.indices(), torch.zeros_like(Vr.values()), Vr.shape)
    m = cls(W=Wr, H=Hr, Z=Z).to(torch.float64 if Vr.is_sparse else torch.float32)
    m._engine_factory = OracleSparsePlcaEngine if Vr.is_sparse else \
        (PlcaOracleEngine if cls is PLCA else SiplcaOracleEngine)
    return m, Vr


SCENARIOS = {
    "negative": (AssertionError, ["Target should be non-negative"] * 2),
    "shape": (ValueError, ["another rank does not match", "target shape (25, 40) does not match"]),
    "sizes": (ValueError, ["C from 40 to 41"] * 2),
    "sizes_siplca": (ValueError, ["kernel_size[0] from 5 to 7"] * 2),
    "empty": (ValueError, ["the target shard of another rank is empty", "the sparse target stores no entry"]),
    "no_rows": (ValueError, ["the target shard of another rank is empty", "this rank's target shard (0, 40) is empty"]),
    "zero_mass": (ValueError, ["the sparse target's values sum to 0"] * 2),
}


def _refusal_worker(rank, world, port, out_dir):
    _init(rank, world, port)
    out = {}
    for name in SCENARIOS:
        m, Vr = _scenario(name, rank)
        try:
            m.fit(Vr, 1e-4, 5, group=dist.group.WORLD)
            out[name] = None
        except (AssertionError, ValueError) as e:
            out[name] = (type(e).__name__, str(e))
    torch.save(out, os.path.join(out_dir, f"rank{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


def test_one_rank_faults_raise_on_every_rank(tmp_path):
    spawn(_refusal_worker, (2, _free_port(), str(tmp_path)))
    parts = [torch.load(os.path.join(tmp_path, f"rank{r}.pt")) for r in range(2)]
    for name, (exc, texts) in SCENARIOS.items():
        for rank, text in enumerate(texts):
            got = parts[rank][name]
            assert got is not None and got[0] == exc.__name__ and text in got[1], (name, rank, got)
