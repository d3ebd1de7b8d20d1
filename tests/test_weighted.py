"""Fits with per-cell weights (`fit(V, ..., weight=Wt)`), without a GPU.

tests/golden/reference_weighted.npz holds fits of the unmodified reference's `trainer.BetaMu` with integer weights, each
cell gathered w times by the closure (tools/make_golden_weighted.py).  Here the float64 weighted oracle
(tests/weighted_oracle.py) is pinned to them, and the host logic of `fit(weight=...)` -- validation, staging, the sparse
weight's observed cells, the loop and the stop rule -- runs through a weighted oracle engine plugged in with the
`_engine_factory` hook.
"""
import ctypes
import datetime
import math
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from conftest import GOLDEN
import masked_oracle as mo
import weighted_oracle as wo

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def load_weighted():
    z = np.load(os.path.join(GOLDEN, "reference_weighted.npz"), allow_pickle=False)
    cases = {}
    for key in z.files:
        name, field = key.split("/", 1)
        v = z[key]
        if field in ("V", "Wt", "W0", "H0", "W", "H"):
            v = torch.from_numpy(v.copy())
        elif field == "kind":
            v = str(v)
        elif field == "losses":
            v = [float(x) for x in v]
        else:
            v = float(v)
            if field in ("n_iter", "max_iter", "trainable_W"):
                v = int(v)
        cases.setdefault(name, {})[field] = v
    return cases


CASES = load_weighted()


def _bars(c):
    # the reference runs in fp32 through autograd, the oracle in float64: the masked fixtures' bars
    return 2e-5 if c["kind"] == "nmf" else 5e-5


def _oracle_fit(c):
    return wo.fit(c["V"], c["W0"], c["H0"], c["Wt"], beta=c["beta"], tol=c["tol"], max_iter=c["max_iter"],
                  alpha=c["alpha"], l1_ratio=c["l1_ratio"], trainable_W=bool(c["trainable_W"]), kind=c["kind"])


@pytest.mark.parametrize("name", sorted(CASES))
def test_weighted_oracle_matches_reference_betamu(name):
    c = CASES[name]
    W, H, n_iter, losses = _oracle_fit(c)
    assert n_iter == c["n_iter"]
    rtol = _bars(c)
    assert torch.allclose(W.float(), c["W"], rtol=rtol, atol=1e-7), (W.float() - c["W"]).abs().max()
    assert torch.allclose(H.float(), c["H"], rtol=rtol, atol=1e-7), (H.float() - c["H"]).abs().max()
    assert len(losses) == len(c["losses"])
    for a, b in zip(losses, c["losses"]):
        assert math.isclose(a, b, rel_tol=1e-4, abs_tol=1e-6)


def test_fixtures_cover_the_contract():
    kinds = {(c["kind"], c["beta"]) for c in CASES.values()}
    assert {("nmf", b) for b in (0, 0.5, 1, 1.5, 2)} <= kinds
    assert {("nmfd", 1), ("nmfd", 0.5), ("nmfd", 2), ("nmf2d", 1), ("nmf2d", 0), ("nmf3d", 1.5)} <= kinds
    assert any(c["alpha"] > 0 for c in CASES.values())
    assert any(not c["trainable_W"] for c in CASES.values())
    assert any(math.isfinite(c["tol"]) for c in CASES.values())
    assert any(torch.isnan(c["V"]).any() for c in CASES.values())
    for c in CASES.values():
        assert set(c["Wt"].unique().tolist()) == {0.0, 1.0, 2.0, 3.0}
        assert torch.isnan(c["V"]).any() == bool(torch.isnan(c["V"][c["Wt"] == 0]).any())   # NaN only at weight 0


# ---- the host logic of fit(weight=...) on a weighted oracle engine ----------------------------------------------------
class WeightedOracleEngine:
    """The engine interface of torchnmf_b200.engine, with set_weight, on tests/weighted_oracle.py (float64 inside)."""
    device = torch.device("cpu")
    precision = "oracle"

    def __init__(self, V, W, H, model, weights=None):
        self.W, self.H, self.model = W, H, model
        self.kind = "nmf" if model == "nmf" else "nmfd"
        self.Wt = None
        if weights is not None:                     # a sparse weight's observed cells, as CudaObservedNmfEngine gets them
            assert V.is_sparse and V.is_coalesced() and weights.shape == (V._nnz(),) and weights.dtype == torch.float32
            assert bool((weights > 0).all())
            self.Wt = torch.zeros(V.shape, dtype=torch.float32)
            self.Wt[V.indices()[0], V.indices()[1]] = weights
            V = V.to_dense()
        self.V = V

    @classmethod
    def factory(cls, model, log=None):
        def make(V, W, H, weights=None):
            eng = cls(V, W, H, model, weights)
            if log is not None:
                log.append(eng)
            return eng
        return make

    def close(self):
        pass

    def sync(self):
        pass

    def set_weight(self, Wt):
        assert Wt is None or (Wt.dtype == torch.float32 and Wt.shape == self.V.shape and Wt.is_contiguous())
        self.Wt = Wt

    def precision_for(self, beta):
        return "f32"

    def minmax(self):
        Vo = self.V[self.Wt != 0]
        if Vo.numel() == 0:
            return float("inf"), float("-inf")
        return float(Vo.min()), float(Vo.max())

    def _d(self):
        return self.V.double(), self.W.double(), self.H.double(), self.Wt.double()

    def loss_tensor(self, beta):
        V, W, H, Wt = self._d()
        return wo.weighted_loss(mo.KINDS[self.model][0](H, W), V, Wt, beta).reshape(1)

    def loss(self, beta):
        return float(self.loss_tensor(beta))

    def update_w(self, beta, gamma, l1, l2):
        V, W, H, Wt = self._d()
        self.W.copy_(wo.weighted_update(V, W, H, Wt, beta, 0, self.model, gamma, l1, l2))

    def update_h(self, beta, gamma, l1, l2):
        V, W, H, Wt = self._d()
        self.H.copy_(wo.weighted_update(V, W, H, Wt, beta, 1, self.model, gamma, l1, l2))

    # sharded pieces: nmfb200_raw_terms(which = 0)'s layout while a weight is set (2 x the factor's numel at every beta)
    def w_partial(self, beta):
        V, W, H, Wt = self._d()
        num, den = wo.weighted_terms(V, W, H, Wt, beta, 0, self.model)
        return torch.cat([num.reshape(-1), den.reshape(-1)]).contiguous()

    def w_apply(self, reduced, beta, gamma, l1, l2):
        from oracle import mu_oracle as orc
        n = self.W.numel()
        num, den = reduced[:n].view(self.W.shape), reduced[n:].view(self.W.shape)
        self.W.copy_(orc._ratio_update(self.W.double(), num, den, gamma, l1, l2, False))


def _module(c, log=None):
    from torchnmf_b200 import NMF, NMF2D, NMF3D, NMFD
    cls = {"nmf": NMF, "nmfd": NMFD, "nmf2d": NMF2D, "nmf3d": NMF3D}[c["kind"]]
    m = cls(W=c["W0"], H=c["H0"], trainable_W=bool(c["trainable_W"]))
    m._engine_factory = WeightedOracleEngine.factory(c["kind"], log)
    return m


def _fit(c, V=None, weight=None, **kw):
    m = _module(c)
    n = m.fit(c["V"] if V is None else V, c["beta"], c["tol"], c["max_iter"], False, c["alpha"], c["l1_ratio"],
              weight=c["Wt"] if weight is None else weight, **kw)
    return m, n


@pytest.mark.parametrize("name", sorted(CASES))
def test_fit_with_weight_matches_reference_betamu(name):
    c = CASES[name]
    m, n_iter = _fit(c)
    assert n_iter == c["n_iter"]
    rtol = _bars(c)
    assert torch.allclose(m.W.data, c["W"], rtol=rtol, atol=1e-7)
    assert torch.allclose(m.H.data, c["H"], rtol=rtol, atol=1e-7)
    assert m.last_fit_precision == "f32"


@pytest.mark.parametrize("name", ["nmf_w03_b0.5", "nmf_w03_b1", "nmfd_w03_b2", "nmf2d_w03_b0"])
def test_zero_one_weights_give_the_masked_fit(name):
    c = CASES[name]
    M = c["Wt"] > 0
    args = dict(beta=c["beta"], tol=c["tol"], max_iter=c["max_iter"], alpha=c["alpha"], l1_ratio=c["l1_ratio"],
                kind=c["kind"])
    Wm, Hm, nm, lm = mo.fit(c["V"].double(), c["W0"].double(), c["H0"].double(), M, **args)
    Ww, Hw, nw, lw = wo.fit(c["V"], c["W0"], c["H0"], M.double(), **args)
    assert nm == nw
    assert torch.equal(Wm, Ww) and torch.equal(Hm, Hw)                     # the updates: bit for bit
    assert all(math.isclose(a, b, rel_tol=1e-12) for a, b in zip(lm, lw))    # the losses: summed in another order


def test_nan_and_garbage_at_zero_weight_cells_change_nothing():
    c = CASES["nmf_w03_b0.5"]
    out = []
    for fill in (0.0, float("nan"), float("inf"), -3.0):
        m, _ = _fit(c, V=c["V"].masked_fill(c["Wt"] == 0, fill))
        out.append((m.W.data.clone(), m.H.data.clone()))
    for W, H in out[1:]:
        assert torch.equal(W, out[0][0]) and torch.equal(H, out[0][1])


def test_validation_looks_at_weighted_cells_only():
    c = CASES["nmf_w03_b0"]                             # beta 0: V floored, no zero among the weighted cells
    off = c["Wt"] == 0
    V = c["V"].masked_fill(off, 0.0)
    miss = off.nonzero()[0]
    V[miss[0], miss[1]] = -1.0
    _fit(c, V=V)
    seen = (~off).nonzero()[0]
    V2 = V.clone(); V2[seen[0], seen[1]] = 0.0
    with pytest.raises(ValueError, match="beta <= 0"):
        _fit(c, V=V2)
    V3 = V.clone(); V3[seen[0], seen[1]] = -1.0
    with pytest.raises(AssertionError, match="non-negative"):
        _module(c).fit(V3, 1, float("-inf"), 10, weight=c["Wt"])


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float64])
def test_staged_weight_dtypes(dtype):
    c = CASES["nmf_w03_b1.5"]
    ref, _ = _fit(c)
    log = []
    m = _module(c, log)
    m.fit(c["V"], c["beta"], c["tol"], c["max_iter"], weight=c["Wt"].to(dtype))
    assert log[0].Wt.dtype == torch.float32                  # one fp32 copy; {0..3} are exact in every dtype
    assert torch.equal(m.W.data, ref.W.data) and torch.equal(m.H.data, ref.H.data)


def test_weight_errors():
    c = CASES["nmf_w03_b1"]
    V, Wt = c["V"], c["Wt"]
    m = _module(c)
    from torchnmf_b200 import NMFD
    with pytest.raises(ValueError, match="exclusive"):
        m.fit(V, mask=Wt > 0, weight=Wt)
    for bad in (Wt.to(torch.int64), Wt > 0, Wt.numpy()):
        with pytest.raises(ValueError, match="floating-point"):
            m.fit(V, weight=bad)
    for val in (-1.0, float("nan"), float("inf"), -float("inf")):
        W2 = Wt.clone(); W2[3, 4] = val
        with pytest.raises(ValueError, match="finite and >= 0"):
            m.fit(V, weight=W2)
    with pytest.raises(ValueError, match="shape"):
        m.fit(V, weight=Wt[:, :-1])
    with pytest.raises(ValueError, match="dense target"):
        m.fit(torch.nan_to_num(V).to_sparse(), weight=Wt)
    with pytest.raises(ValueError, match="zero"):
        m.fit(V, weight=torch.zeros_like(Wt))
    with pytest.raises(ValueError, match="zero"):
        m.fit(V, weight=torch.zeros_like(Wt).to_sparse())
    for prec in ("f16", "f16_split"):
        with pytest.raises(ValueError, match="fp32 kernels"):
            m.fit(V, precision=prec, weight=Wt)
    with pytest.raises(ValueError, match="finite and >= 0"):
        W2 = Wt.clone(); W2[0, 0] = -2.0
        m.fit(V, weight=W2.to_sparse())
    # a negative stored entry is refused even where a duplicate of the same cell would bring the sum above zero
    idx = torch.tensor([[0, 0, 1], [0, 0, 1]])
    with pytest.raises(ValueError, match="finite and >= 0"):
        m.fit(V, weight=torch.sparse_coo_tensor(idx, torch.tensor([-1.0, 2.0, 1.0]), Wt.shape))
    assert torch.equal(m.W.data, c["W0"]) and torch.equal(m.H.data, c["H0"])     # nothing ran
    cd = CASES["nmfd_w03_b1"]
    md = NMFD(W=cd["W0"], H=cd["H0"])
    with pytest.raises(ValueError, match="NMF only"):
        md.fit(cd["V"], weight=cd["Wt"].to_sparse())


@pytest.mark.parametrize("sparse_v", [False, True])
def test_sparse_weight_gives_the_dense_weight_fit(sparse_v):
    """A sparse weight: its stored entries with w > 0 are the observed cells, handed to the engine with their weights in
    the order of its coalesced values; duplicates add up and stored zeros drop out."""
    c = CASES["nmf_w03_b1.5"]
    ref, n_ref = _fit(c)
    Wt = c["Wt"]
    idx = Wt.nonzero().t()
    vals = Wt[idx[0], idx[1]]
    # split every weight 3 into 1 + 2 at a duplicated coordinate, and store a few explicit zeros
    three = vals == 3
    zeros = (Wt == 0).nonzero().t()[:, :5]
    idx = torch.cat([idx, idx[:, three], zeros], 1)
    vals = torch.cat([torch.where(three, 1.0, vals), torch.full((int(three.sum()),), 2.0), torch.zeros(5)])
    Ws = torch.sparse_coo_tensor(idx, vals, Wt.shape)
    assert not Ws.is_coalesced()
    V = torch.nan_to_num(c["V"])
    if sparse_v:
        V = V.to_sparse()
    log = []
    m = _module(c, log)
    n = m.fit(V, c["beta"], c["tol"], c["max_iter"], False, c["alpha"], c["l1_ratio"], weight=Ws)
    assert n == n_ref
    assert log[0].V.shape == Wt.shape and torch.equal(log[0].Wt, Wt)
    assert torch.equal(m.W.data, ref.W.data) and torch.equal(m.H.data, ref.H.data)


def test_weight_entry_points_are_bound_and_refuse_a_null_context():
    from torchnmf_b200 import _capi
    res, args = _capi.SIGNATURES["nmfb200_set_weight"]
    assert res is ctypes.c_int and args == [ctypes.c_void_p] * 3
    res, args = _capi.SIGNATURES["nmfb200_nmf_set_target_observed_weighted"]
    assert res is ctypes.c_int and args == [ctypes.c_void_p, ctypes.c_int64] + [ctypes.c_void_p] * 9
    lib = _capi.load()
    assert lib.nmfb200_set_weight(None, None, None) == 1                     # NMFB200_ERR_INVALID, before any device work
    assert b"null context" in lib.nmfb200_last_error()
    assert lib.nmfb200_nmf_set_target_observed_weighted(None, 0, None, None, None, None, None, None, None, None, None) == 1
    assert b"null context" in lib.nmfb200_last_error()
    header = open(os.path.join(ROOT, "include", "nmf_b200.h")).read()
    assert "int nmfb200_set_weight(nmfb200_ctx* ctx, const float* Wt, void* stream);" in header
    assert "int nmfb200_nmf_set_target_observed_weighted(nmfb200_ctx* ctx, int64_t nnz, const int64_t* crow," in header


# ---- the sharded protocol (gloo, two CPU processes): each rank passes the weight shard of its V shard --------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _sharded_case(c, zero_rows):
    """The fixture's weight with the rows [zero_rows:] zero everywhere (the second rank's whole shard)."""
    Wt = c["Wt"].clone()
    Wt[zero_rows:] = 0.0
    return Wt


def _worker(rank, world, port, name, sparse, bad_rank, out_dir):
    for p in (ROOT, os.path.join(ROOT, "pytorch-nmf_b200"), HERE):
        if p not in sys.path:
            sys.path.insert(0, p)
    torch.set_num_threads(1)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=120))
    import test_weighted as tw
    c = tw.CASES[name]
    n = c["V"].shape[0]
    lo, hi = [(0, (2 * n) // 3), ((2 * n) // 3, n)][rank]
    Wt = tw._sharded_case(c, (2 * n) // 3)[lo:hi].clone()
    if rank == bad_rank:
        Wt[0, 0] = -1.0
    m = tw._module(dict(c, H0=c["H0"][lo:hi]))
    out = {}
    try:
        out["n_iter"] = m.fit(c["V"][lo:hi], c["beta"], c["tol"], c["max_iter"], False, c["alpha"], c["l1_ratio"],
                              group=dist.group.WORLD, weight=Wt.to_sparse() if sparse else Wt)
        out.update(W=m.W.data, H=m.H.data)
    except ValueError as e:
        out["error"] = str(e)
    torch.save(out, os.path.join(out_dir, f"rank{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("sparse", [False, True])
def test_sharded_fit_with_an_all_zero_weight_shard(tmp_path, sparse):
    """The second rank's shard is zero everywhere (sparse: stores nothing): valid input, the rows of an all-missing shard,
    so the fit runs on every rank and equals the unsharded fit of the whole weight."""
    name = "nmf_w03_b1"
    c = CASES[name]
    mp.spawn(_worker, args=(2, _free_port(), name, sparse, None, str(tmp_path)), nprocs=2, join=True)
    n = c["V"].shape[0]
    ref, n_ref = _fit(c, weight=_sharded_case(c, (2 * n) // 3))
    parts = [torch.load(os.path.join(tmp_path, f"rank{r}.pt")) for r in range(2)]
    assert all("error" not in p and p["n_iter"] == n_ref for p in parts)
    assert torch.equal(parts[0]["W"], parts[1]["W"])
    assert torch.allclose(parts[0]["W"], ref.W.data, rtol=1e-4, atol=1e-7)
    assert torch.allclose(torch.cat([p["H"] for p in parts]), ref.H.data, rtol=1e-4, atol=1e-7)
    assert torch.equal(parts[1]["H"], c["H0"][(2 * n) // 3:])                # no weighted cell: its rows of H stay


@pytest.mark.parametrize("sparse", [False, True])
def test_sharded_bad_weight_on_one_rank_raises_on_every_rank(tmp_path, sparse):
    name = "nmf_w03_b1"
    mp.spawn(_worker, args=(2, _free_port(), name, sparse, 0, str(tmp_path)), nprocs=2, join=True)
    parts = [torch.load(os.path.join(tmp_path, f"rank{r}.pt")) for r in range(2)]
    assert all("finite and >= 0" in p.get("error", "") for p in parts)
