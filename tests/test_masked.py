"""Fits on the observed cells of the target only (`fit(V, ..., mask=M)`), without a GPU.

tests/golden/reference_masked.npz holds fits of the unmodified reference's `trainer.BetaMu` with the closure
`(V[M], model()[M])` (tools/make_golden_masked.py).  Here the masked CPU oracle (tests/masked_oracle.py) is pinned to them,
and the host logic of `fit` -- mask validation, the observed-cell min / max checks, the loop, the stop rule, the sharded
protocol -- runs through a masked oracle engine plugged in with the `_engine_factory` hook.
"""
import ctypes
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

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def load_masked(fname="reference_masked.npz"):
    z = np.load(os.path.join(GOLDEN, fname), allow_pickle=False)
    cases = {}
    for key in z.files:
        name, field = key.split("/", 1)
        v = z[key]
        if field in ("V", "M", "W0", "H0", "W", "H"):
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


CASES = load_masked()


def _bars(c):
    # the bars of tests/test_oracle.py: closed form vs autograd differ only inside BLAS / conv reductions
    return 2e-5 if c["kind"] == "nmf" else 5e-5


def _oracle_fit(c):
    return mo.fit(c["V"], c["W0"], c["H0"], c["M"], beta=c["beta"], tol=c["tol"], max_iter=c["max_iter"],
                  alpha=c["alpha"], l1_ratio=c["l1_ratio"], trainable_W=bool(c["trainable_W"]), kind=c["kind"])


@pytest.mark.parametrize("name", sorted(CASES))
def test_masked_oracle_matches_reference_betamu(name):
    c = CASES[name]
    torch.set_num_threads(1)
    W, H, n_iter, losses = _oracle_fit(c)
    assert n_iter == c["n_iter"]
    rtol = _bars(c)
    assert torch.allclose(W, c["W"], rtol=rtol, atol=1e-7), (W - c["W"]).abs().max()
    assert torch.allclose(H, c["H"], rtol=rtol, atol=1e-7), (H - c["H"]).abs().max()
    assert len(losses) == len(c["losses"])
    for a, b in zip(losses, c["losses"]):
        assert math.isclose(a, b, rel_tol=1e-4, abs_tol=1e-6)


def test_fixtures_cover_the_contract():
    kinds = {(c["kind"], c["beta"]) for c in CASES.values()}
    assert {("nmf", b) for b in (0, 0.5, 1, 1.5, 2)} <= kinds
    assert {("nmfd", 1), ("nmfd", 0.5), ("nmfd", 2), ("nmf2d", 1), ("nmf2d", 0), ("nmf3d", 1.5)} <= kinds
    assert any(c["alpha"] > 0 for c in CASES.values())
    assert any(not c["trainable_W"] for c in CASES.values())
    assert any(c["n_iter"] < c["max_iter"] for c in CASES.values())           # a finite tol that stops early
    for c in CASES.values():
        missing = 1 - float(c["M"].float().mean())
        assert 0.05 < missing < 0.45
        assert torch.isnan(c["V"]).any() == bool(torch.isnan(c["V"][~c["M"]]).any())   # NaN only where missing


def test_fully_missing_rows_and_columns_keep_their_factor_rows():
    """A row of V with no observed cell leaves its row of H where it was (num = den = 0, ratio (0 + eps) / (0 + eps)),
    a missing column its row of W -- in the reference and in the oracle."""
    for name in ("nmf_rowcol_b1", "nmf_rowcol_b0.5"):
        c = CASES[name]
        rows = [n for n in range(c["M"].shape[0]) if not c["M"][n].any()]
        cols = [k for k in range(c["M"].shape[1]) if not c["M"][:, k].any()]
        assert rows == [5, 60] and cols == [7, 50]
        W, H, _, _ = _oracle_fit(c)
        for got in (c["H"], H):
            assert torch.equal(got[rows], c["H0"][rows])
        for got in (c["W"], W):
            assert torch.equal(got[cols], c["W0"][cols])


# ---- the host logic of fit(mask=...) on a masked oracle engine --------------------------------------------------------
class MaskedOracleEngine:
    """The engine interface of torchnmf_b200.engine, with set_mask, on tests/masked_oracle.py."""
    device = torch.device("cpu")
    precision = "oracle"

    def __init__(self, V, W, H, model):
        self.V, self.W, self.H, self.model = V, W, H, model
        self.kind = "nmf" if model == "nmf" else "nmfd"
        self.M = None

    @classmethod
    def factory(cls, model):
        return lambda V, W, H: cls(V, W, H, model)

    def close(self):
        pass

    def sync(self):
        pass

    def set_mask(self, M):
        assert M is None or (M.dtype == torch.bool and M.shape == self.V.shape)
        self.M = M

    def precision_for(self, beta):
        return "f32"

    def minmax(self):
        Vo = self.V[self.M]
        if Vo.numel() == 0:
            return float("inf"), float("-inf")
        return float(Vo.min()), float(Vo.max())

    def loss_tensor(self, beta):
        return mo.masked_loss(mo.KINDS[self.model][0](self.H, self.W), self.V, self.M, beta).double().reshape(1)

    def loss(self, beta):
        return float(self.loss_tensor(beta))

    def update_w(self, beta, gamma, l1, l2):
        self.W.copy_(mo.masked_update(self.V, self.W, self.H, self.M, beta, 0, self.model, gamma, l1, l2))

    def update_h(self, beta, gamma, l1, l2):
        self.H.copy_(mo.masked_update(self.V, self.W, self.H, self.M, beta, 1, self.model, gamma, l1, l2))

    # sharded pieces: nmfb200_raw_terms(which = 0)'s layout while a mask is set (2 x the factor's numel at every beta)
    def w_partial(self, beta):
        num, den = mo.masked_terms(self.V, self.W, self.H, self.M, beta, 0, self.model)
        return torch.cat([num.reshape(-1), den.reshape(-1)]).contiguous()

    def w_apply(self, reduced, beta, gamma, l1, l2):
        n = self.W.numel()
        num, den = reduced[:n].view(self.W.shape), reduced[n:].view(self.W.shape)
        from oracle import mu_oracle as orc
        self.W.copy_(orc._ratio_update(self.W, num, den, gamma, l1, l2, False))


def _module(c):
    from torchnmf_b200 import NMF, NMF2D, NMF3D, NMFD
    cls = {"nmf": NMF, "nmfd": NMFD, "nmf2d": NMF2D, "nmf3d": NMF3D}[c["kind"]]
    m = cls(W=c["W0"], H=c["H0"], trainable_W=bool(c["trainable_W"]))
    m._engine_factory = MaskedOracleEngine.factory(c["kind"])
    return m


@pytest.mark.parametrize("name", sorted(CASES))
def test_fit_with_mask_matches_reference_betamu(name):
    c = CASES[name]
    torch.set_num_threads(1)
    m = _module(c)
    n_iter = m.fit(c["V"], c["beta"], c["tol"], c["max_iter"], False, c["alpha"], c["l1_ratio"], mask=c["M"])
    assert n_iter == c["n_iter"]
    rtol = _bars(c)
    assert torch.allclose(m.W.data, c["W"], rtol=rtol, atol=1e-7)
    assert torch.allclose(m.H.data, c["H"], rtol=rtol, atol=1e-7)
    assert m.last_fit_precision == "f32"


def test_nan_and_garbage_in_missing_cells_change_nothing():
    c = CASES["nmf_rand30_b0.5"]
    out = []
    for fill in (0.0, float("nan"), float("inf"), -3.0):
        m = _module(c)
        m.fit(c["V"].masked_fill(~c["M"], fill), 0.5, float("-inf"), 10, mask=c["M"])
        out.append((m.W.data.clone(), m.H.data.clone()))
    for W, H in out[1:]:
        assert torch.equal(W, out[0][0]) and torch.equal(H, out[0][1])


def test_validation_looks_at_observed_cells_only():
    c = CASES["nmf_rand30_b0"]                         # beta 0: V floored, no zero among the observed cells
    V = c["V"].masked_fill(~c["M"], 0.0)               # zeros, and a negative value, where nothing is observed
    miss = (~c["M"]).nonzero()[0]
    V[miss[0], miss[1]] = -1.0
    m = _module(c)
    m.fit(V, 0, float("-inf"), 10, mask=c["M"])       # neither the non-negativity assert nor the beta <= 0 check fires
    seen = c["M"].nonzero()[0]
    V2 = V.clone(); V2[seen[0], seen[1]] = 0.0
    with pytest.raises(ValueError, match="beta <= 0"):
        _module(c).fit(V2, 0, float("-inf"), 10, mask=c["M"])
    V3 = V.clone(); V3[seen[0], seen[1]] = -1.0
    with pytest.raises(AssertionError, match="non-negative"):
        _module(c).fit(V3, 1, float("-inf"), 10, mask=c["M"])


def test_mask_errors():
    c = CASES["nmf_rand30_b1"]
    V, M = c["V"], c["M"]
    m = _module(c)
    with pytest.raises(ValueError, match="torch.bool"):
        m.fit(V, mask=M.to(torch.uint8))
    with pytest.raises(ValueError, match="torch.bool"):
        m.fit(V, mask=M.numpy())
    with pytest.raises(ValueError, match="shape"):
        m.fit(V, mask=M[:, :-1])
    with pytest.raises(ValueError, match="dense target"):
        m.fit(torch.nan_to_num(V).to_sparse(), mask=M)
    for prec in ("f16", "f16_split"):
        with pytest.raises(ValueError, match="fp32 kernels"):
            m.fit(V, precision=prec, mask=M)
    with pytest.raises(ValueError, match="no cell"):
        m.fit(V, mask=torch.zeros_like(M))
    with pytest.raises(TypeError, match="unexpected keyword"):
        m.fit(V, masks=M)
    assert torch.equal(m.W.data, c["W0"]) and torch.equal(m.H.data, c["H0"])     # nothing ran


def test_set_mask_is_bound_and_refuses_a_null_context():
    from torchnmf_b200 import _capi
    res, args = _capi.SIGNATURES["nmfb200_set_mask"]
    assert res is ctypes.c_int and args == [ctypes.c_void_p] * 3
    lib = _capi.load()
    assert lib.nmfb200_set_mask(None, None, None) == 1                      # NMFB200_ERR_INVALID, before any device work
    assert b"null context" in lib.nmfb200_last_error()
    header = open(os.path.join(ROOT, "include", "nmf_b200.h")).read()
    assert "int nmfb200_set_mask(nmfb200_ctx* ctx, const uint8_t* M, void* stream);" in header


# ---- the sharded protocol (gloo, two CPU processes): each rank passes the mask shard of its V shard ----------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, name, out_dir):
    for p in (ROOT, os.path.join(ROOT, "pytorch-nmf_b200"), HERE):
        if p not in sys.path:
            sys.path.insert(0, p)
    torch.set_num_threads(1)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import test_masked as tm
    c = tm.CASES[name]
    n = c["V"].shape[0]
    bounds = [0, (2 * n) // 3, n]                     # uneven shards (NMF: rows; NMFD: the batch axis)
    lo, hi = bounds[rank], bounds[rank + 1]
    shard = dict(c, H0=c["H0"][lo:hi])
    m = tm._module(shard)
    n_iter = m.fit(c["V"][lo:hi], c["beta"], c["tol"], c["max_iter"], False, c["alpha"], c["l1_ratio"],
                   group=dist.group.WORLD, mask=c["M"][lo:hi])
    torch.save({"W": m.W.data, "H": m.H.data, "n_iter": n_iter}, os.path.join(out_dir, f"rank{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("name", ["nmf_rand30_b1", "nmf_rowcol_b0.5", "nmfd_rand30_b2"])
def test_sharded_masked_fit_equals_single(tmp_path, name):
    world = 2
    mp.spawn(_worker, args=(world, _free_port(), name, str(tmp_path)), nprocs=world, join=True)
    c = CASES[name]
    ref = _module(c)
    n_ref = ref.fit(c["V"], c["beta"], c["tol"], c["max_iter"], False, c["alpha"], c["l1_ratio"], mask=c["M"])
    parts = [torch.load(os.path.join(tmp_path, f"rank{r}.pt")) for r in range(world)]
    assert all(p["n_iter"] == n_ref for p in parts)
    assert torch.equal(parts[0]["W"], parts[1]["W"])                      # the W replicas stay bit-identical
    assert torch.allclose(parts[0]["W"], ref.W.data, rtol=1e-4, atol=1e-7)
    assert torch.allclose(torch.cat([p["H"] for p in parts]), ref.H.data, rtol=1e-4, atol=1e-7)
