"""Fits on the observed cells of a sparse mask (`NMF.fit(V, ..., mask=M)` with a sparse COO `M`), without a GPU.

The observed set is built once per fit, on the device, as a coalesced fp32 COO tensor whose stored entries are exactly the
observed cells (explicit zeros kept); the `_engine_factory` test hook receives that tensor.  Here an oracle engine on
tests/masked_oracle.py takes it, so the extraction, the validation on the observed values, the loop and the sharded protocol
are checked against tests/golden/reference_masked.npz (dense targets) and tests/golden/reference_observed.npz (sparse
targets, tools/make_golden_observed.py: the unmodified reference's BetaMu with the closure `(V.to_dense()[M], model()[M])`).
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
import test_masked as tm

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def load_observed():
    z = np.load(os.path.join(GOLDEN, "reference_observed.npz"), allow_pickle=False)
    cases = {}
    for key in z.files:
        name, field = key.split("/", 1)
        v = z[key]
        if field in ("V", "S", "M", "W0", "H0", "W", "H"):
            v = torch.from_numpy(v.copy())
        elif field == "losses":
            v = [float(x) for x in v]
        else:
            v = float(v)
            if field in ("n_iter", "max_iter", "trainable_W"):
                v = int(v)
        cases.setdefault(name, {})[field] = v
    return cases


OBS = load_observed()
NMF_MASKED = sorted(n for n, c in tm.CASES.items() if c["kind"] == "nmf")


def sparse_target(c):
    """The case's sparse target: V's values where S says an entry is stored."""
    return torch.sparse_coo_tensor(c["S"].nonzero().t(), c["V"][c["S"]], c["V"].shape).coalesce()


class ObservedOracleEngine(tm.MaskedOracleEngine):
    """The masked oracle engine on the observed-cell tensor the fit builds (the stored entries are the observed cells)."""
    received = []

    def __init__(self, O, W, H):
        assert O.is_sparse and O.is_coalesced() and O.dtype == torch.float32
        ObservedOracleEngine.received.append(O)
        M = torch.zeros(O.shape, dtype=torch.bool)
        M[O.indices()[0], O.indices()[1]] = True
        super().__init__(O.to_dense(), W, H, "nmf")
        self.M = M

    def set_mask(self, M):
        raise AssertionError("an observed-cell engine takes no dense mask")


def _module(W0, H0, trainable_W=True):
    from torchnmf_b200 import NMF
    m = NMF(W=W0, H=H0, trainable_W=trainable_W)
    m._engine_factory = ObservedOracleEngine
    return m


def _expected(Vd, Md):
    """The observed tensor for a dense view of the target and of the mask."""
    idx = Md.nonzero().t()
    return idx, Vd.float()[Md]


def _received_for(V, M, beta=1):
    c = tm.CASES["nmf_rand30_b1"]
    ObservedOracleEngine.received.clear()
    _module(c["W0"][: V.shape[1]].contiguous(), c["H0"][: V.shape[0]].contiguous()).fit(V, beta, max_iter=1, mask=M)
    return ObservedOracleEngine.received[0]


def _check_observed(O, idx, vals):
    assert O.is_coalesced() and O.dtype == torch.float32
    assert torch.equal(O.indices(), idx)
    assert torch.equal(O.values(), vals)


# ---- extraction ------------------------------------------------------------------------------------------------------
def test_extraction_from_dense_targets_of_every_form():
    c = tm.CASES["nmf_rand30_b1"]
    M = c["M"]
    V = torch.nan_to_num(c["V"], nan=0.5)
    idx, vals = _expected(V, M)
    _check_observed(_received_for(V, M.to_sparse()), idx, vals)
    Vb = V.bfloat16()
    _check_observed(_received_for(Vb, M.to_sparse()), *_expected(Vb, M))
    Vd = V.double()
    _check_observed(_received_for(Vd, M.to_sparse()), idx, vals)
    wide = torch.full((V.shape[0], V.shape[1] + 13), float("nan"))
    wide[:, : V.shape[1]] = V
    Vs = wide[:, : V.shape[1]]                                        # row-strided view, NaN beyond
    assert not Vs.is_contiguous()
    _check_observed(_received_for(Vs, M.to_sparse()), idx, vals)


def test_extraction_from_a_sparse_target_keeps_observed_zeros_and_drops_entries_outside():
    c = OBS["obs_b1"]
    Vs, M = sparse_target(c), c["M"]
    assert bool((M & ~c["S"]).any()) and bool((c["S"] & ~M).any())
    O = _received_for(Vs, M.to_sparse())
    idx, vals = _expected(Vs.to_dense(), M)
    _check_observed(O, idx, vals)
    assert int((O.values() == 0).sum()) == int((M & ~c["S"]).sum())   # observed unstored cells: explicit zeros


def test_extraction_of_uncoalesced_masks_with_duplicates_and_false_entries():
    c = tm.CASES["nmf_rand30_b1"]
    M = c["M"]
    V = torch.nan_to_num(c["V"])
    idx = M.nonzero().t()
    miss = (~M).nonzero().t()[:, :40]
    all_idx = torch.cat([idx.flip(1), idx[:, :25], miss, idx[:, 5:9]], 1)          # out of order, duplicates, False cells
    all_val = torch.cat([torch.ones(idx.shape[1] + 25, dtype=torch.bool), torch.zeros(40, dtype=torch.bool),
                         torch.zeros(4, dtype=torch.bool)])
    Mu = torch.sparse_coo_tensor(all_idx, all_val, M.shape)
    assert not Mu.is_coalesced()
    _check_observed(_received_for(V, Mu), *_expected(V, M))


# ---- validation --------------------------------------------------------------------------------------------------------
def test_refusals_leave_the_factors_untouched():
    from torchnmf_b200 import NMF2D, NMF3D, NMFD
    c = OBS["obs_b1"]
    Vs, M = sparse_target(c), c["M"]
    Ms = M.to_sparse()
    m = _module(c["W0"], c["H0"])
    Vn = Vs.to_dense()
    Vn[M.nonzero()[0][0], M.nonzero()[0][1]] = -1.0
    with pytest.raises(AssertionError, match="non-negative"):
        m.fit(Vn, 1, mask=Ms)
    with pytest.raises(AssertionError, match="non-negative"):
        m.fit(Vn.to_sparse(), 1, mask=Ms)
    with pytest.raises(ValueError, match="beta <= 0"):                  # an observed unstored cell is an observed zero
        m.fit(Vs, 0, mask=Ms)
    with pytest.raises(ValueError, match="no cell"):
        m.fit(Vs, 1, mask=torch.zeros_like(M).to_sparse())
    with pytest.raises(ValueError, match="no cell"):
        m.fit(Vs, 1, mask=torch.sparse_coo_tensor(M.nonzero().t(), torch.zeros(int(M.sum()), dtype=torch.bool), M.shape))
    for prec in ("f16", "f16_split"):
        with pytest.raises(ValueError, match="fp32 kernels"):
            m.fit(Vs, 1, precision=prec, mask=Ms)
    with pytest.raises(ValueError, match="torch.bool"):
        m.fit(Vs, 1, mask=Ms.float())
    with pytest.raises(ValueError, match="shape"):
        m.fit(Vs, 1, mask=M[:, :-1].to_sparse())
    assert torch.equal(m.W.data, c["W0"]) and torch.equal(m.H.data, c["H0"])
    for mc in tm.CASES.values():
        if mc["kind"] == "nmf":
            continue
        cls = {"nmfd": NMFD, "nmf2d": NMF2D, "nmf3d": NMF3D}[mc["kind"]]
        d = cls(W=mc["W0"], H=mc["H0"])
        d._engine_factory = tm.MaskedOracleEngine.factory(mc["kind"])
        with pytest.raises(ValueError, match="NMF only"):
            d.fit(mc["V"], mask=mc["M"].to_sparse())
        assert torch.equal(d.W.data, mc["W0"]) and torch.equal(d.H.data, mc["H0"])


def test_unobserved_garbage_is_accepted_and_changes_nothing():
    c = tm.CASES["nmf_rand30_b0"]                      # beta 0: no zero among the observed cells
    M = c["M"]
    out = []
    for fill in (0.0, float("nan"), float("inf"), -3.0):
        m = _module(c["W0"], c["H0"])
        m.fit(c["V"].masked_fill(~M, fill), 0, float("-inf"), 10, mask=M.to_sparse())
        out.append((m.W.data.clone(), m.H.data.clone()))
    for W, H in out[1:]:
        assert torch.equal(W, out[0][0]) and torch.equal(H, out[0][1])
    # a sparse target whose entries outside the mask are negative or zero, at beta 0
    Vd = torch.nan_to_num(c["V"]).masked_fill(~M, -2.0)
    Vd[~M & (torch.arange(M.shape[1]) % 2 == 0)] = 0.0
    m = _module(c["W0"], c["H0"])
    m.fit(Vd.to_sparse(), 0, float("-inf"), 10, mask=M.to_sparse())
    assert torch.equal(m.W.data, out[0][0]) and torch.equal(m.H.data, out[0][1])


# ---- fits against the reference ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", NMF_MASKED)
def test_sparse_mask_matches_reference_masked(name):
    c = tm.CASES[name]
    torch.set_num_threads(1)
    m = _module(c["W0"], c["H0"], bool(c["trainable_W"]))
    n_iter = m.fit(c["V"], c["beta"], c["tol"], c["max_iter"], False, c["alpha"], c["l1_ratio"], mask=c["M"].to_sparse())
    assert n_iter == c["n_iter"]
    assert torch.allclose(m.W.data, c["W"], rtol=2e-5, atol=1e-7)
    assert torch.allclose(m.H.data, c["H"], rtol=2e-5, atol=1e-7)
    assert m.last_fit_precision == "f32"


@pytest.mark.parametrize("name", sorted(OBS))
def test_sparse_target_and_mask_match_reference_observed(name):
    c = OBS[name]
    torch.set_num_threads(1)
    m = _module(c["W0"], c["H0"], bool(c["trainable_W"]))
    n_iter = m.fit(sparse_target(c), c["beta"], c["tol"], c["max_iter"], False, c["alpha"], c["l1_ratio"],
                   mask=c["M"].to_sparse())
    assert n_iter == c["n_iter"]
    assert torch.allclose(m.W.data, c["W"], rtol=2e-5, atol=1e-7), (m.W.data - c["W"]).abs().max()
    assert torch.allclose(m.H.data, c["H"], rtol=2e-5, atol=1e-7), (m.H.data - c["H"]).abs().max()
    if not c["trainable_W"]:
        assert torch.equal(m.W.data, c["W0"])


@pytest.mark.parametrize("name", sorted(OBS))
def test_observed_oracle_matches_reference_observed(name):
    c = OBS[name]
    torch.set_num_threads(1)
    W, H, n_iter, losses = mo.fit(sparse_target(c).to_dense(), c["W0"], c["H0"], c["M"], beta=c["beta"], tol=c["tol"],
                                  max_iter=c["max_iter"], alpha=c["alpha"], l1_ratio=c["l1_ratio"],
                                  trainable_W=bool(c["trainable_W"]))
    assert n_iter == c["n_iter"]
    assert torch.allclose(W, c["W"], rtol=2e-5, atol=1e-7) and torch.allclose(H, c["H"], rtol=2e-5, atol=1e-7)
    for a, b in zip(losses, c["losses"]):
        assert math.isclose(a, b, rel_tol=1e-4, abs_tol=1e-6)


def test_fixtures_cover_the_contract():
    betas = {c["beta"] for c in OBS.values()}
    assert {1, 0.5, 2} <= betas
    assert any(c["alpha"] > 0 for c in OBS.values())
    assert any(not c["trainable_W"] for c in OBS.values())
    for c in OBS.values():
        S, M = c["S"], c["M"]
        assert bool((M & ~S).any())                                   # observed cells the target does not store
        assert bool((S & ~M).any())                                   # stored entries outside the mask
        assert (~M).all(1).any() and (~M).all(0).any()               # an empty row and an empty column of the mask
        assert bool(((~S).all(1) & M.any(1)).any()) and bool(((~S).all(0) & M.any(0)).any())
        assert torch.equal(c["V"][~S], torch.zeros(int((~S).sum())))


def test_set_target_observed_is_bound_and_refuses_a_null_context():
    from torchnmf_b200 import _capi
    res, args = _capi.SIGNATURES["nmfb200_nmf_set_target_observed"]
    assert res is ctypes.c_int and args == [ctypes.c_void_p, ctypes.c_int64] + [ctypes.c_void_p] * 7
    lib = _capi.load()
    assert lib.nmfb200_nmf_set_target_observed(None, 0, None, None, None, None, None, None, None) == 1
    assert b"null context" in lib.nmfb200_last_error()
    header = " ".join(open(os.path.join(ROOT, "include", "nmf_b200.h")).read().split())
    assert ("int nmfb200_nmf_set_target_observed(nmfb200_ctx* ctx, int64_t nnz, const int64_t* crow, const int64_t* col, "
            "const float* val, const int64_t* ccol, const int64_t* row, const float* val_t, void* stream);") in header


# ---- the sharded protocol (gloo, two CPU processes): each rank passes the row shards of V and of the mask ----------------
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
    import test_observed as to
    c = to.OBS[name]
    n = c["V"].shape[0]
    bounds = [0, (2 * n) // 3, n]                     # uneven row shards
    lo, hi = bounds[rank], bounds[rank + 1]
    m = to._module(c["W0"], c["H0"][lo:hi], bool(c["trainable_W"]))
    Vs = to.sparse_target(c).to_dense()[lo:hi].to_sparse()
    n_iter = m.fit(Vs, c["beta"], c["tol"], c["max_iter"], False, c["alpha"], c["l1_ratio"], group=dist.group.WORLD,
                   mask=c["M"][lo:hi].to_sparse())
    torch.save({"W": m.W.data, "H": m.H.data, "n_iter": n_iter}, os.path.join(out_dir, f"rank{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("name", ["obs_b1", "obs_b0.5"])
def test_sharded_observed_fit_equals_single(tmp_path, name):
    world = 2
    mp.spawn(_worker, args=(world, _free_port(), name, str(tmp_path)), nprocs=world, join=True)
    c = OBS[name]
    ref = _module(c["W0"], c["H0"], bool(c["trainable_W"]))
    n_ref = ref.fit(sparse_target(c), c["beta"], c["tol"], c["max_iter"], False, c["alpha"], c["l1_ratio"],
                    mask=c["M"].to_sparse())
    parts = [torch.load(os.path.join(tmp_path, f"rank{r}.pt")) for r in range(world)]
    assert all(p["n_iter"] == n_ref for p in parts)
    assert torch.equal(parts[0]["W"], parts[1]["W"])                      # the W replicas stay bit-identical
    assert torch.allclose(parts[0]["W"], ref.W.data, rtol=1e-4, atol=1e-7)
    assert torch.allclose(torch.cat([p["H"] for p in parts]), ref.H.data, rtol=1e-4, atol=1e-7)
