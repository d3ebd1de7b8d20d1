"""PLCA fits of sparse COO targets, `PLCA.fit(V)` with V sparse (PLSA on a count matrix), on the CPU (no GPU): the host
logic of the fit through the `_engine_factory` hook with a float64 oracle of the sparse engine, against the reference's
fixtures (tests/golden/reference_sparse_plca.npz, written by tools/make_golden_sparse_plca.py from `PLCA.fit(V.to_dense())`);
the target's dtypes, placement and duplicates; the permutation between the two compressed forms; and every refusal, which
all come before the fit looks for a device.
"""
import math
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import plca_oracle as po
from torchnmf_b200 import PLCA, SIPLCA, SIPLCA2, SIPLCA3
from torchnmf_b200 import engine as _engine
from torchnmf_b200.constants import eps

Z_ = np.load(os.path.join(GOLDEN, "reference_sparse_plca.npz"), allow_pickle=False)
NAMES = sorted({k.split("/")[0] for k in Z_.files})


def case(name):
    c = {k.split("/", 1)[1]: Z_[k] for k in Z_.files if k.startswith(name + "/")}
    for k in ("rows", "cols", "vals", "W0", "H0", "Z0", "W", "H", "Z"):
        c[k] = torch.from_numpy(c[k].copy())
    c["rows"], c["cols"] = c["rows"].long(), c["cols"].long()
    return c


def sparse_target(c, dtype=torch.float64):
    return torch.sparse_coo_tensor(torch.stack([c["rows"], c["cols"]]), c["vals"].to(dtype),
                                   (int(c["N"]), int(c["C"]))).coalesce()


def alphas(c):
    a = tuple(float(c[k]) for k in ("W_alpha", "H_alpha", "Z_alpha"))
    return tuple(torch.tensor(x, dtype=torch.float64) for x in a) if int(c["tensor_alpha"]) else a


def module64(c):
    """A float64 PLCA module holding W0, H0, Z0 normalised in float64, as the reference's float64 modules hold them."""
    W, H, Z = c["W0"].double(), c["H0"].double(), c["Z0"].double()
    m = PLCA(W=W, H=H, Z=Z, **{k: bool(int(c[k])) for k in ("trainable_W", "trainable_H", "trainable_Z")}).double()
    for p, x in ((m.W, W / po.get_norm(W)), (m.H, H / po.get_norm(H)), (m.Z, Z / Z.sum())):
        p.data.copy_(x)
    return m


class OracleSparsePlcaEngine:
    """The sparse PLCA engine's interface (engine.CudaSparsePlcaEngine) in the factors' dtype on the CPU: the gradients from
    the densified target, the loss from its definition at the stored entries and the column sums."""
    precision = "oracle"

    def __init__(self, Vn, W, Hz):
        assert Vn.is_sparse and Vn.is_coalesced() and Vn.dtype == W.dtype
        self.Vn, self.W, self.H = Vn, W, Hz
        self.dense = Vn.to_dense()

    def plca_terms(self, Hz, norm=None):
        P = self.dense / (Hz @ self.W.t() + eps)
        return P.t() @ Hz, P @ self.W

    def loss(self, norm):
        (n, c), t = self.Vn.indices(), self.Vn.values() * norm
        x = norm * (self.H[n] * self.W[c]).sum(1)
        return float((t * (torch.log(t + eps) - torch.log(x + eps))).sum() - t.sum()
                     + norm * (self.W.sum(0) @ self.H.sum(0)))

    def precision_for(self, beta):
        return self.precision

    def check_health(self):
        pass

    def close(self):
        pass


def fit64(c, V=None, iters=None):
    m = module64(c)
    m._engine_factory = OracleSparsePlcaEngine
    n_iter, norm = m.fit(sparse_target(c) if V is None else V, float(c["tol"]),
                         int(c["iters"]) if iters is None else iters, False, *alphas(c))
    return m, n_iter, norm


def test_fixture_covers_the_cases():
    assert {"poisson", "empty", "frozenW", "alpha", "alpha_tensor", "tol", "r300"} <= set(NAMES)
    assert int(case("tol")["n_iter"]) < int(case("tol")["iters"]) - 1                  # a finite-tol stop
    e = case("empty")
    assert (e["vals"] == 0).any() and not bool(((e["rows"] < 20) | (e["cols"] < 15)).any())
    assert case("r300")["W"].shape[1] == 300


@pytest.mark.parametrize("name", NAMES)
def test_fit_matches_reference(name):
    c = case(name)
    m, n_iter, norm = fit64(c)
    assert m.last_fit_precision == "oracle"
    assert n_iter == int(c["n_iter"])
    assert norm.dtype == torch.float64 and abs(float(norm) - float(c["norm"])) <= 1e-6 * float(c["norm"])
    for nm in ("W", "H", "Z"):
        got, want = getattr(m, nm).data, c[nm]
        assert torch.allclose(got, want, rtol=1e-6, atol=1e-12 * float(want.abs().max())), (name, nm)


def test_frozen_factor_stays_as_given():
    c = case("frozenW")
    W0 = module64(c).W.data.clone()
    m, _, _ = fit64(c, iters=5)
    assert torch.equal(m.W.data, W0)


def test_loss_is_the_dense_kl():
    """The oracle engine's sparse loss is the dense fit's _kl(norm q, norm Vn), empty cells included."""
    c = case("empty")
    m = module64(c)
    V = sparse_target(c)
    norm = float(V.values().sum())
    Vn = torch.sparse_coo_tensor(V.indices(), V.values() / norm, V.shape).coalesce()
    Hz = m.H.data * m.Z.data
    eng = OracleSparsePlcaEngine(Vn, m.W.data, Hz)
    q = Hz @ m.W.data.t()
    want = po._loss(q, Vn.to_dense(), norm)
    assert math.isclose(math.sqrt(2 * eng.loss(norm)), want, rel_tol=1e-12)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float32])
def test_target_dtypes(dtype):
    """Small counts are exact in every floating dtype, and the EM step does not see the target's scale: the fit is the
    float64 target's.  norm is V.sum() in V's dtype."""
    c = case("poisson")
    m, n_iter, norm = fit64(c, sparse_target(c, dtype), iters=20)
    m64, n64, _ = fit64(c, iters=20)
    assert norm.dtype == dtype and float(norm) == float(sparse_target(c, dtype).to_dense().sum())
    assert n_iter == n64
    for nm in ("W", "H", "Z"):
        want = getattr(m64, nm).data
        assert torch.allclose(getattr(m, nm).data, want, rtol=1e-9, atol=1e-15 * float(want.abs().max())), nm


def test_uncoalesced_target_sums_its_duplicates():
    c = case("empty")
    V = sparse_target(c)
    idx, vals = V.indices(), V.values()
    U = torch.sparse_coo_tensor(torch.cat([idx, idx], 1).flip(1), torch.cat([vals / 2, vals / 2]).flip(0), V.shape)
    assert not U.is_coalesced()
    m, n_iter, norm = fit64(c, U, iters=20)
    m64, n64, norm64 = fit64(c, iters=20)
    assert n_iter == n64 and float(norm) == float(norm64)
    for nm in ("W", "H", "Z"):
        assert torch.equal(getattr(m, nm).data, getattr(m64, nm).data), nm


def test_compressed_forms_order_links_csc_to_csr():
    c = case("empty")
    V = sparse_target(c, torch.float32)
    crow, col, val, ccol, row, val_t, perm = _engine._compressed_forms(V, with_order=True)
    assert torch.equal(val[perm], val_t) and torch.equal(col[perm], torch.repeat_interleave(
        torch.arange(V.shape[1]), ccol.diff()))
    rows_csr = torch.repeat_interleave(torch.arange(V.shape[0]), crow.diff())
    assert torch.equal(rows_csr[perm], row)
    for a, b in zip(_engine._compressed_forms(V), (crow, col, val, ccol, row, val_t)):
        assert torch.equal(a, b)


# ---- refusals: before any device work, and nothing runs after one ----------------------------------------------------------
@pytest.fixture
def no_engine(monkeypatch):
    calls = []

    def engine(*a, **k):
        calls.append(a)
        raise AssertionError("an engine was opened after a refusal")

    monkeypatch.setattr(_engine, "CudaSparsePlcaEngine", engine)
    for cls in (PLCA, SIPLCA, SIPLCA2, SIPLCA3):
        monkeypatch.setattr(cls, "_engine", staticmethod(engine))
    return calls


def _module():
    torch.manual_seed(0)
    return PLCA((6, 5), rank=2)


def _params(m):
    return [p.detach().clone() for p in (m.W, m.H, m.Z)]


def _sparse(dense):
    return dense.to_sparse()


@pytest.mark.parametrize("make, exc, match", [
    (lambda: _sparse(torch.tensor([[1., 0, 0, 0, 0]] * 5 + [[0, 0, -1., 0, 0]])), AssertionError, "non-negative"),
    (lambda: torch.sparse_coo_tensor(torch.zeros(2, 0, dtype=torch.int64), torch.zeros(0), (6, 5)), ValueError, "no entry"),
    (lambda: torch.sparse_coo_tensor(torch.tensor([[0, 3], [1, 2]]), torch.zeros(2), (6, 5)), ValueError, "sum to 0"),
    (lambda: torch.rand(6, 5).to_sparse_csr(), ValueError, "COO"),
    (lambda: torch.rand(5, 6).to_sparse(), ValueError, "shape"),
])
def test_target_refusals(make, exc, match, no_engine):
    m = _module()
    before = _params(m)
    with pytest.raises(exc, match=match):
        m.fit(make())
    assert not no_engine
    for a, b in zip(before, _params(m)):
        assert torch.equal(a, b)


@pytest.mark.parametrize("precision", ["f16", "f16_split", "auto", "bf16"])
def test_precision_refusals(precision, no_engine):
    m = _module()
    with pytest.raises(ValueError, match="precision"):
        m.fit(torch.rand(6, 5).to_sparse(), precision=precision)
    assert not no_engine


def test_valid_target_reaches_the_device_check(no_engine):
    if torch.cuda.is_available():
        pytest.skip("the fit would run on a GPU machine")
    m = _module()
    V = torch.rand(6, 5).to_sparse()
    with pytest.raises(RuntimeError, match="CUDA device"):
        m.fit(V)
    assert not no_engine


def test_mask_with_a_sparse_target_is_still_refused(no_engine):
    m = _module()
    V = torch.rand(6, 5)
    with pytest.raises(ValueError, match="dense target"):
        m.fit(V.to_sparse(), mask=V > 0.3)
    assert not no_engine


@pytest.mark.parametrize("cls, shape, kw", [(SIPLCA, (1, 3, 12), {"T": 3}), (SIPLCA2, (1, 2, 6, 7), {"kernel_size": 2}),
                                            (SIPLCA3, (1, 2, 4, 5, 6), {"kernel_size": 2})])
def test_shift_invariant_models_refuse_sparse_targets(cls, shape, kw, no_engine):
    m = cls(shape, rank=2, **kw)
    with pytest.raises(NotImplementedError, match="dense targets"):
        m.fit(torch.rand(*shape).to_sparse())
    assert not no_engine
