"""PLCA / SIPLCA / SIPLCA2 / SIPLCA3 fits on partially observed targets, `fit(V, ..., mask=M)`, on the CPU (no GPU): the
oracle (tests/masked_plca_oracle.py) against the reference's fixtures (tests/golden/reference_masked_plca.npz, written by
tools/make_golden_masked_plca.py), the oracle's EM properties, and every refusal of the masked fit, which all come before
the fit looks for a device.
"""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from masked_plca_oracle import fit_masked, log_likelihood
from oracle import plca_oracle as po
from torchnmf_b200 import PLCA, SIPLCA, SIPLCA2, SIPLCA3, BatchedPLCA, BatchedSIPLCA

Z_ = np.load(os.path.join(GOLDEN, "reference_masked_plca.npz"), allow_pickle=False)
NAMES = sorted({k.split("/")[0] for k in Z_.files})
CLS = {0: PLCA, 1: SIPLCA, 2: SIPLCA2, 3: SIPLCA3}


def case(name):
    c = {k.split("/", 1)[1]: Z_[k] for k in Z_.files if k.startswith(name + "/")}
    for k in ("V", "M", "W0", "H0", "Z0", "W", "H", "Z"):
        c[k] = torch.from_numpy(c[k].copy())
    return c


def alphas(c):
    a = tuple(float(c[k]) for k in ("W_alpha", "H_alpha", "Z_alpha"))
    return tuple(torch.tensor(x, dtype=torch.float64) for x in a) if int(c["tensor_alpha"]) else a


def normalised64(c):
    """W0, H0, Z0 in float64, normalised as the modules' constructors normalise them (plca.py:110-144)."""
    W, H, Z = c["W0"].double(), c["H0"].double(), c["Z0"].double()
    return W / po.get_norm(W), H / po.get_norm(H), Z / Z.sum()


def trainables(c):
    return tuple(bool(int(c[k])) for k in ("trainable_W", "trainable_H", "trainable_Z"))


# ---- the oracle is pinned by the reference's outputs -----------------------------------------------------------------------
def test_fixture_covers_the_cases():
    assert {"plca_rand30", "plca_gap", "plca_frozenW", "plca_alpha", "plca_alpha_tensor", "plca_tol", "plca_all",
            "plca_nan", "plca_r300", "siplca_rand30", "siplca2_rand30", "siplca3_rand30"} <= set(NAMES)
    assert int(case("plca_tol")["n_iter"]) < int(case("plca_tol")["iters"]) - 1          # a finite-tol stop
    assert bool(case("plca_all")["M"].all())
    c = case("plca_nan")
    assert torch.isnan(c["V"][~c["M"]]).all() and not torch.isnan(c["V"][c["M"]]).any()
    assert case("plca_r300")["W"].shape[1] == 300
    gap = case("plca_gap")["M"]
    assert not gap[:, 30:46].any()


@pytest.mark.parametrize("name", NAMES)
def test_oracle_matches_reference(name):
    c = case(name)
    W0, H0, Z0 = normalised64(c)
    tol = float(c["tol"])
    W, H, Z, n_iter, norm, losses = fit_masked(c["V"].double(), c["M"], W0, H0, Z0, tol, int(c["iters"]), *alphas(c),
                                               *trainables(c))
    assert n_iter == int(c["n_iter"])
    assert abs(float(norm) - float(c["norm"])) <= 1e-10 * float(c["norm"])
    np.testing.assert_allclose(losses, c["losses"], rtol=1e-9)
    for nm, got in (("W", W), ("H", H), ("Z", Z)):
        want = c[nm]
        assert torch.allclose(got, want, rtol=1e-8, atol=1e-12 * float(want.abs().max())), (name, nm)


def test_frozen_factor_stays_as_given():
    c = case("plca_frozenW")
    W0, H0, Z0 = normalised64(c)
    W = fit_masked(c["V"].double(), c["M"], W0, H0, Z0, float("-inf"), 5, trainable_W=False)[0]
    assert torch.equal(W, W0)
    assert torch.allclose(c["W"], W0, rtol=1e-15, atol=0)


# ---- properties of the definition -------------------------------------------------------------------------------------------
def _random_problem(model, seed, missing):
    g = torch.Generator().manual_seed(seed)
    if model == "PLCA":
        V = torch.rand(40, 33, generator=g, dtype=torch.float64) * 3
        W, H = torch.rand(33, 5, generator=g, dtype=torch.float64), torch.rand(40, 5, generator=g, dtype=torch.float64)
    else:
        V = torch.rand(2, 7, 29, generator=g, dtype=torch.float64) * 3
        W = torch.rand(7, 4, 5, generator=g, dtype=torch.float64)
        H = torch.rand(2, 4, 25, generator=g, dtype=torch.float64)
    Z = torch.rand(W.shape[1], generator=g, dtype=torch.float64) + 0.1
    M = torch.rand(V.shape, generator=g, dtype=torch.float64) >= missing
    return V, M, W / po.get_norm(W), H / po.get_norm(H), Z / Z.sum()


@pytest.mark.parametrize("model", ["PLCA", "SIPLCA"])
def test_every_cell_observed_is_the_unmasked_fit(model):
    V, _, W0, H0, Z0 = _random_problem(model, 5, 0.0)
    M = torch.ones(V.shape, dtype=torch.bool)
    for kw in ({}, dict(W_alpha=1.05, H_alpha=1.02, Z_alpha=1.1), dict(trainable_Z=False)):
        W, H, Z, n_iter, norm, losses = fit_masked(V, M, W0, H0, Z0, 1e-4, 40, **kw)
        Wr, Hr, Zr, n_r, norm_r = po.fit(V, W0, H0, Z0, 1e-4, 40, **kw)
        assert n_iter == n_r
        assert abs(float(norm) - float(norm_r)) <= 1e-12 * float(norm_r)
        for got, want in ((W, Wr), (H, Hr), (Z, Zr)):
            assert torch.allclose(got, want, rtol=1e-12, atol=1e-12 * float(want.abs().max()))
        # the loss is the reference's: sqrt(2 kl_div(q norm, V)) at the initial factors
        assert abs(losses[0] - po._loss(po.reconstruct(H0, W0, Z0), V / V.sum(), V.sum())) <= 1e-10 * losses[0]


@pytest.mark.parametrize("model", ["PLCA", "SIPLCA"])
@pytest.mark.parametrize("seed,missing", [(11, 0.3), (12, 0.6), (13, 0.1)])
def test_em_never_decreases_the_observed_likelihood(model, seed, missing):
    V, M, W0, H0, Z0 = _random_problem(model, seed, missing)
    history = []
    fit_masked(V, M, W0, H0, Z0, float("-inf"), 25, eps=0.0, history=history)
    ll = [log_likelihood(V, M, W0, H0, Z0)] + [log_likelihood(V, M, *f) for f in history]
    for a, b in zip(ll, ll[1:]):
        assert b >= a - 1e-13 * abs(a), (a, b)
    assert ll[-1] > ll[0]


def test_zeroing_the_missing_cells_is_a_different_fit():
    """The naive treatment -- the missing cells as observed zeros -- is exactly the unmasked fit of V * M, and it moves
    the model's mass away from the missing cells; the EM keeps it there."""
    V, M, W0, H0, Z0 = _random_problem("PLCA", 21, 0.3)
    M[:, :8] = False
    W, H, Z = fit_masked(V, M, W0, H0, Z0, float("-inf"), 30)[:3]
    Wz, Hz, Zz = po.fit(V * M, W0, H0, Z0, float("-inf"), 30)[:3]
    assert float(po.reconstruct(H, W, Z)[:, :8].sum()) > 4 * float(po.reconstruct(Hz, Wz, Zz)[:, :8].sum())


# ---- refusals: before any device work, and nothing runs after one -----------------------------------------------------------
@pytest.fixture
def no_engine(monkeypatch):
    calls = []

    def engine(*a, **k):
        calls.append(a)
        raise AssertionError("an engine was opened after a refusal")

    for cls in (PLCA, SIPLCA):
        monkeypatch.setattr(cls, "_engine", staticmethod(engine))
    return calls


def _module():
    torch.manual_seed(0)
    return PLCA((6, 5), rank=2)


def _params(m):
    return [p.detach().clone() for p in (m.W, m.H, m.Z)]


@pytest.mark.parametrize("bad, match", [
    (lambda V: V > 0.5, None),                                                   # fine: reaches the device check
    (lambda V: (V > 0.5).to(torch.uint8), "torch.bool"),
    (lambda V: (V > 0.5).float(), "torch.bool"),
    (lambda V: (V > 0.5).numpy(), "torch.bool"),
    (lambda V: (V > 0.5).to_sparse(), "dense mask"),
    (lambda V: torch.ones(6, 4, dtype=torch.bool), "shape"),
    (lambda V: torch.ones(5, 6, dtype=torch.bool), "shape"),
    (lambda V: torch.zeros(6, 5, dtype=torch.bool), "no cell"),
])
def test_mask_refusals(bad, match, no_engine):
    m = _module()
    before = _params(m)
    V = torch.rand(6, 5)
    if match is None:
        if torch.cuda.is_available():
            pytest.skip("the valid mask case runs the fit on a GPU machine")
        with pytest.raises(RuntimeError, match="CUDA device"):
            m.fit(V, mask=bad(V))
    else:
        with pytest.raises(ValueError, match=match):
            m.fit(V, mask=bad(V))
    assert not no_engine
    for a, b in zip(before, _params(m)):
        assert torch.equal(a, b)


def test_target_and_precision_refusals(no_engine):
    m = _module()
    before = _params(m)
    V = torch.rand(6, 5)
    M = V > 0.3
    with pytest.raises(ValueError, match="dense target"):
        m.fit(V.to_sparse(), mask=M)
    for p in ("f16", "f16_split", "auto", "bf16"):
        with pytest.raises(ValueError, match="precision"):
            m.fit(V, mask=M, precision=p)
    with pytest.raises(ValueError, match="sum to 0"):
        m.fit(torch.where(M, torch.zeros(()), V), mask=M)
    Vneg = V.clone()
    Vneg[0, 0] = -1.0
    Mneg = M.clone()
    Mneg[0, 0] = True
    with pytest.raises(AssertionError, match="non-negative"):
        m.fit(Vneg, mask=Mneg)
    with pytest.raises(TypeError):
        m.fit(V, mask=M, weight=torch.ones(6, 5))
    assert not no_engine
    for a, b in zip(before, _params(m)):
        assert torch.equal(a, b)


def test_missing_cells_are_not_checked():
    """Negative or NaN values off O pass the checks (they are never read): the fit goes on to look for a device."""
    if torch.cuda.is_available():
        pytest.skip("the fit would run on a GPU machine")
    m = SIPLCA((1, 3, 12), rank=2, T=3)
    V = torch.rand(1, 3, 12)
    M = torch.ones_like(V, dtype=torch.bool)
    M[0, 1, 4:8] = False
    V[~M] = float("nan")
    V[0, 1, 4] = -5.0
    with pytest.raises(RuntimeError, match="CUDA device"):
        m.fit(V, mask=M)


def test_unmasked_fit_still_refuses_negative_targets():
    m = _module()
    V = torch.rand(6, 5)
    V[1, 1] = -1
    with pytest.raises(AssertionError, match="non-negative"):
        m.fit(V)


@pytest.mark.parametrize("cls, shape, kw", [(BatchedPLCA, (2, 6, 5), {}), (BatchedSIPLCA, (2, 1, 3, 12), {"T": 3})])
def test_batched_fits_still_take_no_mask(cls, shape, kw):
    m = cls(shape, rank=2, **kw)
    V = torch.rand(*shape)
    with pytest.raises(TypeError):
        m.fit(V, mask=torch.ones(shape, dtype=torch.bool))
