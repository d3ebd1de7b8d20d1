"""Fixed components of W (`fit(V, ..., fixed_W=F)`), without a GPU.

The host logic runs through oracle engines plugged in with the `_engine_factory` hook: the refusals before any engine is
built, the plain fit when no component is fixed, the frozen-W fit when every component is, and a partial fit against float64
oracles in which the multiplicative updates and the EM step update the free columns only and coordinate descent skips the
fixed k inside the sweep.
"""
import pytest
import torch

import cd_oracle as cdo
from masked_plca_oracle import em_step
from oracle import mu_oracle as orc
from oracle import plca_oracle as po
from oracle_engine import OracleNmfdEngine, OracleNmfEngine, OracleNmfndEngine
from test_plca import PlcaOracleEngine, SiplcaOracleEngine
from test_sparse_plca import OracleSparsePlcaEngine
from torchnmf_b200 import (NMF, NMF2D, NMF3D, NMFD, PLCA, SIPLCA, BatchedNMF, BatchedPLCA)


class _Fixing:
    """An oracle engine that honours set_fixed_w as the C ABI does: a W update leaves the fixed columns as they were.  For
    the multiplicative updates (element-wise in W) that is the update of the free columns only.  Logs every call."""
    log = None

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.fixed = None
        self.calls = _Fixing.log if _Fixing.log is not None else []

    def set_fixed_w(self, fixed):
        assert fixed is None or (fixed.dtype == torch.uint8 and fixed.numel() == self.W.shape[1])
        self.calls.append(("set_fixed_w", None if fixed is None else fixed.tolist()))
        self.fixed = None if fixed is None else fixed.bool()

    def update_w(self, *a):
        self.calls.append(("update_w",) + a)
        keep = self.W[:, self.fixed].clone() if self.fixed is not None else None
        super().update_w(*a)
        if keep is not None:
            self.W[:, self.fixed] = keep

    def update_h(self, *a):
        self.calls.append(("update_h",) + a)
        super().update_h(*a)


class FixNmf(_Fixing, OracleNmfEngine):
    def cd_update(self, which, l1, l2):
        self.calls.append(("cd_update", which, l1, l2))
        if which == 0:
            self.W.copy_(skip_sweep(self.V, self.W, self.H, l1, l2, self.fixed))
        else:
            self.H.copy_(cdo.update(self.V, self.W, self.H, 1, l1, l2))


class FixNmfd(_Fixing, OracleNmfdEngine):
    pass


class FixNmfnd(_Fixing, OracleNmfndEngine):
    pass


class NoEngine:
    def __init__(self, *a, **k):
        raise AssertionError("an engine was built")


def skip_sweep(V, W, H, l1=0.0, l2=0.0, fixed=None):
    """One HALS update of W (float64) that skips each fixed column k inside the sweep: later columns see its value."""
    A, B = cdo.terms(V, W, H, 0)
    X = W.double().clone()
    for k in range(X.shape[1]):
        hess = float(B[k, k]) + l2
        if hess != 0.0 and not (fixed is not None and bool(fixed[k])):
            X[:, k] = (X[:, k] + (A[:, k] - X @ B[:, k] - l1 - l2 * X[:, k]) / hess).clamp_min(0.0)
    return X


def restore_sweep(V, W, H, l1=0.0, l2=0.0, fixed=None):
    """The wrong semantics: the plain sweep, then the fixed columns put back."""
    X = cdo.update(V, W, H, 0, l1, l2)
    if fixed is not None:
        X[:, fixed] = W.double()[:, fixed]
    return X


def _nmf_problem(seed=0, N=23, C=17, R=5):
    g = torch.Generator().manual_seed(seed)
    V = torch.rand(N, R, generator=g, dtype=torch.float64) @ torch.rand(R, C, generator=g, dtype=torch.float64)
    V += 0.05 * torch.rand(N, C, generator=g, dtype=torch.float64)
    W, H = torch.rand(C, R, generator=g) + 0.1, torch.rand(N, R, generator=g) + 0.1
    return V, W.double(), H.double()        # fp32 values: the modules store them exactly


def _module(cls, W, H, engine, **kw):
    m = cls(W=W.clone(), H=H.clone(), **kw).double()
    m._engine_factory = engine
    return m


# ---- refusals ---------------------------------------------------------------------------------------------------------

def _nmf_like():
    V, W, H = _nmf_problem()
    yield NMF, V, W, H, {}
    g = torch.Generator().manual_seed(1)
    yield NMFD, torch.rand(2, 6, 12, generator=g), torch.rand(6, 5, 3, generator=g), torch.rand(2, 5, 10, generator=g), {}
    yield NMF2D, torch.rand(1, 4, 6, 7, generator=g), torch.rand(4, 5, 2, 2, generator=g), torch.rand(1, 5, 5, 6, generator=g), {}
    yield (NMF3D, torch.rand(1, 3, 4, 5, 6, generator=g), torch.rand(3, 5, 2, 2, 2, generator=g),
           torch.rand(1, 5, 3, 4, 5, generator=g), {})


@pytest.mark.parametrize("case", range(4))
@pytest.mark.parametrize("bad", ["int", "float", "short", "long", "2d", "sparse", "list"])
def test_bad_fixed_w_is_refused_before_any_engine(case, bad):
    cls, V, W, H, _ = list(_nmf_like())[case]
    R = W.shape[1]
    F = {"int": torch.zeros(R, dtype=torch.int64), "float": torch.zeros(R), "short": torch.zeros(R - 1, dtype=torch.bool),
         "long": torch.zeros(R + 1, dtype=torch.bool), "2d": torch.zeros(1, R, dtype=torch.bool),
         "sparse": torch.zeros(R, dtype=torch.bool).to_sparse(), "list": [False] * R}[bad]
    m = _module(cls, W, H, NoEngine)
    with pytest.raises(ValueError, match="fixed_W"):
        m.fit(V, 1, 1e-4, 5, fixed_W=F)


@pytest.mark.parametrize("case", range(4))
def test_fixed_w_with_frozen_w_or_group_is_refused(case):
    cls, V, W, H, _ = list(_nmf_like())[case]
    F = torch.zeros(W.shape[1], dtype=torch.bool)
    F[0] = True
    m = _module(cls, W, H, NoEngine, trainable_W=False)
    with pytest.raises(ValueError, match="not trainable"):
        m.fit(V, 1, 1e-4, 5, fixed_W=F)
    m = _module(cls, W, H, NoEngine)
    with pytest.raises(ValueError, match="group"):
        m.fit(V, 1, 1e-4, 5, group=object(), fixed_W=F)


def _plca_problem(cls, seed=0):
    """A target and a module in fp32, as the dense PLCA fits stage them."""
    g = torch.Generator().manual_seed(seed)
    if cls is PLCA:
        V = torch.rand(13, 9, generator=g)
        m = PLCA(W=torch.rand(9, 4, generator=g), H=torch.rand(13, 4, generator=g), Z=torch.rand(4, generator=g))
    else:
        V = torch.rand(2, 6, 14, generator=g)
        m = SIPLCA(W=torch.rand(6, 4, 3, generator=g), H=torch.rand(2, 4, 12, generator=g), Z=torch.rand(4, generator=g))
    return V, m


@pytest.mark.parametrize("cls", [PLCA, SIPLCA])
def test_plca_refusals_before_any_engine(cls):
    V, m = _plca_problem(cls)
    m._engine_factory = NoEngine
    for F in (torch.zeros(4), torch.zeros(3, dtype=torch.bool), torch.zeros(5, dtype=torch.bool)):
        with pytest.raises(ValueError, match="fixed_W"):
            m.fit(V, fixed_W=F)
    F = torch.tensor([True, False, False, False])
    with pytest.raises(ValueError, match="group"):
        m.fit(V, group=object(), fixed_W=F)
    m.W.requires_grad_(False)
    with pytest.raises(ValueError, match="not trainable"):
        m.fit(V, fixed_W=F)
    if cls is PLCA:          # a masked or sparse target is refused the same way, before its own checks
        m.W.requires_grad_(True)
        with pytest.raises(ValueError, match="fixed_W"):
            m.fit(V, mask=torch.ones(V.shape, dtype=torch.bool), fixed_W=torch.zeros(4))
        with pytest.raises(ValueError, match="fixed_W"):
            m.fit(V.to_sparse(), fixed_W=torch.zeros(4))


def test_sparse_fit_and_batched_fits_take_no_fixed_w():
    V, W, H = _nmf_problem()
    F = torch.zeros(W.shape[1], dtype=torch.bool)
    with pytest.raises(TypeError):
        NMF(W=W, H=H).sparse_fit(V, fixed_W=F)
    with pytest.raises(TypeError):
        BatchedNMF(W=W[None].float(), H=H[None].float()).fit(V[None].float(), fixed_W=F)
    with pytest.raises(TypeError):
        BatchedPLCA(W=W[None].float(), H=H[None].float(), Z=torch.ones(1, W.shape[1])).fit(V[None].float(), fixed_W=F)


# ---- none fixed, all fixed ---------------------------------------------------------------------------------------------

ENGINES = {NMF: FixNmf, NMFD: FixNmfd, NMF2D: FixNmfnd, NMF3D: FixNmfnd}


@pytest.mark.parametrize("case", range(4))
@pytest.mark.parametrize("beta", [1, 2])
def test_none_fixed_is_the_plain_fit_and_all_fixed_is_frozen_w(case, beta):
    cls, V, W, H, _ = list(_nmf_like())[case]
    V = V.double()
    R = W.shape[1]
    runs = {}
    for name, F, kw in (("plain", None, {}), ("none", torch.zeros(R, dtype=torch.bool), {}),
                        ("frozen", None, {"trainable_W": False}), ("all", torch.ones(R, dtype=torch.bool), {})):
        _Fixing.log = []
        m = _module(cls, W, H, ENGINES[cls], **kw)
        extra = {} if F is None else {"fixed_W": F}
        n = m.fit(V, beta, -1.0, 23, alpha=0.1, l1_ratio=0.5, **extra)
        runs[name] = (n, m.W.data.clone(), m.H.data.clone(), list(_Fixing.log))
    _Fixing.log = None
    for a, b in (("plain", "none"), ("frozen", "all")):
        assert runs[a][0] == runs[b][0]
        assert torch.equal(runs[a][1], runs[b][1]) and torch.equal(runs[a][2], runs[b][2]), (a, b)
        assert runs[a][3] == runs[b][3], (a, b)       # the same engine calls: nothing passed down
    assert torch.equal(runs["all"][1], W.double())
    assert not any(c[0] == "set_fixed_w" for c in runs["none"][3] + runs["all"][3])


# ---- partial fits against float64 oracles ------------------------------------------------------------------------------

FIXED_SETS = {"first": [0, 1], "last": [3, 4], "scattered": [0, 2, 4]}


def _flags(R, idx):
    F = torch.zeros(R, dtype=torch.bool)
    F[idx] = True
    return F


@pytest.mark.parametrize("which", list(FIXED_SETS))
@pytest.mark.parametrize("beta", [0.5, 1, 2])
def test_partial_mu_matches_free_column_oracle(which, beta):
    V, W, H = _nmf_problem(3)
    F = _flags(W.shape[1], FIXED_SETS[which])
    _Fixing.log = []
    m = _module(NMF, W, H, FixNmf)
    n = m.fit(V, beta, -1.0, 17, alpha=0.2, l1_ratio=0.3, fixed_W=F)
    calls = list(_Fixing.log)
    _Fixing.log = None
    assert calls[0] == ("set_fixed_w", F.to(torch.uint8).tolist())
    # float64 oracle: every W update applied to the free columns only, penalties included
    gamma = orc.gamma_of(beta)
    l1, l2 = 0.2 * 0.3, 0.2 * 0.7
    Wo, Ho = W.clone(), H.clone()
    for _ in range(n):
        Wn = orc.nmf_update_w(V, Wo, Ho, beta, gamma, l1, l2)
        Wo[:, ~F] = Wn[:, ~F]
        Ho = orc.nmf_update_h(V, Wo, Ho, beta, gamma, l1, l2)
    assert torch.equal(m.W.data[:, F], W[:, F])                 # fixed columns: bit for bit their input
    torch.testing.assert_close(m.W.data, Wo, rtol=1e-10, atol=1e-12)
    torch.testing.assert_close(m.H.data, Ho, rtol=1e-10, atol=1e-12)


@pytest.mark.parametrize("which", list(FIXED_SETS))
def test_partial_cd_skips_fixed_columns_inside_the_sweep(which):
    V, W, H = _nmf_problem(5)
    F = _flags(W.shape[1], FIXED_SETS[which])
    m = _module(NMF, W, H, FixNmf)
    n = m.fit(V, 2, -1.0, 12, solver="cd", alpha=0.1, l1_ratio=0.5, fixed_W=F)
    l1, l2 = 0.05, 0.05

    def oracle(sweep):
        Wo, Ho = W.clone(), H.clone()
        for _ in range(n):
            Wo = sweep(V, Wo, Ho, l1, l2, F)
            Ho = cdo.update(V, Wo, Ho, 1, l1, l2)
        return Wo, Ho

    Wo, Ho = oracle(skip_sweep)
    assert torch.equal(m.W.data[:, F], W[:, F])
    torch.testing.assert_close(m.W.data, Wo, rtol=1e-10, atol=1e-12)
    torch.testing.assert_close(m.H.data, Ho, rtol=1e-10, atol=1e-12)
    # restoring the fixed columns after a plain sweep is a different update wherever a fixed column precedes a free one:
    # the test above would fail on it
    Wr, _ = oracle(restore_sweep)
    if which != "last":
        assert (Wr - Wo).abs().max() > 1e-3


def _plca_free_oracle(V, W, H, Z, F, n, W_alpha=1.):
    """The reference EM step (float64) with W's step kept on the free columns only; Z from every component's gradient."""
    for _ in range(n):
        Wn, H, Z = em_step(V, W, H, Z, W_alpha=W_alpha)
        W = torch.where(po._over(F, W).expand_as(W) if W.dim() > 2 else F.expand_as(W), W, Wn)
    return W, H, Z


@pytest.mark.parametrize("cls", [PLCA, SIPLCA])
@pytest.mark.parametrize("which", ["first", "scattered"])
@pytest.mark.parametrize("W_alpha", [1., 1.2])
def test_partial_em_updates_free_columns_only(cls, which, W_alpha):
    V, m = _plca_problem(cls, 7)
    F = _flags(4, [0, 1] if which == "first" else [1, 3])
    W0, H0, Z0 = m.W.data.clone(), m.H.data.clone(), m.Z.data.clone()
    m._engine_factory = PlcaOracleEngine if cls is PLCA else SiplcaOracleEngine
    n, _ = m.fit(V, -1.0, 14, False, W_alpha, fixed_W=F)
    Wo, Ho, Zo = _plca_free_oracle(V.double(), W0.double(), H0.double(), Z0.double(), F, n + 1, W_alpha)
    assert torch.equal(m.W.data[:, F], W0[:, F])
    for got, want in ((m.W.data, Wo), (m.H.data, Ho), (m.Z.data, Zo)):
        torch.testing.assert_close(got.double(), want, rtol=1e-4, atol=1e-6)


def test_partial_em_on_a_sparse_plca_target():
    V, m = _plca_problem(PLCA, 9)
    V, m = V.double(), m.double()            # the sparse fit computes in the factors' dtype
    V[V < 0.3] = 0
    F = _flags(4, [2])
    W0, H0, Z0 = m.W.data.clone(), m.H.data.clone(), m.Z.data.clone()
    m._engine_factory = OracleSparsePlcaEngine
    n, _ = m.fit(V.to_sparse(), -1.0, 11, fixed_W=F)
    Wo, Ho, Zo = _plca_free_oracle(V, W0, H0, Z0, F, n + 1)
    assert torch.equal(m.W.data[:, F], W0[:, F])
    for got, want in ((m.W.data, Wo), (m.H.data, Ho), (m.Z.data, Zo)):
        torch.testing.assert_close(got, want, rtol=1e-9, atol=1e-12)
    # every component fixed: the frozen-W fit, bit for bit
    runs = []
    for kw, fw in (({"trainable_W": False}, None), ({}, torch.ones(4, dtype=torch.bool))):
        mm = PLCA(W=W0.clone(), H=H0.clone(), Z=Z0.clone(), **kw).double()
        mm._engine_factory = OracleSparsePlcaEngine
        out = mm.fit(V.to_sparse(), -1.0, 11, **({} if fw is None else {"fixed_W": fw}))
        runs.append((out[0], mm.W.data, mm.H.data, mm.Z.data))
    assert runs[0][0] == runs[1][0] and all(torch.equal(a, b) for a, b in zip(runs[0][1:], runs[1][1:]))
