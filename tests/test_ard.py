"""Automatic relevance determination (`fit(V, ..., ard=ARD(...))`), without a GPU.

The float64 ARD oracle (tests/ard_oracle.py) is checked against the objective it descends and on planted-rank problems;
then the host logic of `fit(..., ard=...)` -- the refusals, the default b of every target form, the loop and its stop rule
-- runs through an oracle engine plugged in with the `_engine_factory` hook.
"""
import ctypes
import math
import os

import pytest
import torch

import ard_oracle as ao
from ard_cases import PLANTED_ITERS, planted_nmf, planted_nmfd, relevant
from oracle import mu_oracle as orc
from oracle_engine import OracleNmfEngine, OracleNmfdEngine
from torchnmf_b200 import NMF, NMF2D, NMFD, BatchedNMF, PLCA
from torchnmf_b200.nmf import ARD

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F64 = torch.float64


def _mean(V):
    """mean(V) as fit() takes it for b: the float64 sum over the cells, divided by their count."""
    return float(V.sum(dtype=F64)) / V.numel()


def _nmf_problem(seed, N=24, C=18, R=5, positive=False):
    g = torch.Generator().manual_seed(seed)
    V = torch.rand(N, 3, generator=g, dtype=F64) @ torch.rand(3, C, generator=g, dtype=F64)
    V += (0.05 if positive else 0.0) + 0.05 * torch.rand(N, C, generator=g, dtype=F64)
    if not positive:
        V[torch.rand(N, C, generator=g) < 0.1] = 0.0
    return V, torch.rand(C, R, generator=g, dtype=F64) + 0.1, torch.rand(N, R, generator=g, dtype=F64) + 0.1


def _nmfd_problem(seed, B=2, C=6, T=3, Lin=15, R=4):
    g = torch.Generator().manual_seed(seed)
    V = torch.rand(B, C, Lin + T - 1, generator=g, dtype=F64) + 0.05
    return V, torch.rand(C, R, T, generator=g, dtype=F64) + 0.1, torch.rand(B, R, Lin, generator=g, dtype=F64) + 0.1


def _selector(form, shape, seed):
    g = torch.Generator().manual_seed(seed + 100)
    if form == "mask":
        return torch.rand(shape, generator=g) < 0.7
    if form == "weight":
        w = torch.rand(shape, generator=g, dtype=F64) * 2
        w[torch.rand(shape, generator=g) < 0.2] = 0.0
        return w
    return None


# ---- the oracle ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("form", ["dense", "mask", "weight"])
@pytest.mark.parametrize("kind,beta", [("nmf", b) for b in (0, 0.5, 1, 1.5, 2, 3)] + [("nmfd", 0.5), ("nmfd", 1)])
def test_oracle_objective_never_increases(kind, beta, form):
    V, W, H = _nmf_problem(3, positive=beta == 0) if kind == "nmf" else _nmfd_problem(3)
    S = _selector(form, V.shape, 3)
    trace = []
    phi = 1.0 if beta != 2 else 0.05
    ao.fit(V, W, H, beta=beta, tol=float("-inf"), max_iter=40, a=5.0, phi=phi, kind=kind, S=S, trace=trace)
    for i in range(1, len(trace)):
        assert trace[i] <= trace[i - 1] + 1e-12 * abs(trace[i - 1]), (i, trace[i - 1], trace[i])


def test_oracle_keeps_the_planted_rank_of_nmf():
    V, W0, H0 = planted_nmf()
    _, _, lam, _, b, c = ao.fit(V, W0, H0, beta=1, tol=float("-inf"), max_iter=PLANTED_ITERS, a=5.0)
    assert len(relevant(lam, b / c)) == 4


def test_oracle_keeps_the_planted_kernels_of_nmfd():
    V, W0, H0 = planted_nmfd()
    _, _, lam, _, b, c = ao.fit(V, W0, H0, beta=1, tol=float("-inf"), max_iter=PLANTED_ITERS, a=5.0, kind="nmfd")
    assert len(relevant(lam, b / c)) == 2


def test_oracle_pruned_components_settle_at_the_bound():
    V, W0, H0 = planted_nmf()
    _, _, lam, _, b, c = ao.fit(V, W0, H0, beta=1, tol=float("-inf"), max_iter=PLANTED_ITERS, a=5.0)
    pruned = [k for k in range(lam.numel()) if k not in relevant(lam, b / c)]
    assert pruned and all(abs(float(lam[k]) / (b / c) - 1) < 1e-3 for k in pruned)


@pytest.mark.parametrize("beta", [0.5, 1, 2])
def test_oracle_step_with_equal_penalties_is_the_l1_update(beta):
    V, W, H = _nmf_problem(5)
    p = 0.37
    gamma = orc.gamma_of(beta)
    lam = torch.full((W.shape[1],), 1.0 / p, dtype=F64)
    pen = 1.0 / lam
    assert torch.equal(pen, torch.full_like(pen, p))
    num, den, cs = ao.terms(V, W, H, beta, 0)
    W1 = ao.ratio(W, num, den, gamma, pen, cs)
    assert torch.equal(W1, orc.nmf_update_w(V, W, H, beta, gamma, l1_reg=p))
    num, den, cs = ao.terms(V, W1, H, beta, 1)
    assert torch.equal(ao.ratio(H, num, den, gamma, pen, cs), orc.nmf_update_h(V, W1, H, beta, gamma, l1_reg=p))


# ---- host logic through an oracle engine -------------------------------------------------------------------------------

class _ArdMixin:
    """The ARD calls of the engine interface on the oracle: the penalties enter update_w / update_h while registered."""
    log = None
    ard_kind = "nmf"

    def _init_log(self):
        self.calls = _ArdMixin.log if _ArdMixin.log is not None else []
        self._ard = None

    def set_ard(self, b, c, phi):
        self.calls.append(("set_ard", b, c, phi))
        if b is None:
            self._ard = None
            return
        lam = ao.init_lambda(self.W, self.H, b, c)
        self._ard = dict(b=b, c=c, phi=phi, lam=lam, pen=phi / lam, change=0.0)

    def ard_update(self):
        self.calls.append(("ard_update",))
        s = self._ard
        new = ao.init_lambda(self.W, self.H, s["b"], s["c"])
        s["change"] = float(((new - s["lam"]).abs() / s["lam"]).max())
        s["lam"], s["pen"] = new, s["phi"] / new

    def ard_state(self):
        return self._ard["lam"], self._ard["pen"], self._ard["change"]

    def ard_change(self):
        self.calls.append(("ard_change",))
        return self._ard["change"]

    def _pen_update(self, which, beta, gamma):
        X = self.W if which == 0 else self.H
        num, den, cs = ao.terms(self.V, self.W, self.H, beta, which, self.ard_kind)
        X.copy_(ao.ratio(X, num, den, gamma, self._ard["pen"], cs))

    def update_w(self, beta, gamma, l1, l2):
        self.calls.append(("update_w", l1, l2))
        if self._ard is not None:
            assert l1 == 0 and l2 == 0
            return self._pen_update(0, beta, gamma)
        super().update_w(beta, gamma, l1, l2)

    def update_h(self, beta, gamma, l1, l2):
        self.calls.append(("update_h", l1, l2))
        if self._ard is not None:
            assert l1 == 0 and l2 == 0
            return self._pen_update(1, beta, gamma)
        super().update_h(beta, gamma, l1, l2)


class ArdNmfEngine(_ArdMixin, OracleNmfEngine):
    def __init__(self, V, W, H):
        super().__init__(V, W, H)
        self._init_log()

    def iterate(self, n, beta, gamma, l1, l2):
        self.calls.append(("iterate", n, l1, l2))
        for _ in range(n):
            self.update_w(beta, gamma, l1, l2)
            self.update_h(beta, gamma, l1, l2)
            if self._ard is not None:
                self.ard_update()


class ArdNmfdEngine(_ArdMixin, OracleNmfdEngine):
    ard_kind = "nmfd"

    def __init__(self, V, W, H):
        super().__init__(V, W, H)
        self._init_log()


@pytest.mark.parametrize("beta", [0.5, 1, 2])
def test_fit_follows_the_oracle(beta):
    V, W0, H0 = _nmf_problem(7)
    V, W0, H0 = V.float(), W0.float(), H0.float()
    m = NMF(W=W0, H=H0)
    m._engine_factory = ArdNmfEngine
    n = m.fit(V, beta, tol=float("-inf"), max_iter=35, ard=ARD(a=6.0, phi=0.5))
    W, H, lam, n_ref, b, c = ao.fit(V, W0, H0, beta=beta, tol=float("-inf"), max_iter=35, a=6.0, phi=0.5,
                                    mean_v=_mean(V), dtype=torch.float32)
    assert n == n_ref == 35
    assert torch.equal(m.W.data, W) and torch.equal(m.H.data, H)
    assert torch.equal(m.ard_lambda, lam)
    assert m.ard_lambda.dtype == torch.float32 and m.ard_lambda.shape == (5,)
    assert m.ard_bound == b / c


def test_nmfd_fit_follows_the_oracle_with_one_call_per_update():
    V, W0, H0 = _nmfd_problem(8)
    V, W0, H0 = V.float(), W0.float(), H0.float()
    m = NMFD(W=W0, H=H0)
    log = _ArdMixin.log = []
    try:
        m._engine_factory = ArdNmfdEngine
        n = m.fit(V, 1, tol=float("-inf"), max_iter=12, ard=ARD())
    finally:
        _ArdMixin.log = None
    W, H, lam, n_ref, b, c = ao.fit(V, W0, H0, beta=1, tol=float("-inf"), max_iter=12, kind="nmfd",
                                    mean_v=_mean(V), dtype=torch.float32)
    assert n == n_ref == 12
    assert torch.equal(m.W.data, W) and torch.equal(m.H.data, H) and torch.equal(m.ard_lambda, lam)
    steps = [c[0] for c in log if c[0] in ("update_w", "update_h", "ard_update")]
    assert steps == ["update_w", "update_h", "ard_update"] * 12
    assert ao.constants(W0, H0, 5.0) == 6 * 3 + 2 * 15 + 6.0 and math.isclose(m.ard_bound, b / c)


def test_stop_rule_matches_the_oracle():
    V, W0, H0 = planted_nmf()
    tol = 1e-3
    m = NMF(W=W0, H=H0)
    m._engine_factory = ArdNmfEngine
    n = m.fit(V, 1, tol=tol, max_iter=300, ard=ARD())
    _, _, _, n_ref, _, _ = ao.fit(V, W0, H0, beta=1, tol=tol, max_iter=300, mean_v=_mean(V),
                                  dtype=torch.float32)
    assert n == n_ref and n % 10 == 0 and 10 <= n < 300


class _ScriptedEngine:
    """Records the ARD registration and reports scripted changes: what the host loop does with them."""
    changes = []
    seen = []
    device = torch.device("cpu")
    precision = "oracle"
    kind = "nmf"

    def __init__(self, V, W, H, **kw):
        self.V, self.W, self.H = V, W, H
        self.checks = 0

    def close(self):
        pass

    def minmax(self):
        return 0.0, 1.0

    def set_mask(self, M):
        pass

    def set_weight(self, Wt):
        pass

    def loss(self, beta):
        return 1.0

    def set_ard(self, b, c, phi):
        _ScriptedEngine.seen.append((b, c, phi))

    def iterate(self, n, beta, gamma, l1, l2):
        pass

    def ard_change(self):
        self.checks += 1
        return _ScriptedEngine.changes[self.checks - 1]

    def ard_state(self):
        R = self.W.shape[1]
        return torch.ones(R), torch.ones(R), 0.0


@pytest.mark.parametrize("changes,tol,want", [([0.5, 0.2, 1e-5, 0.0], 1e-4, 30), ([1e-5], 1e-4, 10),
                                              ([0.5] * 5, 1e-4, 50), ([0.5, float("nan"), 0.0], 1e-4, 30)])
def test_stop_rule_fires_at_the_first_check_below_tol(changes, tol, want):
    _ScriptedEngine.changes, _ScriptedEngine.seen = changes, []
    m = NMF(W=torch.rand(6, 3), H=torch.rand(5, 3))
    m._engine_factory = _ScriptedEngine
    assert m.fit(torch.rand(5, 6), 1, tol=tol, max_iter=50, ard=ARD()) == want


def _default_b(mean_v, R=3, a=5.0, prod_k=1):
    return math.sqrt((a - 1) * (a - 2) * mean_v / (R * prod_k))


def _b_seen(model, V, **kw):
    _ScriptedEngine.changes, _ScriptedEngine.seen = [0.0], []
    model._engine_factory = _ScriptedEngine
    model.fit(V, 1, max_iter=10, ard=ARD(), **kw)
    (b, c, phi), = _ScriptedEngine.seen
    return b, c


def test_default_b_of_every_target_form():
    g = torch.Generator().manual_seed(4)
    N, C, R = 7, 9, 3
    V = torch.rand(N, C, generator=g)

    def nmf():
        return NMF(W=torch.rand(C, R, generator=g), H=torch.rand(N, R, generator=g))

    b, c = _b_seen(nmf(), V)
    assert math.isclose(b, _default_b(float(V.double().mean())), rel_tol=1e-12) and c == C + N + 6.0
    Vh = V.half()
    b, _ = _b_seen(nmf(), Vh)
    assert math.isclose(b, _default_b(float(Vh.double().mean())), rel_tol=1e-12)
    M = torch.rand(N, C, generator=g) < 0.6
    Vn = V.clone()
    Vn[~M] = float("nan")
    b, _ = _b_seen(nmf(), Vn, mask=M)
    assert math.isclose(b, _default_b(float(V.double()[M].mean())), rel_tol=1e-12)
    Wt = torch.rand(N, C, generator=g) * (torch.rand(N, C, generator=g) < 0.5)
    b, _ = _b_seen(nmf(), V, weight=Wt)
    assert math.isclose(b, _default_b(float(V.double()[Wt > 0].mean())), rel_tol=1e-12)
    Vs = (V * (V > 0.6)).to_sparse()
    b, _ = _b_seen(nmf(), Vs)
    assert math.isclose(b, _default_b(float((V * (V > 0.6)).double().sum()) / (N * C)), rel_tol=1e-12)
    b, _ = _b_seen(nmf(), Vn, mask=M.to_sparse())
    assert math.isclose(b, _default_b(float(V.double()[M].mean())), rel_tol=1e-12)
    b, _ = _b_seen(nmf(), V, weight=Wt.to_sparse())
    assert math.isclose(b, _default_b(float(V.double()[Wt > 0].mean())), rel_tol=1e-12)
    Vd = torch.rand(2, 4, 12, generator=g)
    md = NMFD(W=torch.rand(4, R, 5, generator=g), H=torch.rand(2, R, 8, generator=g))
    b, c = _b_seen(md, Vd)
    assert math.isclose(b, _default_b(float(Vd.double().mean()), prod_k=5), rel_tol=1e-12)
    assert c == 4 * 5 + 2 * 8 + 6.0


def test_explicit_b_and_phi_are_passed_through():
    _ScriptedEngine.changes, _ScriptedEngine.seen = [0.0], []
    m = NMF(W=torch.rand(6, 3), H=torch.rand(5, 3))
    m._engine_factory = _ScriptedEngine
    m.fit(torch.rand(5, 6), 2, max_iter=10, ard=ARD(a=1.5, b=0.25, phi=3.0))
    assert _ScriptedEngine.seen == [(0.25, 6 + 5 + 2.5, 3.0)]
    assert m.ard_bound == 0.25 / 13.5


class _NoEngine:
    def __init__(self, *a, **k):
        raise AssertionError("an engine was built")


@pytest.mark.parametrize("ard,kw,match", [
    ("x", {}, "ARD instance"),
    (ARD(a=float("nan")), {}, "ARD.a"),
    (ARD(a=-1.0, b=1.0), {}, "ARD.a"),
    (ARD(b=0.0), {}, "ARD.b"),
    (ARD(b=float("inf")), {}, "ARD.b"),
    (ARD(phi=0.0), {}, "ARD.phi"),
    (ARD(phi=float("nan")), {}, "ARD.phi"),
    (ARD(a=2.0), {}, "a must be > 2"),
    (ARD(), {"alpha": 0.1}, "alpha"),
    (ARD(), {"solver": "cd"}, "solver"),
    (ARD(), {"group": object()}, "group"),
    (ARD(), {"fixed_W": torch.tensor([True, False, False])}, "fixed_W"),
])
def test_refusals_before_any_engine(ard, kw, match):
    m = NMF(W=torch.rand(6, 3), H=torch.rand(5, 3))
    m._engine_factory = _NoEngine
    with pytest.raises(ValueError, match=match):
        m.fit(torch.rand(5, 6), 2, ard=ard, **kw)


@pytest.mark.parametrize("frozen", ["W", "H"])
def test_frozen_factor_is_refused(frozen):
    m = NMF(W=torch.rand(6, 3), H=torch.rand(5, 3), trainable_W=frozen != "W", trainable_H=frozen != "H")
    m._engine_factory = _NoEngine
    with pytest.raises(ValueError, match="trainable"):
        m.fit(torch.rand(5, 6), 1, ard=ARD())


def test_explicit_b_lifts_the_shape_limit():
    _ScriptedEngine.changes, _ScriptedEngine.seen = [0.0], []
    m = NMF(W=torch.rand(6, 3), H=torch.rand(5, 3))
    m._engine_factory = _ScriptedEngine
    m.fit(torch.rand(5, 6), 1, max_iter=10, ard=ARD(a=2.0, b=1.0))
    assert len(_ScriptedEngine.seen) == 1


def test_other_fits_do_not_take_the_keyword():
    with pytest.raises(TypeError):
        NMF(W=torch.rand(6, 3), H=torch.rand(5, 3)).sparse_fit(torch.rand(5, 6), ard=ARD())
    with pytest.raises(TypeError):
        BatchedNMF(W=torch.rand(2, 6, 3), H=torch.rand(2, 5, 3)).fit(torch.rand(2, 5, 6), ard=ARD())
    with pytest.raises(TypeError):
        PLCA(W=torch.rand(6, 3), H=torch.rand(5, 3)).fit(torch.rand(5, 6), ard=ARD())


class _NoArdEngine(OracleNmfEngine):
    def __getattribute__(self, name):
        if name.startswith("ard") or name == "set_ard":
            raise AssertionError(f"{name} called without ard")
        return super().__getattribute__(name)


def test_without_ard_no_ard_call_is_made():
    V, W0, H0 = _nmf_problem(9)
    m = NMF(W=W0.float(), H=H0.float())
    m._engine_factory = _NoArdEngine
    n = m.fit(V.float(), 1, tol=float("-inf"), max_iter=12)
    W, H, n_ref, _ = orc.fit(V.float(), W0.float(), H0.float(), beta=1, tol=float("-inf"), max_iter=12)
    assert n == n_ref and torch.equal(m.W.data, W) and torch.equal(m.H.data, H)
    assert not hasattr(m, "ard_lambda")


def test_nmf2d_takes_the_keyword():
    from oracle_engine import OracleNmfndEngine

    class Engine(_ArdMixin, OracleNmfndEngine):
        ard_kind = "nmf2d"

        def __init__(self, V, W, H):
            super().__init__(V, W, H)
            self._init_log()

    g = torch.Generator().manual_seed(2)
    V = torch.rand(1, 3, 6, 9, generator=g) + 0.1
    W0, H0 = torch.rand(3, 2, 2, 3, generator=g) + 0.1, torch.rand(1, 2, 5, 7, generator=g) + 0.1
    m = NMF2D(W=W0, H=H0)
    m._engine_factory = Engine
    assert m.fit(V, 1, tol=float("-inf"), max_iter=5, ard=ARD()) == 5
    W, H, lam, _, b, c = ao.fit(V, W0, H0, beta=1, tol=float("-inf"), max_iter=5, kind="nmf2d",
                                mean_v=_mean(V), dtype=torch.float32)
    assert torch.equal(m.W.data, W) and torch.equal(m.ard_lambda, lam)
    assert math.isclose(b, _default_b(float(V.double().mean()), R=2, prod_k=6), rel_tol=1e-12)


# ---- the C ABI ----------------------------------------------------------------------------------------------------------

def test_ard_entry_points_are_bound_and_refuse_a_null_context():
    from torchnmf_b200 import _capi
    _vp, _dbl, _int = ctypes.c_void_p, ctypes.c_double, ctypes.c_int
    assert _capi.SIGNATURES["nmfb200_set_ard"] == (_int, [_vp, _vp, _vp, _dbl, _dbl, _dbl, _vp])
    assert _capi.SIGNATURES["nmfb200_ard_update"] == (_int, [_vp, _vp, _vp, _vp])
    assert _capi.SIGNATURES["nmfb200_ard_read"] == (_int, [_vp, _vp, _vp, _vp, _vp])
    lib = _capi.load()
    assert lib.nmfb200_set_ard(None, None, None, 1.0, 1.0, 1.0, None) == 1          # NMFB200_ERR_INVALID
    assert b"null context" in lib.nmfb200_last_error()
    assert lib.nmfb200_ard_update(None, None, None, None) == 1
    assert b"null context" in lib.nmfb200_last_error()
    assert lib.nmfb200_ard_read(None, None, None, None, None) == 1
    assert b"null context" in lib.nmfb200_last_error()
    header = " ".join(open(os.path.join(ROOT, "include", "nmf_b200.h")).read().split())
    assert ("int nmfb200_set_ard(nmfb200_ctx* ctx, const float* W, const float* H, double b, double c, double phi, "
            "void* stream);") in header
    assert "int nmfb200_ard_update(nmfb200_ctx* ctx, const float* W, const float* H, void* stream);" in header
    assert "int nmfb200_ard_read(nmfb200_ctx* ctx, float* lambda, float* pen, float* change, void* stream);" in header
