"""BatchedPLCA.fit(V, ..., lengths=L) -- a ragged batch, problem p being the EM fit of V[p, :L[p]] -- on the CPU (no GPU):
the host logic through a float64 engine that fits each problem on its real rows (the `_engine_factory` hook), every
refusal, and the fits against tests/golden/reference_batched_plca_ragged.npz (tools/make_golden_batched_plca_ragged.py: the
unmodified reference's `PLCA.fit` on each prefix V[p, :L[p]], in float64)."""
import os

import numpy as np
import pytest
import torch

from batched_plca_oracle import BatchedPlcaOracleEngine, em_step, kl_loss, raw_terms
from conftest import GOLDEN
from torchnmf_b200 import BatchedNMF, BatchedPLCA, BatchedSIPLCA, BatchedSIPLCA2, BatchedSIPLCA3

Z_GOLD = np.load(os.path.join(GOLDEN, "reference_batched_plca_ragged.npz"), allow_pickle=False)
CASES = sorted({k.split("/")[0] for k in Z_GOLD.files})


class RaggedPlcaOracleEngine(BatchedPlcaOracleEngine):
    """The ragged form of BatchedPlcaOracleEngine: problem p's EM step and loss in float64 on V[p, :L_p], W[p], H[p, :L_p],
    Hz[p, :L_p] and Z[p] alone, as that engine runs a batch of one problem of L_p rows.  Rows past L_p of H and Hz are
    never read or written."""

    def __init__(self, Vn, W, Hz, lengths):
        super().__init__(Vn, W, Hz)
        self.lengths = list(lengths)

    def plca_iterate(self, n_iter, H, Z, train_w, train_h, train_z, W_alpha=None, H_alpha=None, Z_alpha=None):
        self.alphas = (W_alpha, H_alpha, Z_alpha)
        for _ in range(n_iter):
            for p, n in enumerate(self.lengths):
                if not self.active[p]:
                    continue
                one = [None if a is None else a[p:p + 1].double() for a in (W_alpha, Z_alpha)]
                aH = None if H_alpha is None else H_alpha[p:p + 1, :n].double()
                W64 = self.W[p:p + 1].double()
                dW, dHz = raw_terms(self.Vn[p:p + 1, :n], W64, self.H[p:p + 1, :n].double())
                Wn, Hn, Zn = em_step(W64, H[p:p + 1, :n].double(), Z[p:p + 1].double(), dW, dHz, train_w, train_h, train_z,
                                     one[0], aH, one[1])
                self.W[p] = Wn[0].float(); H[p, :n] = Hn[0].float(); Z[p] = Zn[0].float()
                self.H[p, :n] = H[p, :n] * Z[p]
                self.steps[p] += 1

    def plca_losses(self, norm):
        for p, n in enumerate(self.lengths):
            if self.active[p]:
                self._last[p] = kl_loss(self.Vn[p:p + 1, :n], self.W[p:p + 1].double(), self.H[p:p + 1, :n].double(),
                                        norm[p:p + 1].double())[0]
        return self._last.clone()


def _hook(m, log=None):
    """Fit m through the ragged oracle; `log` collects the factory's keyword arguments and the engines."""
    log = [] if log is None else log

    def factory(Vn, W, Hz, **kw):
        log.append(kw)
        eng = RaggedPlcaOracleEngine(Vn, W, Hz, kw["lengths"]) if kw else BatchedPlcaOracleEngine(Vn, W, Hz)
        log.append(eng)
        return eng
    m._engine_factory = factory
    return log


def _inputs(lengths=(12, 1, 7, 10), N=12, C=9, R=3, seed=0, pad=float("nan"), sentinel=5.0):
    P = len(lengths)
    g = torch.Generator().manual_seed(seed)
    V = torch.rand(P, N, C, generator=g) * torch.linspace(0.2, 2.0, P).view(P, 1, 1) + 0.01
    V[0] = torch.rand(N, 1, generator=g) @ torch.rand(1, C, generator=g) + 0.01          # rank 1: stops early
    W0 = torch.rand(P, C, R, generator=g) + 0.1
    H0 = torch.rand(P, N, R, generator=g) + 0.1
    Z0 = torch.rand(P, R, generator=g) + 0.2
    for p, n in enumerate(lengths):
        V[p, n:] = pad
        H0[p, n:] = sentinel
    return V, W0, H0, Z0


def _module(W0, H0, Z0, **kw):
    """A BatchedPLCA whose factors are exactly W0, H0 and Z0 (the constructor's normalisation undone by a copy)."""
    m = BatchedPLCA(W=W0, H=H0, Z=Z0, **kw)
    for k, t in (("W", W0), ("H", H0), ("Z", Z0)):
        getattr(m, k).data.copy_(t)
    return m


def _normalised(W0, H0, Z0, lengths):
    """Each problem's factors normalised over its real rows; H's padding rows kept as they are."""
    H = H0.clone()
    for p, n in enumerate(lengths):
        H[p, :n] = H0[p, :n] / H0[p, :n].sum(0)
    return W0 / W0.sum(1, keepdim=True), H, Z0 / Z0.sum(1, keepdim=True)


def _fit(m, V, **kw):
    n_iter, norm = m.fit(V, **kw)
    return n_iter, norm, m.W.data.clone(), m.H.data.clone(), m.Z.data.clone()


def _single(V, W0, H0, Z0, p, n, trainable=(True, True, True), **kw):
    """The P = 1 fit without lengths of problem p's real rows, through the oracle."""
    tw, th, tz = trainable
    m = _module(W0[p:p + 1], H0[p:p + 1, :n], Z0[p:p + 1], trainable_W=tw, trainable_H=th, trainable_Z=tz)
    _hook(m)
    return _fit(m, V[p:p + 1, :n], **kw)


def golden_case(name):
    c = {k.split("/", 1)[1]: Z_GOLD[k] for k in Z_GOLD.files if k.startswith(name + "/")}
    return {k: (torch.from_numpy(v.copy()) if v.dtype != np.float64 or v.ndim else float(v)) for k, v in c.items()}


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference(name):
    c = golden_case(name)
    lengths = c["lengths"].tolist()
    m = BatchedPLCA(W=c["W0"], H=c["H0"], Z=c["Z0"], trainable_W=bool(c["trainable_W"]), trainable_Z=bool(c["trainable_Z"]))
    _hook(m)
    W_alpha = c["W_alpha"].reshape(-1, 1, 1) if isinstance(c["W_alpha"], torch.Tensor) else c["W_alpha"]
    n_iter, norm = m.fit(c["V"], tol=c["tol"], max_iter=int(c["max_iter"]), W_alpha=W_alpha, H_alpha=c["H_alpha"],
                         Z_alpha=c["Z_alpha"], lengths=lengths)
    assert n_iter.tolist() == c["n_iter"].tolist()
    assert torch.allclose(norm.double(), c["norm"], rtol=1e-6)
    for k in ("W", "H", "Z"):
        got, want = getattr(m, k).data, c[k]
        assert torch.allclose(got, want, rtol=1e-3, atol=1e-5 * float(want.abs().max())), k
    for p, n in enumerate(lengths):
        assert bool((m.H.data[p, n:] == 0).all())          # zero padding stays zero


def test_fixtures_cover_the_cases():
    lens = [golden_case(n)["lengths"].tolist() for n in CASES]
    assert any(1 in L for L in lens) and any(30 in L for L in lens)
    assert any(len(set(golden_case(n)["n_iter"].tolist())) > 1 for n in CASES)
    assert bool(torch.isnan(golden_case(CASES[0])["V"]).any())


@pytest.mark.parametrize("as_tensor", [False, True])
def test_each_problem_is_its_own_fit(as_tensor):
    lengths = [12, 1, 7, 10]
    V, W0, H0, Z0 = _inputs(lengths)
    m = _module(W0, H0, Z0)
    log = _hook(m)
    L = torch.tensor(lengths, dtype=torch.int32) if as_tensor else lengths
    n_iter, norm, W, H, Z = _fit(m, V, tol=1e-3, max_iter=200, lengths=L)
    eng = log[1]
    assert log[0] == {"lengths": lengths}
    assert len(set(n_iter.tolist())) > 1
    for p, n in enumerate(lengths):
        # the EM steps problem p received: its own loop index + 1, none after it stopped
        assert eng.steps[p] == n_iter[p] + 1
        n1, norm1, W1, H1, Z1 = _single(V, W0, H0, Z0, p, n, tol=1e-3, max_iter=200)
        assert n1.tolist() == [int(n_iter[p])]
        assert torch.equal(norm1[0], norm[p]) and torch.equal(norm[p], V[p, :n].sum())
        assert torch.equal(W1[0], W[p]) and torch.equal(H1[0], H[p, :n]) and torch.equal(Z1[0], Z[p])
        assert bool((H[p, n:] == 5.0).all())


def test_padding_of_v_is_never_read():
    lengths = [12, 1, 7, 10]
    outs = []
    for pad in (float("nan"), -3.0, 0.0):
        V, W0, H0, Z0 = _inputs(lengths, pad=pad)
        m = _module(W0, H0, Z0)
        _hook(m)
        outs.append(_fit(m, V, tol=1e-4, max_iter=40, lengths=lengths))
    for o in outs[1:]:
        for a, b in zip(outs[0], o):
            assert torch.equal(a, b)


def test_h_alpha_padding_and_every_alpha_form():
    lengths = [12, 1, 7, 10]
    V, W0, H0, Z0 = _inputs(lengths)
    aH = torch.full((4, 12, 3), 1.2)
    aH_nan = aH.clone()
    for p, n in enumerate(lengths):
        aH_nan[p, n:] = float("nan")
    kw = dict(tol=float("-inf"), max_iter=12, W_alpha=torch.full((9, 3), 1.3), Z_alpha=torch.tensor([[1.1], [0.9], [1.0],
                                                                                                     [1.2]]))
    outs = []
    for H_alpha in (1.2, aH, aH_nan):
        m = _module(W0, H0, Z0)
        log = _hook(m)
        outs.append(_fit(m, V, H_alpha=H_alpha, lengths=lengths, **kw))
        assert log[1].alphas[1].shape == (4, 12, 3)
    for o in outs[1:]:
        for a, b in zip(outs[0], o):
            assert torch.equal(a, b)
    for p, n in enumerate(lengths):
        one = _single(V, W0, H0, Z0, p, n, H_alpha=1.2, W_alpha=kw["W_alpha"], Z_alpha=kw["Z_alpha"][p:p + 1],
                      tol=kw["tol"], max_iter=kw["max_iter"])
        assert torch.equal(one[2][0], outs[0][2][p]) and torch.equal(one[3][0], outs[0][3][p, :n])


@pytest.mark.parametrize("frozen", ["Z", "W", "WZ", "H"])
def test_frozen_factors(frozen):
    lengths = [12, 1, 7, 10]
    V, W0, H0, Z0 = _inputs(lengths)
    trainable = tuple(k not in frozen for k in "WHZ")
    m = _module(W0, H0, Z0, trainable_W=trainable[0], trainable_H=trainable[1], trainable_Z=trainable[2])
    _hook(m)
    n_iter, norm, W, H, Z = _fit(m, V, tol=float("-inf"), max_iter=6, lengths=lengths)
    for k, got, start in (("W", W, W0), ("H", H, H0), ("Z", Z, Z0)):
        assert torch.equal(got, start) == (k in frozen)
    for p, n in enumerate(lengths):
        one = _single(V, W0, H0, Z0, p, n, trainable, tol=float("-inf"), max_iter=6)
        assert torch.equal(one[2][0], W[p]) and torch.equal(one[3][0], H[p, :n]) and torch.equal(one[4][0], Z[p])


def test_full_lengths_equal_no_lengths():
    V, W0, H0, Z0 = _inputs((12, 12, 12, 12))
    outs = []
    for lengths in (None, [12] * 4):
        m = _module(W0, H0, Z0)
        _hook(m)
        outs.append(_fit(m, V, tol=1e-3, max_iter=60, lengths=lengths))
    for a, b in zip(*outs):
        assert torch.equal(a, b)


@pytest.mark.parametrize("dtype", [torch.float64, torch.float16, torch.bfloat16])
def test_targets_and_modules_of_other_dtypes(dtype):
    lengths = [12, 1, 7, 10]
    V, W0, H0, Z0 = _inputs(lengths)
    m = _module(W0, H0, Z0)
    _hook(m)
    Vt = V.to(dtype)
    n_iter, norm, *_ = _fit(m, Vt, tol=1e-3, max_iter=30, lengths=lengths)
    assert norm.dtype == dtype and all(torch.equal(norm[p], Vt[p, :n].sum()) for p, n in enumerate(lengths))
    # a float64 module keeps its padding sentinels
    m64 = _module(W0, H0, Z0).double()
    _hook(m64)
    m64.fit(V.double(), tol=1e-3, max_iter=30, lengths=lengths)
    assert m64.H.dtype == torch.float64
    for p, n in enumerate(lengths):
        assert bool((m64.H.data[p, n:] == 5.0).all())


def test_three_argument_factory_on_uniform_fits():
    V, W0, H0, Z0 = _inputs((12, 12, 12, 12))
    m = _module(W0, H0, Z0)
    m._engine_factory = lambda Vn, W, Hz: BatchedPlcaOracleEngine(Vn, W, Hz)
    n_iter, _ = m.fit(V, tol=1e-3, max_iter=30)
    assert n_iter.shape == (4,)


def test_refusals_before_any_engine():
    lengths = [12, 1, 7, 10]
    V, W0, H0, Z0 = _inputs(lengths)
    m = _module(W0, H0, Z0)
    log = _hook(m)
    bad = [
        ([12, 1, 7], "holds 3 values for 4 problems"),
        ([12, 0, 7, 10], r"every length must be in \[1, N = 12\] \(got 0\)"),
        ([12, 13, 7, 10], r"every length must be in \[1, N = 12\] \(got 13\)"),
        (torch.tensor([12., 1., 7., 10.]), "must hold integers"),
        (torch.tensor([[12, 1, 7, 10]]), "must be 1-D"),
        ([12, True, 7, 10], "sequence of ints"),
        (torch.tensor([True] * 4), "must hold integers"),
        ([12, 1.0, 7, 10], "sequence of ints"),
        (12, "sequence of ints or an integer tensor"),
        ("abcd", "sequence of ints or an integer tensor"),
    ]
    for L, msg in bad:
        with pytest.raises(ValueError, match=msg):
            m.fit(V, lengths=L)
    with pytest.raises(ValueError, match="a shared target"):
        m.fit(V[0], lengths=lengths)
    for kw in ("mask", "weight", "group"):
        with pytest.raises(TypeError):
            m.fit(V, lengths=lengths, **{kw: None})
    with pytest.raises(NotImplementedError):
        m.fit(V.nan_to_num().to_sparse(), lengths=lengths)
    with pytest.raises(ValueError):
        m.fit(V, precision="f16", lengths=lengths)
    with pytest.raises(AssertionError, match="Target should be non-negative."):
        m.fit(torch.where(torch.isnan(V), V, -V), lengths=lengths)
    big = BatchedPLCA((2, 4, 3), rank=257)
    _hook(big)
    with pytest.raises(ValueError, match="rank <= 256"):
        big.fit(torch.rand(2, 4, 3), lengths=[4, 2])
    assert log == []
    for cls, shape, kw in ((BatchedSIPLCA, (2, 1, 3, 8), {"T": 2}), (BatchedSIPLCA2, (2, 1, 3, 5, 6), {"kernel_size": 2}),
                           (BatchedSIPLCA3, (2, 1, 3, 4, 5, 6), {"kernel_size": 2})):
        s = cls(shape, rank=2, **kw)
        slog = _hook(s)
        with pytest.raises(ValueError, match=f"lengths is not supported by {cls.__name__}"):
            s.fit(torch.rand(*shape), lengths=[2, 2])
        assert slog == []


def test_nmf_lengths_messages_unchanged():
    m = BatchedNMF((2, 6, 4), rank=2)
    with pytest.raises(ValueError, match="solver='cd' does not fit ragged batches"):
        m.fit(torch.rand(2, 6, 4), beta=2, solver="cd", lengths=[6, 3])
    with pytest.raises(ValueError, match=r"every length must be in \[1, N = 6\] \(got 7\)"):
        m.fit(torch.rand(2, 6, 4), lengths=[7, 3])
