"""CPU-side tests: module surface (mirrors reference tests/test_nmf.py:8-69), the C-ABI library's
symbols, loud failure without CUDA, and the host logic of fit() driven by an oracle-backed engine."""
import ctypes
import math
import os
import re

import pytest
import torch

from conftest import ROOT, load_golden
from oracle import mu_oracle as orc
from torchnmf_b200 import NMF, NMFD, BaseComponent, _capi
from oracle_engine import OracleNmfEngine, OracleNmfdEngine

CASES = load_golden()


# ---- constructor validity matrix: reference tests/test_nmf.py:8-37 ------------------------------
@pytest.mark.parametrize("W", [(50, 8), torch.rand(50, 8), None])
@pytest.mark.parametrize("H", [(100, 8), torch.rand(100, 8), None])
def test_base_valid_construct(W, H):
    m = BaseComponent(8, W, H)
    assert (m.H is None) == (H is None)
    assert (m.W is None) == (W is None)


@pytest.mark.parametrize("rank, W, H", [
    (None, None, None),
    (None, (50, 8), (100, 10)),
    (None, torch.rand(50, 8), (100, 10)),
    (None, -torch.rand(50, 8) - 1, (100, 8)),
    (None, (50, 8), torch.rand(100, 10)),
    (None, (50, 8), -torch.rand(100, 8) - 1),
    (None, torch.rand(50, 8), torch.rand(100, 10)),
])
def test_base_invalid_construct(rank, W, H):
    with pytest.raises(Exception):
        BaseComponent(rank, W, H)


def test_shapes_and_repr():
    # reference tests/test_nmf.py:40-69
    m = NMF((100, 50))
    assert m().shape == (100, 50) and m.rank == 50
    m = NMF((20, 30), 5)
    assert m.W.shape == (30, 5) and m.H.shape == (20, 5)
    assert "out_channels=30" in repr(m)
    d = NMFD((100, 50, 100))
    assert d().shape == (100, 50, 100)
    d = NMFD((1, 33, 50), 16, 3)
    assert d.W.shape == (33, 16, 3) and d.H.shape == (1, 16, 48) and d().shape == (1, 33, 50)
    for bad in [(100, 50, 50), (100,)]:
        with pytest.raises(Exception):
            NMF(bad)
    for bad in [(100, 50), (100,), (100, 50) * 2]:
        with pytest.raises(Exception):
            NMFD(bad)


def test_given_tensor_is_copied_and_trainable_flag():
    W0 = torch.rand(30, 4)
    m = NMF(W=W0, H=(20, 4), trainable_W=False)
    assert m.W.data_ptr() != W0.data_ptr() and torch.equal(m.W.data, W0)
    assert not m.W.requires_grad and m.H.requires_grad
    sd = m.state_dict()
    assert set(sd) == {"W", "H"}


def test_forward_accepts_external_factors_and_autograd():
    m = NMF(W=(30, 4), rank=4)           # H is None: module used as a layer (tests/test_trainer.py:17-18)
    H = torch.rand(7, 4, requires_grad=True)
    out = m(H=H)
    out.sum().backward()
    assert out.shape == (7, 30) and H.grad is not None


# ---- the C-ABI library ---------------------------------------------------------------------------
def test_library_exports_every_declared_symbol():
    header = open(os.path.join(ROOT, "include", "nmf_b200.h")).read()
    declared = set(re.findall(r"\b(nmfb200_[a-z0-9_]+)\s*\(", header))
    declared.discard("nmfb200_ctx")
    assert declared == set(_capi.SIGNATURES), declared ^ set(_capi.SIGNATURES)
    lib = ctypes.CDLL(_capi.LIB_PATH)
    for name in declared:
        assert hasattr(lib, name), name
    assert _capi.load().nmfb200_abi_version() == 1


def test_library_was_built_from_these_sources():
    """The .so that runs (here and on the GPU machine) carries the hash of the sources it was compiled
    from; a stale or foreign binary fails this test instead of silently passing the parity suite."""
    import importlib.util
    spec = importlib.util.spec_from_file_location("nmf_b200_build", os.path.join(ROOT, "pytorch-nmf_b200", "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    info = _capi.build_info()
    assert f"src={mod.source_hash()} " in info, (info, mod.source_hash())
    assert "arch=sm_90a" in info and "nvcc=12." in info


def test_library_rejects_bad_arguments_without_gpu_work():
    lib = _capi.load()
    ctx = ctypes.c_void_p()
    assert lib.nmfb200_nmf_create(None, 0, 4, 4, 2, 0) != 0
    assert lib.nmfb200_nmf_create(ctypes.byref(ctx), 0, 0, 4, 2, 0) != 0
    assert b"positive" in lib.nmfb200_last_error()
    assert lib.nmfb200_nmf_create(ctypes.byref(ctx), 0, 4, 4, 2, 77) != 0
    assert lib.nmfb200_nmf_w_partial_numel(None, 1.0) == -1


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the loud failure on a CUDA-less host")
def test_fit_fails_loudly_without_cuda():
    m = NMF((10, 8), 3)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m.fit(torch.rand(10, 8))


def test_sparse_target_validation_like_reference():
    # nmf.py:329-336: negative values and beta <= 0 are refused for sparse targets before any device work
    m = NMF((10, 8), 3)
    V = torch.rand(10, 8).to_sparse()
    with pytest.raises(ValueError, match="beta <= 0"):
        m.fit(V, beta=0)
    with pytest.raises(AssertionError, match="non-negative"):
        m.fit((-torch.rand(10, 8)).to_sparse())


# ---- fit() host logic against the reference's outputs, with the oracle standing in for the GPU ----
@pytest.mark.parametrize("name", ["nmf_b1_a0_l0", "nmf_b0.5_a0.1_l0.5", "nmf_b3_a0_l0", "nmf_stoprule",
                                  "nmf_frozenW", "nmfd_b1_a0_l0", "nmfd_b0_a0.1_l0.5"])
def test_fit_loop_matches_reference(name):
    c = CASES[name]
    cls, eng = (NMF, OracleNmfEngine) if c["kind"] == "nmf" else (NMFD, OracleNmfdEngine)
    m = cls(W=c["W0"], H=c["H0"], trainable_W=bool(c.get("trainable_W", 1)))
    m._engine_factory = eng            # host-logic test hook (an attribute, not a fit() parameter)
    n_iter = m.fit(c["V"], c["beta"], c["tol"], int(c["max_iter"]), False, c["alpha"], c["l1_ratio"])
    assert n_iter == c["n_iter"]
    assert torch.allclose(m.W.data, c["W"], rtol=5e-5, atol=1e-7)
    assert torch.allclose(m.H.data, c["H"], rtol=5e-5, atol=1e-7)


def test_fit_validation_errors():
    V = torch.rand(12, 9)
    m = NMF(V.shape, 3)
    m._engine_factory = OracleNmfEngine
    Vneg = V.clone(); Vneg[0, 0] = -1
    with pytest.raises(AssertionError, match="non-negative"):
        m.fit(Vneg)
    Vz = V.clone(); Vz[0, 0] = 0
    with pytest.raises(ValueError, match="beta <= 0"):
        m.fit(Vz, beta=0)
    with pytest.raises(RuntimeError, match="does not match"):
        m.fit(torch.rand(5, 5))


def test_fit_returns_niter_plus_one_and_verbose_runs():
    V = torch.rand(20, 10)
    m = NMF(V.shape, 3)
    m._engine_factory = OracleNmfEngine
    assert m.fit(V, 1, float("-inf"), 7, True) == 7
    assert not torch.isnan(m.W).any() and not torch.isnan(m.H).any()


def test_fit_signature_is_the_references():
    import inspect
    sig = inspect.signature(NMF.fit)
    assert list(sig.parameters)[:8] == ["self", "V", "beta", "tol", "max_iter", "verbose", "alpha", "l1_ratio"]   # nmf.py:298-306
    extras = [p for p in sig.parameters.values() if p.kind is inspect.Parameter.KEYWORD_ONLY]
    assert sorted(p.name for p in extras) == ["group", "precision"]


# ---- NMF2D / NMF3D constructors: reference tests/test_nmf.py:72-101 and the docstring examples nmf.py:830-841, :912-923 ----
def test_nmf2d_valid_construct():
    from torchnmf_b200 import NMF2D
    m = NMF2D((2, 5, 30, 20), 4)
    assert m().shape == (2, 5, 30, 20)
    m = NMF2D((1, 1, 33, 50), 16, 3)
    assert m.W.shape == (1, 16, 3, 3) and m.H.shape == (1, 16, 31, 48) and m().shape == (1, 1, 33, 50)
    m = NMF2D((1, 2, 12, 9), 3, (2, 4))
    assert m.W.shape == (2, 3, 2, 4) and m.H.shape == (1, 3, 11, 6)


@pytest.mark.parametrize("Vshape", [(100, 50), (100,), (100, 50) * 6])
def test_nmf2d_invalid_construct(Vshape):
    from torchnmf_b200 import NMF2D
    with pytest.raises(Exception):
        NMF2D(Vshape)


def test_nmf3d_valid_construct():
    from torchnmf_b200 import NMF3D
    m = NMF3D((1, 3, 16, 16, 20), 8, (5, 5, 6))
    assert m.W.shape == (3, 8, 5, 5, 6) and m.H.shape == (1, 8, 12, 12, 15) and m().shape == (1, 3, 16, 16, 20)
    assert NMF3D((2, 4, 6, 7, 8), 2)().shape == (2, 4, 6, 7, 8)


@pytest.mark.parametrize("Vshape", [(100, 50), (100,), (100, 50) * 4])
def test_nmf3d_invalid_construct(Vshape):
    from torchnmf_b200 import NMF3D
    with pytest.raises(Exception):
        NMF3D(Vshape)


def test_convolutive_models_refuse_sparse_targets_like_the_reference():
    """nmf.py:294-295: only NMF derives the sparse update; NMFD / NMF2D / NMF3D raise NotImplementedError."""
    from torchnmf_b200 import NMFD, NMF2D
    V = torch.rand(1, 4, 12).to_sparse()
    with pytest.raises(NotImplementedError):
        NMFD(V.shape, 2, 3).fit(V)
    V = torch.rand(1, 2, 6, 7).to_sparse()
    with pytest.raises(NotImplementedError):
        NMF2D(V.shape, 2, 2).fit(V)


def test_fit_asks_for_the_prefetched_loss_only_when_a_w_update_follows():
    """Host logic of the folded loss (nmfb200_nmf_loss_prefetch_w): every 10th iteration's loss may come out of the next W
    update's pass -- but not the last evaluation of a fit, and not when W is frozen."""
    calls = []

    class Eng(OracleNmfEngine):
        def loss(self, beta):
            calls.append("loss")
            return super().loss(beta)

        def loss_prefetch_w(self, beta):
            calls.append("prefetch")
            return OracleNmfEngine.loss(self, beta)

    torch.manual_seed(0)
    V = torch.rand(20, 15)
    m = NMF(W=torch.rand(15, 3), H=torch.rand(20, 3))
    m._engine_factory = Eng
    assert m.fit(V, 1, float("-inf"), 30) == 30
    assert calls == ["loss", "prefetch", "prefetch", "loss"]          # init, @9, @19, @29 (nothing follows)
    calls.clear()
    m.fit(V, 1, float("-inf"), 25)
    assert calls == ["loss", "prefetch", "prefetch"]
    calls.clear()
    f = NMF(W=torch.rand(15, 3), H=torch.rand(20, 3), trainable_W=False)
    f._engine_factory = Eng
    f.fit(V, 1, float("-inf"), 20)
    assert calls == ["loss", "loss", "loss"]
