"""Sparse-target PLCA on the GPU (csrc/sparse_plca.cu through nmfb200_plca_sparse_*, and `PLCA.fit` on a sparse COO V):

(1) the gradients dW, dHz and the loss of one EM step against float64 at ranks on both sides of every rank-per-lane plan and
    of the 256-wide rank blocks, on a target with empty rows and columns, single-entry rows, a row of 3000 entries and
    explicit zeros;
(2) at R <= 256, dW and dHz bit for bit the beta-1 numerators of the sparse NMF gathers (nmfb200_raw_terms on a
    nmfb200_nmf_set_target_sparse context) on the factor pair (W, Hz): the same rank slots, dot product and ratio per entry;
(3) whole fits against the reference's fixtures (tests/golden/reference_sparse_plca.npz) and against the dense fp32 fit of
    V.to_dense(): the same iteration counts, factors as close to the float64 reference as the dense fp32 fit's;
(4) determinism, frozen factors, host-resident modules and targets;
(5) one fit of a target whose dense form (2^20 x 2^17 fp32, 512 GiB) could not be stored, with the device memory bounded by
    O(nnz + (N + C) R).
"""
import math

import pytest
import torch

from test_sparse_plca import NAMES, alphas, case, sparse_target
from torchnmf_b200 import PLCA
from torchnmf_b200.constants import eps
from torchnmf_b200.engine import CudaSparseNmfEngine, CudaSparsePlcaEngine

pytestmark = pytest.mark.gpu

RANKS = [1, 7, 32, 64, 128, 255, 256, 257, 300, 512, 1024]
N, C = 300, 3000


def _pattern():
    """(rows, cols, vals) of a 300 x 3000 target at ~0.5 %: rows 0-9 and columns 0-4 empty, rows 10-19 one entry each, row 20
    every column from 5 on, 10 % of the stored values explicit zeros."""
    g = torch.Generator().manual_seed(7)
    stored = torch.rand(N, C, generator=g) < 0.005
    stored[:20] = False
    stored[10:20, 5 + torch.arange(10) * 7] = True
    stored[20] = True
    stored[:, :5] = False
    rows, cols = stored.nonzero(as_tuple=True)
    vals = 1.0 + torch.poisson(torch.full((len(rows),), 2.0), generator=g)
    vals[torch.rand(len(rows), generator=g) < 0.1] = 0.0
    return rows, cols, vals


def _problem(R, seed=0):
    rows, cols, vals = _pattern()
    norm = torch.tensor(float(vals.sum()), dtype=torch.float32)
    Vn = torch.sparse_coo_tensor(torch.stack([rows, cols]), vals / norm, (N, C)).coalesce().cuda()
    g = torch.Generator().manual_seed(seed)
    W = torch.rand(C, R, generator=g) + 0.05
    H = torch.rand(N, R, generator=g) + 0.05
    Z = torch.rand(R, generator=g) + 0.1
    Hz = (H / H.sum(0)) * (Z / Z.sum())
    return Vn, (W / W.sum(0)).cuda(), Hz.cuda(), float(norm)


def _reference(Vn, W, Hz, norm):
    """dW, dHz and the loss in float64 from the densified normalised target, and the loss's magnitude."""
    V64, W64, H64 = Vn.to_dense().double().cpu(), W.double().cpu(), Hz.double().cpu()
    q = H64 @ W64.t()
    P = V64 / (q + eps)
    (n, c), v = Vn.indices().cpu(), Vn.values().cpu()
    t = (v * torch.tensor(norm, dtype=torch.float32)).double()            # the fp32 de-normalised target the fit sees
    x = norm * q[n, c]
    lt, lx = t * torch.log(t + eps), t * torch.log(x + eps)
    loss = float(lt.sum() - lx.sum() - t.sum() + norm * q.sum())
    scale = float(lt.abs().sum() + lx.abs().sum() + t.sum() + norm * q.sum())
    return P.t() @ H64, P @ W64, loss, scale


def _close(got, want, rtol):
    return torch.allclose(got, want, rtol=rtol, atol=rtol * float(want.abs().max()))


def _worst(got, want):
    return float(((got - want).abs() / (want.abs() + 1e-5 * want.abs().max())).max())


@pytest.mark.parametrize("R", RANKS)
def test_terms_against_float64(R):
    Vn, W, Hz, norm = _problem(R)
    eng = CudaSparsePlcaEngine(Vn, W, Hz)
    try:
        dW, dHz, loss = eng.plca_terms(Hz, norm)
        dW, dHz, loss = dW.double().cpu(), dHz.double().cpu(), float(loss.item())
        assert eng.loss(norm) == loss                     # the loss alone: the same row-gather pass
        eng.check_health()
    finally:
        eng.close()
    rW, rH, rloss, scale = _reference(Vn, W, Hz, norm)
    assert _close(dW, rW, 1e-5), (R, _worst(dW, rW))
    assert _close(dHz, rH, 1e-5), (R, _worst(dHz, rH))
    assert abs(loss - rloss) <= 1e-6 * scale, (R, loss, rloss, scale)
    assert torch.all(dHz[:10] == 0) and torch.all(dW[:5] == 0)            # documents without words, unused terms
    assert torch.all(dHz[10:21].abs().sum(1) > 0)


@pytest.mark.parametrize("R", [r for r in RANKS if r <= 256])
def test_terms_are_the_sparse_nmf_gathers_bit_for_bit(R):
    Vn, W, Hz, _ = _problem(R)
    eng = CudaSparsePlcaEngine(Vn, W, Hz)
    nmf = CudaSparseNmfEngine(Vn, W, Hz, "f32")
    try:
        dW, dHz = (t.clone() for t in eng.plca_terms(Hz))
        numW, _ = nmf.raw_terms(0, 1.0)
        numH, _ = nmf.raw_terms(1, 1.0)
        assert torch.equal(dW, numW) and torch.equal(dHz, numH)
    finally:
        eng.close()
        nmf.close()


def _module(c, device="cuda"):
    kw = {k: bool(int(c[k])) for k in ("trainable_W", "trainable_H", "trainable_Z")}
    return PLCA(W=c["W0"], H=c["H0"], Z=c["Z0"], **kw).to(device)


@pytest.mark.parametrize("name", NAMES)
def test_fit_matches_reference(name):
    c = case(name)
    m = _module(c)
    n_iter, norm = m.fit(sparse_target(c, torch.float32).cuda(), float(c["tol"]), int(c["iters"]), False, *alphas(c))
    assert m.last_fit_precision == "f32"
    assert n_iter == int(c["n_iter"]) and abs(float(norm) - float(c["norm"])) <= 1e-6 * float(c["norm"])
    for nm in ("W", "H", "Z"):
        got, want = getattr(m, nm).data.double().cpu(), c[nm]
        assert torch.allclose(got, want, rtol=1e-3, atol=1e-5 * float(want.abs().max())), (name, nm, _worst(got, want))


@pytest.mark.parametrize("name", NAMES)
def test_fit_matches_the_dense_fp32_fit(name):
    """The same iteration count and norm as the dense fp32 fit of V.to_dense(); factors within 1e-4 of it relative to the
    factor's largest entry plus the entry (the two sum in different orders, and the EM recursion carries that through to
    the entries far below the factor's largest, whose error relative to themselves reaches 1e-3), and no further from the
    reference's float64 factors than the dense fp32 fit is, up to fp32 rounding."""
    c = case(name)
    V = sparse_target(c, torch.float32).cuda()
    ms, md = _module(c), _module(c)
    ns, norm_s = ms.fit(V, float(c["tol"]), int(c["iters"]), False, *alphas(c))
    nd, norm_d = md.fit(V.to_dense(), float(c["tol"]), int(c["iters"]), False, *alphas(c), precision="f32")
    assert ns == nd and float(norm_s) == float(norm_d)
    for nm in ("W", "H", "Z"):
        got, want, ref = getattr(ms, nm).data, getattr(md, nm).data, c[nm]
        es, ed = (float(((x.double().cpu() - ref).abs() / (ref.abs() + ref.abs().max())).max()) for x in (got, want))
        print(f"SPPLCA dense {name} {nm} worst {_worst(got, want):.3g} vs float64: sparse {es:.3g} dense {ed:.3g}")
        assert _close(got, want, 1e-4), (name, nm, _worst(got, want))
        assert es <= 4 * ed + 1e-6, (name, nm, es, ed)


def test_fits_are_deterministic_and_frozen_factors_stay():
    c = case("poisson")
    V = sparse_target(c, torch.float32).cuda()
    runs = []
    for _ in range(2):
        m = _module(c)
        m.fit(V, float("-inf"), 30)
        runs.append([getattr(m, nm).data.clone() for nm in ("W", "H", "Z")])
    for a, b in zip(*runs):
        assert torch.equal(a, b)
    for frozen in ("W", "H", "Z"):
        kw = {f"trainable_{frozen}": False}
        m = PLCA(W=c["W0"], H=c["H0"], Z=c["Z0"], **kw).cuda()
        before = getattr(m, frozen).data.clone()
        m.fit(V, float("-inf"), 20)
        assert torch.equal(getattr(m, frozen).data, before), frozen


def test_host_module_and_host_target_are_staged():
    c = case("empty")
    m = _module(c, "cpu").double()
    n_iter, norm = m.fit(sparse_target(c, torch.float64), float("-inf"), 20)     # float64 on the host
    md = _module(c)
    nd, _ = md.fit(sparse_target(c, torch.float32).cuda(), float("-inf"), 20)
    assert m.W.device.type == "cpu" and m.W.dtype == torch.float64 and norm.dtype == torch.float64
    assert n_iter == nd
    for nm in ("W", "H", "Z"):
        assert torch.equal(getattr(m, nm).data.float(), getattr(md, nm).data.cpu()), nm


class _Recording(CudaSparsePlcaEngine):
    last = None

    def __init__(self, *a):
        super().__init__(*a)
        self.losses = []
        _Recording.last = self

    def loss(self, norm):
        val = super().loss(norm)
        self.losses.append(val)
        self.bytes = self.device_bytes()
        return val


def test_fit_of_a_target_too_large_to_densify():
    """2^20 x 2^17, 10^7 stored entries, R = 64.  The model's cells start near 1 / (N C) = 7e-12, far below the ratio's eps
    (1.2e-7), which then dominates the EM step as it does the dense fit's; 4096 heavy entries (10^4 each) carry most of the
    mass, so that the step still moves the model toward the target and the loss falls."""
    Nb, Cb, R, nnz = 1 << 20, 1 << 17, 64, 10 ** 7
    g = torch.Generator(device="cuda").manual_seed(0)
    idx = torch.stack([torch.randint(0, Nb, (nnz,), device="cuda", generator=g),
                       torch.randint(0, Cb, (nnz,), device="cuda", generator=g)])
    vals = torch.randint(1, 6, (nnz,), device="cuda", generator=g).float()
    vals[:4096] = 1e4
    V = torch.sparse_coo_tensor(idx, vals, (Nb, Cb))          # uncoalesced: duplicates sum
    torch.manual_seed(0)
    m = PLCA((Nb, Cb), rank=R).cuda()
    m._engine_factory = _Recording
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    n_iter, norm = m.fit(V, float("-inf"), 20)
    peak = torch.cuda.max_memory_allocated()
    eng = _Recording.last
    total = eng.bytes + peak
    bound = 128 * nnz + 64 * (Nb + Cb) * R
    print(f"SPPLCA scale ctx {eng.bytes / 2**20:.1f} MiB torch peak {peak / 2**20:.1f} MiB bound {bound / 2**20:.1f} MiB "
          f"dense {4 * Nb * Cb / 2**30:.0f} GiB losses {eng.losses}")
    assert n_iter == 19 and abs(float(norm) - float(vals.sum())) <= 1e-6 * float(vals.sum())
    assert total <= bound
    assert eng.bytes <= 4 * nnz + 8 * (Nb // 8 + 1) + 8 * R * 2048
    assert all(math.isfinite(x) for x in eng.losses) and all(b < a for a, b in zip(eng.losses, eng.losses[1:]))
