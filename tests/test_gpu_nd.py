"""GPU parity of NMF2D / NMF3D (reference nmf.py:782-942) against reference-generated goldens
(tests/golden/reference_nd.npz, written by `python oracle/make_golden.py --nd` from the real torchnmf 0.3.5) and against the
oracle on seeded shapes.  Module surface -> ctypes -> C ABI (nmfb200_nmfnd_create + the calls that serve every context)."""
import pytest
import torch

from conftest import load_golden
from oracle import mu_oracle as orc
from torchnmf_b200 import NMF2D, NMF3D, NMFD

pytestmark = pytest.mark.gpu
CASES = load_golden("reference_nd.npz")
CLS = {"nmf2d": NMF2D, "nmf3d": NMF3D}


def _close(got, want, rtol, atol_rel):
    atol = atol_rel * float(want.abs().max())
    err = ((got - want).abs() / (rtol * want.abs() + atol)).max().item()
    return err <= 1.0, err


@pytest.mark.parametrize("name", sorted(CASES))
def test_fit_matches_reference_golden(name):
    c = CASES[name]
    m = CLS[c["kind"]](W=c["W0"], H=c["H0"], trainable_W=bool(c.get("trainable_W", 1)),
                       trainable_H=bool(c.get("trainable_H", 1))).cuda()
    n_iter = m.fit(c["V"].cuda(), c["beta"], c["tol"], int(c["max_iter"]), False, c["alpha"], c["l1_ratio"])
    assert m.last_fit_precision == "f32"
    assert n_iter == c["n_iter"]
    for got, want, nm in ((m.W.data.cpu(), c["W"], "W"), (m.H.data.cpu(), c["H"], "H")):
        ok, err = _close(got, want, 1e-3, 1e-5)           # the north-star tolerance
        assert ok, f"{name} {nm}: {err:.3f} x tolerance"
    if not bool(c.get("trainable_H", 1)):
        assert torch.equal(m.H.data.cpu(), c["H0"])


@pytest.mark.parametrize("beta", [0, 1, 2, 2.5])
@pytest.mark.parametrize("shape", [((2, 70, 9, 130), 5, (3, 40)), ((1, 3, 5, 6, 70), 4, (2, 3, 33)), ((1, 2, 4, 40), 3, (4, 1))])
def test_updates_match_oracle_on_seeded_shapes(beta, shape):
    """Tiles that cross the 64-wide output tile and the 32-wide shift chunk on the sliding axis; kernels as long as an
    outer axis; three iterations with penalties, checked against the closed-form oracle."""
    vs, R, K = shape
    B, C, X = vs[0], vs[1], vs[2:]
    torch.manual_seed(sum(vs))
    V = torch.rand(*vs) + (0.01 if beta <= 0 else 0)
    W0 = torch.rand(C, R, *K) + 0.1
    H0 = torch.rand(B, R, *(x - k + 1 for x, k in zip(X, K))) + 0.1
    kind, cls = ("nmf2d", NMF2D) if len(K) == 2 else ("nmf3d", NMF3D)
    W, H, _, losses = orc.fit(V, W0, H0, beta=beta, tol=float("-inf"), max_iter=3, alpha=0.05, l1_ratio=0.3, kind=kind)
    m = cls(W=W0, H=H0).cuda()
    m.fit(V.cuda(), beta, float("-inf"), 3, False, 0.05, 0.3)
    assert _close(m.W.data.cpu(), W, 2e-4, 1e-6)[0]
    assert _close(m.H.data.cpu(), H, 2e-4, 1e-6)[0]


def test_nmf2d_with_unit_outer_axis_equals_nmfd():
    """An NMF2D whose first convolved axis has size 1 is NMFD: same kernels, same bits."""
    torch.manual_seed(5)
    V = torch.rand(2, 9, 1, 80)
    W0, H0 = torch.rand(9, 3, 1, 7), torch.rand(2, 3, 1, 74)
    a = NMF2D(W=W0, H=H0).cuda()
    a.fit(V.cuda(), 1, float("-inf"), 5, precision="f32")
    b = NMFD(W=W0[:, :, 0], H=H0[:, :, 0]).cuda()
    b.fit(V[:, :, 0].cuda(), 1, float("-inf"), 5, precision="f32")
    assert torch.equal(a.W.data[:, :, 0], b.W.data) and torch.equal(a.H.data[:, :, 0], b.H.data)


def test_fit_smoke_like_reference():
    """Reference tests/test_nmf.py:104-120 shape of test for the 2-D / 3-D models: n_iter <= max_iter and no NaN."""
    for cls, vs, k in ((NMF2D, (1, 4, 20, 30), (3, 5)), (NMF3D, (1, 2, 8, 9, 10), 2)):
        V = torch.rand(*vs).cuda()
        m = cls(vs, 3, k).cuda()
        n = m.fit(V, 1, 1e-4, 40)
        assert n <= 40 and not torch.isnan(m.W).any() and not torch.isnan(m.H).any()
