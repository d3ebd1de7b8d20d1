"""NMF2D / NMF3D on the tensor-core sliding GEMMs (csrc/tc_nmfd.cu with outer axes): the plan restated in Python, the case
catalogue of tests/test_nd_tc_plan.py and tests/test_gpu_nd_tc.py, and the float64 restatement and rounding model of the
ND terms.

TEST INFRASTRUCTURE ONLY.  Shapes are (B, C, vdims, R, kdims) as NMF2D / NMF3D take them: V (B, C, *vdims), W (C, R, *kdims),
H (B, R, *(vdims - kdims + 1)).  The last axis slides; the outer ones (X1, X2 / T1, T2 / J1, J2, right-aligned, 1 where a
shape has fewer axes) are the lines the kernels loop over.

The model is tests/tc_model.py's 1-D NMFD model summed over the outer kernel offsets: every contraction of the ND path is a
sum, over (t1, t2), of 1-D sliding contractions between lines (b, j1, j2) of H and lines (b, j1 + t1, j2 + t2) of the target
side.  Its roundings are the 1-D path's (fp16 operand copies with one power-of-two scale each, the centred fp16 ratio tile,
fp32 accumulation), with the term counts of the ND sums:
  * recon      KS = R T1 T2 T products per output element at most;
  * wgrad      K = B J1 J2 Lin products per sum;
  * dgrad      K = C T1 T2 T.
"""
import torch

import tc_model as tcm
from oracle import mu_oracle as orc

KM, KKB, KWIN = 128, 64, 256
INT32_MAX = 2 ** 31 - 1
MAX_GRID_X, MAX_GRID_YZ = 2 ** 31 - 1, 65535


def cdiv(a, b):
    return -(-a // b)


def round_up(a, b):
    return cdiv(a, b) * b


def outer(vdims, kdims):
    """(X1, X2, L), (T1, T2, T) right-aligned."""
    X = (1,) * (3 - len(vdims)) + tuple(vdims)
    K = (1,) * (3 - len(kdims)) + tuple(kdims)
    return X, K


def plan(B, C, vdims, R, kdims):
    """tc_nmfd_plan (csrc/tc_nmfd.cu) in Python: (plan dict, None) or (None, the refusal message)."""
    (X1, X2, L), (T1, T2, T) = outer(vdims, kdims)
    one_d = X1 == X2 == T1 == T2 == 1
    if not (1 <= R <= 256 and 1 <= T <= L):
        return None, "the tensor-core NMFD path needs 1 <= R <= 256 and 1 <= T <= L"
    J1, J2, Lin = X1 - T1 + 1, X2 - T2 + 1, L - T + 1
    X12, T12, J12 = X1 * X2, T1 * T2, J1 * J2
    p = {}
    p["Tp"] = Tp = round_up(T, KKB)
    p["padl"] = round_up(Tp + 136, 8)
    p["Lp"] = round_up(p["padl"] + round_up(L, 2048) + 256 + KWIN + 136, 8)
    p["Lq"] = round_up(round_up(L, 2048) + 1024 + Tp + KKB + KWIN + 8, 8)
    p["Cpad"] = round_up(C, KM)
    lkb, tkb = cdiv(L, KKB), Tp // KKB
    tiles_w, tiles_h = cdiv(C, KM) * R * T12 * cdiv(T, KM), cdiv(Lin, KM) * B * J12
    kb_w, kb_h = B * J12 * lkb, C * T12 * tkb
    for side, kb, tiles in (("w", kb_w, tiles_w), ("h", kb_h, tiles_h)):
        ws = max(1, min(kb // 8, cdiv(132 * 4, tiles)))
        kbs = cdiv(kb, ws)
        p["ws_" + side], p["kbs_" + side] = cdiv(kb, kbs), kbs
    p["kb_w"], p["kb_h"] = kb_w, kb_h
    p["nch"] = cdiv(Lin, 2048)
    p["bslice"] = min(B * X12, MAX_GRID_YZ)
    p["slices"] = cdiv(B * X12, p["bslice"])
    p["hslice"] = min(B * J12, MAX_GRID_YZ)
    p["hslices"] = cdiv(B * J12, p["hslice"])
    p["dgrad_rblocks"] = cdiv(R, KM)
    p["prep_w"] = (C, 1, 1)
    p["prep_h"] = (B * R * J12 * p["nch"], 1, 1)
    p["recon"] = (cdiv(L, KM), cdiv(C, KM), p["bslice"])
    p["wgrad"] = (cdiv(C, KM), R * T12 * cdiv(T, KM), p["ws_w"])
    p["dgrad"] = (cdiv(Lin, KM), p["ws_h"], p["hslice"])
    p["loss_blocks"] = p["recon"][0] * p["recon"][1] * B * X12

    def fits(g):
        return 1 <= g[0] <= MAX_GRID_X and 1 <= g[1] <= MAX_GRID_YZ and 1 <= g[2] <= MAX_GRID_YZ
    if not fits(p["wgrad"]):
        return None, ("the tensor-core NMFD wgrad grid needs R ceil(T / 128) <= 65535" if one_d else
                      "the tensor-core NMFD wgrad grid needs R T1 T2 ceil(T / 128) <= 65535")
    if not all(fits(p[k]) for k in ("prep_w", "prep_h", "recon", "dgrad")):
        return None, "a tensor-core NMFD grid passes the CUDA grid limits"
    if one_d:
        if B * C + KM > INT32_MAX:
            return None, "the tensor-core NMFD path needs B C < 2^31 - 128 (TMA row coordinate)"
        if max(kb_w, kb_h, p["loss_blocks"], p["Lp"], p["Lq"], p["Cpad"] * R) > INT32_MAX:
            return None, "a tensor-core NMFD block or k-block count passes 2^31 - 1"
        return p, None
    nd = "the tensor-core NMF2D / NMF3D path needs "
    checks = [
        (B * X12 * C + KM, nd + "B X1 X2 C < 2^31 - 128 (TMA row coordinate of the ratio tile)"),
        (kb_w, nd + "B J1 J2 ceil(L / 64) < 2^31 (wgrad k-blocks)"),
        (kb_h, nd + "C T1 T2 Tp / 64 < 2^31 (dgrad k-blocks)"),
        (R * T12 * Tp, nd + "R T1 T2 Tp < 2^31 (kernel copy pitch, recon k-blocks)"),
        (p["Cpad"] * R, nd + "ceil(C / 128) 128 R < 2^31 (dgrad rows)"),
        (p["loss_blocks"], nd + "fewer than 2^31 recon-loss partials"),
        (max(p["Lp"], p["Lq"]), nd + "row pitches below 2^31"),
    ]
    for v, msg in checks:
        if v > INT32_MAX:
            return None, msg
    return p, None


def recon_kblocks(C, vdims, R, kdims, x1, x2):
    """k-blocks of the recon CTA of target line (x1, x2): R x (valid t1) x (valid t2) x Tp / 64."""
    (X1, X2, L), (T1, T2, T) = outer(vdims, kdims)
    J1, J2 = X1 - T1 + 1, X2 - T2 + 1
    n1 = min(T1 - 1, x1) - max(0, x1 - J1 + 1) + 1
    n2 = min(T2 - 1, x2) - max(0, x2 - J2 + 1) + 1
    return R * n1 * n2 * (round_up(T, KKB) // KKB), n1, n2


# ---- the catalogue: each case named for what it covers --------------------------------------------------------------------
CASES = {
    "border-2d":          (1, 5, (6, 40), 3, (3, 8)),             # outer X = 6, T = 3: lines 0, 1, 4, 5 meet a border
    "border-3d":          (1, 4, (5, 4, 30), 2, (2, 3, 5)),       # NMF3D: borders in both outer axes
    "x-eq-k":             (1, 6, (3, 50), 4, (3, 7)),             # J1 = 1: every target line meets both borders
    "t1-1":               (2, 7, (5, 60), 3, (1, 9)),             # T1 = 1, B = 2
    "t-above-128":        (1, 3, (3, 300), 2, (2, 150)),          # two blocks of 128 shifts, Tp = 192
    "c-ragged":           (1, 130, (3, 70), 5, (2, 6)),           # C = 130: a second channel tile of 2 rows
    "single-channel":     (1, 1, (33, 50), 16, (3, 3)),           # the reference's NMF2D((1, 1, 33, 50), ...) shape
    "r1":                 (1, 9, (4, 80), 1, (2, 16)),
    "r129":               (1, 20, (3, 40), 129, (2, 2)),          # a second dgrad launch of one component
    "r256":               (1, 12, (3, 32), 256, (2, 4)),          # two full dgrad launches
    "b3":                 (3, 10, (4, 50), 4, (2, 5)),
    "split-short-last":   (2, 43, (6, 8, 60), 2, (2, 2, 3)),      # NMF3D: ws_w, ws_h > 1, both with a short last split
}


def covers(cases=CASES):
    """What the cases reach, as a set of branch names (tests/test_nd_tc_plan.py asserts every one)."""
    got = set()
    for B, C, vd, R, kd in cases.values():
        (X1, X2, L), (T1, T2, T) = outer(vd, kd)
        J1, J2 = X1 - T1 + 1, X2 - T2 + 1
        for ax, (X, K, J) in (("x1", (X1, T1, J1)), ("x2", (X2, T2, J2))):
            if K > 1 and any(min(K - 1, x) - max(0, x - J + 1) + 1 < K for x in range(X)):
                got.add("border-" + ax)
            if K > 1 and J == 1:
                got.add("j1-axis")
        got.add("t1-1" if T1 == 1 else "t1-gt-1")
        if T > 128:
            got.add("t-above-128")
        if C % 128:
            got.add("c-ragged")
        if R in (1, 129, 256):
            got.add(f"r{R}")
        if B > 1:
            got.add("b-gt-1")
        if len(vd) == 3:
            got.add("ndim-3")
        p, _ = plan(B, C, vd, R, kd)
        for s in ("w", "h"):
            ws, kbs, kb = p["ws_" + s], p["kbs_" + s], p["kb_" + s]
            if ws > 1 and kb - (ws - 1) * kbs < kbs:
                got.add("split-short-last-" + s)
    return got


BRANCHES = {"border-x1", "border-x2", "j1-axis", "t1-1", "t1-gt-1", "t-above-128", "c-ragged", "r1", "r129", "r256",
            "b-gt-1", "ndim-3", "split-short-last-w", "split-short-last-h"}


def data(B, C, vdims, R, kdims, seed):
    """Seeded factors bounded away from zero (as tests/test_gpu_tc_terms.py's _nmfd_data)."""
    g = torch.Generator().manual_seed(seed)
    J = tuple(x - k + 1 for x, k in zip(vdims, kdims))
    V = torch.rand(B, C, *vdims, generator=g) + 0.1
    W = torch.rand(C, R, *kdims, generator=g) + 0.1
    H = torch.rand(B, R, *J, generator=g) + 0.1
    return V, W, H


# ---- float64 restatement and model --------------------------------------------------------------------------------------
def _as5(x):
    """(B or C, R or C, *outer, last) -> 5-D with the outer axes right-aligned to (X1, X2)."""
    return x.reshape(x.shape[0], x.shape[1], *((1,) * (5 - x.dim())), *x.shape[2:])


def _lines(x):
    """(B, R, J1, J2, n) -> (B J1 J2, R, n): the lines as a batch of 1-D rows."""
    B, R, J1, J2, n = x.shape
    return x.permute(0, 2, 3, 1, 4).reshape(B * J1 * J2, R, n)


def _unlines(y, B, J1, J2):
    n, R, m = y.shape
    return y.reshape(B, J1, J2, R, m).permute(0, 3, 1, 2, 4)


def reconstruct(H, W):
    """S[b, c, x] = sum_{r, t} W[c, r, t] H[b, r, x - t]: tc_model.nmfd_reconstruct over the lines, summed over (t1, t2)."""
    H5, W5 = _as5(H), _as5(W)
    B, R, J1, J2, Lin = H5.shape
    C, _, T1, T2, T = W5.shape
    out = torch.zeros(B, C, J1 + T1 - 1, J2 + T2 - 1, Lin + T - 1, dtype=H.dtype, device=H.device)
    for t1 in range(T1):
        for t2 in range(T2):
            s = tcm.nmfd_reconstruct(_lines(H5), W5[:, :, t1, t2])
            out[:, :, t1:t1 + J1, t2:t2 + J2] += _unlines(s, B, J1, J2)
    return out.reshape(B, C, *(j + k - 1 for j, k in zip(H.shape[2:], W.shape[2:])))


def grad_w(G, H, kdims):
    """gW[c, r, t] = sum_{b, j} G[b, c, j + t] H[b, r, j]."""
    G5, H5 = _as5(G), _as5(H)
    B, R, J1, J2, Lin = H5.shape
    (T1, T2, T) = outer((1,) * len(kdims), kdims)[1]
    gW = torch.zeros(G.shape[1], R, T1, T2, T, dtype=H.dtype, device=H.device)
    for t1 in range(T1):
        for t2 in range(T2):
            gW[:, :, t1, t2] = tcm.nmfd_grad_w(_lines(G5[:, :, t1:t1 + J1, t2:t2 + J2]), _lines(H5), T)
    return gW.reshape(G.shape[1], R, *kdims)


def grad_h(G, W, jdims):
    """gH[b, r, j] = sum_{c, t} W[c, r, t] G[b, c, j + t]."""
    G5, W5 = _as5(G), _as5(W)
    C, R, T1, T2, T = W5.shape
    B = G.shape[0]
    (J1, J2, Lin) = outer(jdims, (1,) * len(jdims))[0]
    gH = torch.zeros(B, R, J1, J2, Lin, dtype=W.dtype, device=W.device)
    for t1 in range(T1):
        for t2 in range(T2):
            gH += _unlines(tcm.nmfd_grad_h(_lines(G5[:, :, t1:t1 + J1, t2:t2 + J2]), W5[:, :, t1, t2], Lin), B, J1, J2)
    return gH.reshape(B, R, *jdims)


class NdModel:
    """NMF2D / NMF3D on the fp16 sliding-GEMM kernels at beta 1 (rounding=False: exact float64)."""

    def __init__(self, V, W, H, rounding=True):
        self.rounding = rounding
        self.V, self.W, self.H = V.double(), W.double(), H.double()
        self.Wq = tcm.operand(W, False, rounding)[0]
        self.Hq = tcm.operand(H, False, rounding)[0]
        dims = lambda x: [d for d in range(x.dim()) if d != 1]
        self.cs_w, self.cs_h = self.W.sum(dims(W)), self.H.sum(dims(H))
        self.kappa = float(self.V.sum()) / float(self.cs_w @ self.cs_h)
        self.S = reconstruct(self.Hq, self.Wq)
        self.KS = W[0].numel()                       # R T1 T2 T: terms of one recon sum at most

    def raw_terms(self, which, nchunks=1):
        """(numerator, denominator (R,), bar on |kernel - model| of the numerator) of the W (0) or H (1) update."""
        kdims, jdims = tuple(self.W.shape[2:]), tuple(self.H.shape[2:])
        P = self.V / (self.S + tcm.EPS)
        kap = self.kappa if self.rounding else 0.0
        p = tcm.ratio_exp(self.kappa)
        tile = tcm._round_tile(P - kap, p, self.rounding)
        flips = tcm.flip_ulps(P - kap, p, tcm.U * (tcm.KSTEP_ULP * tcm.ksteps(self.KS) + 3) * P)
        if which == 0:
            contract, other, cs = (lambda G, X: grad_w(G, X, kdims)), self.Hq, self.cs_h
            K = self.H.shape[0] * self.H[0, 0].numel()              # B J1 J2 Lin
        else:
            contract, other, cs = (lambda G, X: grad_h(G, X, jdims)), self.Wq, self.cs_w
            K = self.W.shape[0] * self.W[0, 0].numel()              # C T1 T2 T
        shape = (1, -1) + (1,) * (self.V.dim() - 2)
        num = contract(tile, other) + kap * cs.view(shape)
        A, Bv = contract(tile.abs(), other), contract(P, other)
        bar = tcm.U * (tcm.KSTEP_ULP * tcm.ksteps(K) * A + 2 * (tcm.KSTEP_ULP * tcm.ksteps(self.KS) + 3) * Bv
                       + (nchunks + 1) * A + (kap * cs).abs().view(shape)) + tcm._spread(flips, other, contract)
        return num, cs, bar

    def loss(self):
        """(KL loss, bar on |kernel - model|, sum of the absolute values of the summed terms)."""
        V, x = self.V, self.S
        cross = V * (x + tcm.EPS).log()
        val = (V * (V + tcm.EPS).log()).sum() - cross.sum() - V.sum() + x.sum()
        terms = (V * (V + tcm.EPS).log()).abs().sum() + cross.abs().sum() + V.sum() + x.sum()
        rel_s = tcm.U * (tcm.KSTEP_ULP * tcm.ksteps(self.KS) + 2)
        bar = rel_s * (V.sum() + x.sum()) + 64 * tcm.U * terms
        return float(val), float(bar), float(terms)


def exact_terms(V, W, H, which):
    """float64 (numerator, denominator) of one beta-1 update through the oracle's ND contractions (oracle/mu_oracle.py)."""
    V, W, H = V.double(), W.double(), H.double()
    P = orc.phi(V, orc.nmfnd_reconstruct(H, W), 1)[0]
    dims = lambda x: [d for d in range(x.dim()) if d != 1]
    if which == 0:
        return orc.nmfnd_grad_w(P, H, tuple(W.shape[2:])), H.sum(dims(H))
    return orc.nmfnd_grad_h(P, W, tuple(H.shape[2:])), W.sum(dims(W))


def exact_loss(V, W, H):
    return float(orc.beta_div(orc.nmfnd_reconstruct(H.double(), W.double()), V.double(), 1))


RTOL64 = tcm.RTOL64["f16"]


def splits(B, C, vdims, R, kdims):
    p, why = plan(B, C, vdims, R, kdims)
    assert why is None, why
    return p["ws_w"], p["ws_h"]
