"""Float64 model of what the tensor-core kernels round (csrc/tc_nmf.cu, csrc/tc_nmfd.cu), and nothing of how they schedule.

TEST INFRASTRUCTURE ONLY.  Every function takes fp32 factors / targets on any device and works in float64 there.  With
`rounding=False` the model is the exact float64 arithmetic of the oracle (oracle/mu_oracle.py; tests/test_tc_model.py pins
that); with `rounding=True` it applies, at the exact inputs, every rounding the kernels apply:

  * operand copies: fp16(x 2^a), a = 14 - frexp_exponent(max x) (pow2_exp_for, pow2_exp14); in split mode
    hi = fp16(x 2^a) and lo = fp16(x 2^a - hi) at the same scale (tc_finish_kernel).  The NMF target gets its own copy
    V16 with the exponent of max(V); the NMFD kernels read V in fp32.
  * S = the product of the rounded operands: fast hi hi^T; split hi hi^T + lo hi^T + hi lo^T (the three wgmma terms).
  * beta 1: P = V16 / (S + eps), kappa = sum(V) / <colsum W, colsum H>, the ratio tile fp16((P - kappa) 2^p) with
    kappa 2^p in [2^-4, 2^-3) (publish_scales, fold_colsum_kernel), numerator = tile G + kappa colsum(G) with G the
    rounded operand (hi + lo in split mode: O = P Ghi + P Glo).
  * beta 2: the residual tile fp16((V16 - kappa S) 2^pe), pe = -rint(log2 mean V); numerator = tile G + kappa F (G^T G),
    denominator F (G^T G), both Gram products of the fp32 factors.
  * other betas: from the hi halves only, Pn = fp16(V16 x^(beta-2) 2^en), Pp = fp16(x^(beta-1) 2^ed), x = S + eps, with
    the exponents of publish_scales; numerator Pn Ghi, denominator Pp Ghi.
  * losses: the kernels' formulas with S and V16 in place of WH and V where the kernels use them.

Every term also comes with `bar`, the per-element bound of |kernel - model| under this error model (u = 2^-23, one fp32
ulp):
  * wgmma adds each 16-term k-step of exact fp16 products into the fp32 accumulator the way NVIDIA tensor cores are
    documented to (Fasi, Higham, Mikaitis, Pranesh, "Numerical behavior of NVIDIA tensor cores", PeerJ Comput. Sci. 7,
    e330, 2021): the products and the accumulator are aligned to the largest exponent among them and the bits shifted
    out are truncated.  Each of the 16 products then loses less than one ulp of that exponent, half an ulp on average,
    always in the same direction: KSTEP_ULP = 8 ulp per step (16 x 1/2; the worst case, 17, is not reached by products
    with independent low bits).  KSTEP_ULP u ceil(K / 16) A for the second MMA, A = sum |tile| |G| bounding every
    partial sum.  (The H100 measured ~5 ulp per step on these tests; an earlier bar of 2 ulp per step was too tight.)
  * S carries the same error over its KS = terms x padded rank products; x' = S c1 + c2, rcp.approx and the product with
    V16 add one ulp each: P is off by d = u (KSTEP_ULP ceil(KS / 16) + 3) relative, which moves the sum by d B,
    B = sum |P| |G|.
  * the ratio tile is rounded to fp16 from that perturbed P: an entry whose exact value lies within d |P| 2^p of a rounding
    midpoint may round to the neighbouring fp16 value, one fp16 ulp away.  The chance of that is proportional to d, so
    the expected sum of these steps is another d B; which of the flagged entries (those within reach of a midpoint,
    found entry by entry) actually step is left to chance: 4 sqrt(sum over them of (ulp G)^2) bounds that spread at
    4 sigma, and is the whole difference where a sum has a single flagged term.
  * the fp32 chunk sums and the kappa colsum addition: u ((nchunks + 1) A + |kappa colsum|).
"""
import json
import math

import torch

EPS = float(torch.finfo(torch.float32).eps)
U = 2.0 ** -23
F16_MAX = 65504.0
KSTEP_ULP = 8


def pow2_exp(mx):
    """Operand exponent a with mx 2^a in [2^13, 2^14); 0 for an all-zero / non-finite maximum."""
    mx = float(mx)
    if not (mx > 0) or not math.isfinite(mx):
        return 0
    return 14 - math.frexp(mx)[1]


def ratio_exp(kappa):
    """Ratio-tile exponent p with kappa 2^p in [2^-4, 2^-3)."""
    kappa = float(kappa)
    if not (kappa > 0) or not math.isfinite(kappa):
        return 0
    return -3 - math.frexp(kappa)[1]


def f16(x):
    """fp16 round-to-nearest-even of the fp32 value the kernel holds, saturating at the fp16 maximum (pack_f16x2_sat)."""
    return x.float().clamp(-F16_MAX, F16_MAX).half().double()


def operand(x, split, rounding=True):
    """(hi, lo) of the fp16 operand copy of x in true scale; lo is zero in fast mode, (x, 0) without rounding."""
    x = x.double()
    if not rounding:
        return x, torch.zeros_like(x)
    a = pow2_exp(x.max())
    xs = x * 2.0 ** a
    hi = f16(xs)
    lo = f16(xs - hi) if split else torch.zeros_like(xs)
    return hi * 2.0 ** -a, lo * 2.0 ** -a


def target(V, rounding=True):
    """The NMF kernels' fp16 copy of V (one exponent from max V), true scale."""
    V = V.double()
    if not rounding:
        return V
    e = pow2_exp(V.max())
    return f16(V * 2.0 ** e) * 2.0 ** -e


def _spread(flips, G, contract=torch.matmul):
    """Bound on the tile's possible one-ulp steps (flip_ulps) through the contraction with G: 4 sigma of their sum, or
    all of them in one direction where that is smaller (sums with one or a few flagged terms)."""
    return torch.minimum(4 * contract(flips * flips, G * G).sqrt(), contract(flips, G))


def ksteps(k):
    return math.ceil(k / 16)


def _round_tile(x, e, rounding):
    return f16(x * 2.0 ** e) * 2.0 ** -e if rounding else x


def flip_ulps(x, e, delta):
    """Per entry of the tile fp16(x 2^e), in true scale: the fp16 ulp by which it may differ from the model's rounding when
    the kernel's value is off by up to delta (true scale), 0 where x is farther than delta from every rounding midpoint."""
    xs = (x * 2.0 ** e).float().double()
    r = f16(xs)
    tiny = 2.0 ** -24                                   # fp16 subnormal spacing
    def ulp(v):
        ex = torch.frexp(v.abs().clamp_min(2.0 ** -14))[1].double()
        return torch.maximum(torch.exp2(ex - 11), torch.full_like(v, tiny))
    below = xs.abs() < r.abs()                          # the midpoint between r and its smaller neighbour is nearer
    u_side = torch.where(below, ulp(r.abs() * (1 - 2.0 ** -12)), ulp(r))
    dist = u_side / 2 - (xs - r).abs()
    return torch.where(dist <= delta * 2.0 ** e, u_side, torch.zeros_like(xs)) * 2.0 ** -e


class NmfModel:
    """Dense NMF, V (N, C) ~ H W^T, in the precision mode "f16" or "f16_split" (rounding=False: exact float64)."""

    def __init__(self, V, W, H, precision, rounding=True):
        self.rounding = rounding
        self.split = precision == "f16_split"
        self.R = W.shape[1]
        self.Rp = 64 if self.R <= 64 else 128
        self.V, self.W, self.H = V.double(), W.double(), H.double()
        self.Vq = target(V, rounding)
        self.Wh, self.Wl = operand(W, self.split, rounding)
        self.Hh, self.Hl = operand(H, self.split, rounding)
        self.cells = V.numel()
        self.dot = float(self.W.sum(0) @ self.H.sum(0))
        self.kappa = float(self.V.sum()) / self.dot

    def _orient(self, which):
        """(F hi, F lo, G hi, G lo, target rows x contracted columns, F fp32, G fp32) of the W (0) or H (1) update."""
        if which == 0:
            return self.Wh, self.Wl, self.Hh, self.Hl, self.Vq.t(), self.W, self.H
        return self.Hh, self.Hl, self.Wh, self.Wl, self.Vq, self.H, self.W

    def product(self, which, hi_only=False):
        """S = F G^T from the rounded operands, as the first MMA forms it, and the number of its k-steps' terms."""
        Fh, Fl, Gh, Gl = self._orient(which)[:4]
        S = Fh @ Gh.t()
        if self.split and not hi_only:
            S = S + Fl @ Gh.t() + Fh @ Gl.t()
            return S, 3 * self.Rp
        return S, self.Rp

    def raw_terms(self, which, beta, nchunks=1):
        """(numerator, denominator, bar on |kernel - model| of the numerator, the same for the denominator or None where
        it is not a contraction) of one update, before the ratio stage."""
        Fh, Fl, Gh, Gl, Vm, F32, G32 = self._orient(which)
        K = Vm.shape[1]
        if beta == 1 or beta == 2:
            S, KS = self.product(which)
            G = Gh + Gl
        else:
            S, KS = self.product(which, hi_only=True)
            G = Gh
        if beta == 1:
            P = Vm / (S + EPS)
            kap = self.kappa if self.rounding else 0.0
            p = ratio_exp(self.kappa)
            tile = _round_tile(P - kap, p, self.rounding)
            colsum = G32.sum(0)
            num = tile @ G + kap * colsum
            A, B = tile.abs() @ G, P @ G
            extra = kap * colsum
            den = colsum
            flip = _spread(flip_ulps(P - kap, p, U * (KSTEP_ULP * ksteps(KS) + 3) * P), G)
        elif beta == 2:
            gram = G32.t() @ G32
            den = F32 @ gram
            kap = self.kappa if self.rounding else 0.0
            pe = -round(math.log2(float(self.V.sum()) / self.cells))
            tile = _round_tile(Vm - kap * S, pe, self.rounding)
            num = tile @ G + kap * den
            A, B = tile.abs() @ G, (kap * S) @ G
            extra = kap * den
            flip = _spread(flip_ulps(Vm - kap * S, pe, U * (KSTEP_ULP * ksteps(KS) + 3) * kap * S), G)
        else:
            x = S + EPS
            Pn, Pp = Vm * x.pow(beta - 2), x.pow(beta - 1)
            lx = math.log2(self.dot / self.cells)
            lv = math.log2(float(self.V.sum()) / self.cells)
            en, ed = -round(lv + (beta - 2) * lx), -round((beta - 1) * lx)
            num = _round_tile(Pn, en, self.rounding) @ G
            den = _round_tile(Pp, ed, self.rounding) @ G
            # both sums are all-positive (A = the sum itself); x^g carries |g| times the relative error of S, the
            # pow / log2 / exp2 approximations a few ulp more
            dn = U * (KSTEP_ULP * ksteps(KS) + 3) * (abs(beta - 2) + 1)
            dd = U * (KSTEP_ULP * ksteps(KS) + 3) * (abs(beta - 1) + 1)
            bar = U * (KSTEP_ULP * ksteps(K) + nchunks + 1) * num + 2 * dn * num + _spread(flip_ulps(Pn, en, dn * Pn), G)
            dbar = U * (KSTEP_ULP * ksteps(K) + nchunks + 1) * den + 2 * dd * den + _spread(flip_ulps(Pp, ed, dd * Pp), G)
            return num, den, bar, dbar
        bar = U * (KSTEP_ULP * ksteps(K) * A + 2 * (KSTEP_ULP * ksteps(KS) + 3) * B + (nchunks + 1) * A + extra.abs())
        return num, den, bar + flip, None

    def loss(self, beta, fold=False):
        """(loss, bar on |kernel - model|, sum of the absolute values of the summed terms) at the current factors."""
        S, KS = self.product(0 if fold else 1)
        Vq = self.Vq.t() if fold else self.Vq
        V = self.V.t() if fold else self.V
        rel_s = U * (KSTEP_ULP * ksteps(KS) + 2)    # relative error of S (accumulation, x = S c1 + c2)
        if beta == 2:
            d = Vq - S
            val = 0.5 * (d * d).sum()
            terms = 0.5 * (d * d).sum() + (d.abs() * S).sum()
            bar = rel_s * (d.abs() * S).sum() + 64 * U * terms
            return float(val), float(bar), float(terms)
        x = S + EPS
        if beta == 1:
            cross = Vq * x.log()
            val = (V * (V + EPS).log()).sum() - V.sum() - cross.sum() + S.sum()
            terms = (V * (V + EPS).log()).abs().sum() + V.sum() + cross.abs().sum() + S.sum()
            # __log2f: ~2^-22 absolute per element, on top of the relative error of S in log(x) and in sum S
            bar = rel_s * (Vq.sum() + S.sum()) + 2.0 ** -21 * Vq.sum() + 64 * U * terms
            return float(val), float(bar), float(terms)
        if beta == 0:
            a, b = (Vq + EPS) / x, x.log()
            vb = (V + EPS).log()
            val = a.sum() - vb.sum() + b.sum() - V.numel()
            terms = a.sum() + vb.abs().sum() + b.abs().sum() + V.numel()
            bar = rel_s * (a.sum() + x.numel()) + 2.0 ** -21 * x.numel() + 64 * U * terms
            return float(val), float(bar), float(terms)
        t, tq = (V + EPS, Vq + EPS) if beta < 0 else (V, Vq)
        a, b = tq * x.pow(beta - 1), x.pow(beta)
        val = (t.pow(beta).sum() + (beta - 1) * b.sum() - beta * a.sum()) / (beta * (beta - 1))
        terms = (t.pow(beta).sum() + abs(beta - 1) * b.sum() + abs(beta) * a.sum()) / abs(beta * (beta - 1))
        g = max(abs(beta), abs(beta - 1))
        bar = (rel_s * g + 2.0 ** -20 * g) * terms + 64 * U * terms
        return float(val), float(bar), float(terms)


def nmfd_reconstruct(H, W):
    """S[b, c, l] = sum_{r,t} W[c, r, t] H[b, r, l - t] (on the inputs' device)."""
    B, R, Lin = H.shape
    C, _, T = W.shape
    out = torch.zeros(B, C, Lin + T - 1, dtype=H.dtype, device=H.device)
    for t in range(T):
        out[:, :, t:t + Lin] += torch.matmul(W[:, :, t], H)
    return out


def nmfd_grad_w(G, H, T):
    B, R, Lin = H.shape
    gW = torch.zeros(G.shape[1], R, T, dtype=H.dtype, device=H.device)
    for t in range(T):
        gW[:, :, t] = torch.matmul(G[:, :, t:t + Lin], H.transpose(1, 2)).sum(0)
    return gW


def nmfd_grad_h(G, W, Lin):
    C, R, T = W.shape
    gH = torch.zeros(G.shape[0], R, Lin, dtype=W.dtype, device=W.device)
    for t in range(T):
        gH += torch.matmul(W[:, :, t].t(), G[:, :, t:t + Lin])
    return gH


class NmfdModel:
    """1-D NMFD, V (B, C, L) ~ sum_t W[:, :, t] H shifted by t, on the fp16 sliding-GEMM kernels (beta 1)."""

    def __init__(self, V, W, H, rounding=True):
        self.rounding = rounding
        self.V, self.W, self.H = V.double(), W.double(), H.double()
        self.Wq = operand(W, False, rounding)[0]
        self.Hq = operand(H, False, rounding)[0]
        self.cs_w, self.cs_h = self.W.sum((0, 2)), self.H.sum((0, 2))
        self.kappa = float(self.V.sum()) / float(self.cs_w @ self.cs_h)
        self.S = nmfd_reconstruct(self.Hq, self.Wq)
        self.KS = W.shape[1] * W.shape[2]             # terms of one recon sum (zero-padded shifts add nothing)

    def raw_terms(self, which, nchunks=1):
        """(numerator, denominator (R,), bar on |kernel - model| of the numerator) of the W (0) or H (1) update."""
        B, C, L = self.V.shape
        T, Lin = self.W.shape[2], self.H.shape[2]
        P = self.V / (self.S + EPS)
        kap = self.kappa if self.rounding else 0.0
        p = ratio_exp(self.kappa)
        tile = _round_tile(P - kap, p, self.rounding)
        flips = flip_ulps(P - kap, p, U * (KSTEP_ULP * ksteps(self.KS) + 3) * P)
        if which == 0:
            # K = the nonzero products of one sum (the Toeplitz rows are zero outside the Lin values of H)
            contract, other, cs, K = (lambda G, X: nmfd_grad_w(G, X, T)), self.Hq, self.cs_h, B * Lin
        else:
            contract, other, cs, K = (lambda G, X: nmfd_grad_h(G, X, Lin)), self.Wq, self.cs_w, C * T
        shape = (1, -1, 1)
        num = contract(tile, other) + kap * cs.view(shape)
        A, Bv = contract(tile.abs(), other), contract(P, other)
        bar = U * (KSTEP_ULP * ksteps(K) * A + 2 * (KSTEP_ULP * ksteps(self.KS) + 3) * Bv + (nchunks + 1) * A
                   + (kap * cs).abs().view(shape)) + _spread(flips, other, contract)
        return num, cs, bar

    def loss(self):
        """(KL loss, bar on |kernel - model|, sum of the absolute values of the summed terms)."""
        V, x = self.V, self.S
        cross = V * (x + EPS).log()
        val = (V * (V + EPS).log()).sum() - cross.sum() - V.sum() + x.sum()
        terms = (V * (V + EPS).log()).abs().sum() + cross.abs().sum() + V.sum() + x.sum()
        rel_s = U * (KSTEP_ULP * ksteps(self.KS) + 2)
        # logf / fp32 per-16-element partial sums: a few ulp of each term
        bar = rel_s * (V.sum() + x.sum()) + 64 * U * terms
        return float(val), float(bar), float(terms)

# ---- bars and plans shared by the term tests (tests/test_gpu_tc_terms.py) and the call sequences (tests/sequence_cases.py) ----
RTOL64 = {"f16": 1.25e-3, "f16_split": 2.5e-4}            # the bars of tests/test_gpu_tc_terms.py (its docstring)
LOSS_RELS = {"f16": 2.0 ** -11, "f16_split": 2.0 ** -20}
# The model bar must stay below the float64 bar, so that a kernel within the model bar of the model passes the float64 bar
# by construction (tests/test_tc_model.py checks that on the CPU).  It is not 5x below it everywhere: the split mode's is
# dominated by the truncation of S over up to 24 k-steps of 3 x 128 products (2 x 195 ulp = 4.6e-5 relative), the
# sliding GEMMs' by the possible one-ulp steps of the ratio tile in sums with few terms.  Each case reports the ratio.
# What the model bar can see is checked directly instead: on STRUCT_CASES each of the three split terms, dropped, misses
# the model by more than twice the bar (tests/test_tc_model.py).
TIGHTER = 1.0


def cdiv(a, b):
    return -(-a // b)


def plan(Mr, Nc, num_sms, TN):
    """make_plan (csrc/tc_nmf.cu): (row blocks, tiles, chunks, tiles per chunk)."""
    rb, tiles = cdiv(Mr, 128), cdiv(Nc, TN)
    best, best_eff = 1, -1.0
    for nch in range(1, min(tiles, 64) + 1):
        tpc = cdiv(tiles, nch)
        if tpc * TN < 512 and nch > 1:
            break
        if cdiv(tiles, tpc) != nch:
            continue
        items = rb * nch
        eff = items / (cdiv(items, num_sms) * num_sms)
        if eff > best_eff + 0.03:
            best_eff, best = eff, nch
        if best_eff >= 0.97:
            break
    return rb, tiles, best, cdiv(tiles, best)


def tn(prec, R):
    return 64 if (prec == "f16_split" and R > 64) else 128


def _report(**kw):
    print("TCTERMS " + json.dumps(kw))


def check_terms(tag, got, model, bar, exact, rtol64):
    """got / model / bar / exact: float64 on one device.  Asserts both bars and the tightness of the model bar."""
    got, model, bar, exact = (t.double().cpu() for t in (got, model, bar, exact))
    scale = exact.abs()
    tight = float((bar / scale).max())
    e_model = float(((got - model).abs() / bar).max())
    e64 = float(((got - exact).abs() / scale).max())
    _report(case=tag, model_err_over_bar=e_model, err64=e64, bar64=rtol64, model_bar_rel=tight)
    assert tight * TIGHTER < rtol64, f"{tag}: the model bar ({tight:.2e} relative) is not below {rtol64:.1e}"
    assert e_model <= 1.0, f"{tag}: {e_model:.2f} x the model bar"
    assert e64 <= rtol64, f"{tag}: relative error {e64:.2e} against float64 > {rtol64:.1e}"
    return max(e_model, e64 / rtol64)


def check_loss(tag, got, model, exact, prec, beta):
    val, bar, terms = model
    g = max(1.0, abs(beta), abs(beta - 1))
    bar64 = (LOSS_RELS[prec] * g + 2.0 ** -12) * terms
    e_model, e64 = abs(got - val) / bar, abs(got - exact) / bar64
    _report(case=tag, model_err_over_bar=e_model, err64_over_bar=e64, model_bar_rel=bar / terms, bar64_rel=bar64 / terms)
    assert bar * TIGHTER < bar64, f"{tag}: model bar {bar:.3e} not below {bar64:.3e}"
    assert e_model <= 1.0, f"{tag}: {got!r} vs model {val!r}: {e_model:.2f} x the model bar"
    assert e64 <= 1.0, f"{tag}: {got!r} vs float64 {exact!r}: {e64:.2f} x the bar"
    return max(e_model, e64)


def nmfd_splits(B, C, L, R, T):
    """tc_nmfd_create (csrc/tc_nmfd.cu): (ws_w, k-blocks per split, last split's), then the same for dgrad."""
    Tp, Lin = cdiv(T, 64) * 64, L - T + 1
    tiles_w, tiles_h = cdiv(C, 128) * R * cdiv(T, 128), cdiv(Lin, 128) * B
    kb_w, kb_h = B * cdiv(L, 64), C * (Tp // 64)
    out = []
    for kb, tiles in ((kb_w, tiles_w), (kb_h, tiles_h)):
        ws = max(1, min(kb // 8, cdiv(132 * 4, tiles)))
        kbs = cdiv(kb, ws)
        ws = cdiv(kb, kbs)
        out += [ws, kbs, kb - (ws - 1) * kbs]
    return out


def nmfd_rtol64(case, V, W, H):
    """The f16 bar, widened where the W numerator is a single-term sum (L = T): there the ratio tile's fp16 rounding,
    up to 2^-11 |P - kappa| relative to P, is not averaged over any other term, and the kernel's tile may sit one fp16 ulp
    (another 2^-11 |P - kappa|) from the exactly rounded one."""
    B, C, L, R, T = case
    if L != T:
        return RTOL64["f16"]
    m = NmfdModel(V, W, H, rounding=False)
    P = m.V / (m.S + EPS)
    return RTOL64["f16"] + 2.0 ** -10 * float(((P - m.kappa) / P).abs().max())
