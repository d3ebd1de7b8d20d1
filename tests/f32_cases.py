"""Cases, data and float64 references of the fp32 CUDA-core kernel tests (tests/test_gpu_f32_terms.py), and what they must
cover (checked against the library's own tile planners on the CPU by tests/test_f32_plan_cover.py).

Exact cases.  The fp32 kernels round only where a value is not representable.  With small non-negative integer factors and
targets for which every product and every partial sum is an integer below 2^24, every fmaf, chunk or split sum, reduce_chunks
and column sum is exact in any order, so the kernels must equal float64 bit for bit:
  * beta 2: Pn = V and Pp = S (no eps): numerator sum V G and denominator sum S G are exact integers; so is the loss
    1/2 (s - v)^2 when 16 of its terms (one thread's `float local` per tile) stay below 2^23 (half-integers).
  * beta 1: factors in {2, 3}, so every S is an integer >= 4 (every position of a full convolution has at least one product
    of two factors) and s + eps rounds back to s; V = Q * S with Q in {0..3} makes v / (s + eps) = q exactly (IEEE division).
    The numerator is sum Q G, the denominator the column sums of the other factor.
Every partial sum of non-negative terms is at most the full sum, so `bound()` (the largest full sum or product of the case,
from its shapes and value range) below 2^24 proves exactness.
"""
import itertools
import math

import torch

EXACT = 2 ** 24
EXACT_LOSS = 2 ** 23                  # half-integer loss terms keep one fraction bit
POISON = 2.0 ** 12                    # factor value of the poisoning pass: huge stale partials everywhere


# ---- NMF ---------------------------------------------------------------------------------------------------------------
# (N, C, R): every RB (ranks 1 ... 256), rows and contracted columns at residues {1, 63, 0} mod 64 over one to three tiles
NMF_EDGE = [(1, 1, 1), (63, 129, 16), (64, 191, 17), (65, 192, 32), (127, 1, 33), (128, 63, 64), (129, 64, 65),
            (191, 65, 128), (192, 127, 129), (129, 191, 200), (65, 128, 256), (191, 63, 1)]
NMF_CHUNKED = [
    (4000, 1050, 20),      # H update: 9 chunks of 2 tiles, the last one short (1 tile)
    (1050, 4000, 20),      # the same for the W update
    (64, 2112, 17),        # H update: 32 chunks (the cap) of 2 tiles over 33 tiles: 15 chunks hold no tile
    (2112, 64, 200),       # the same for the W update, rank 200
    (66555, 65, 17),       # N > 65536: W update 32 chunks of 33 tiles (short last); column sum over 1024 blocks (short last)
]
NMF_EXACT = NMF_EDGE + NMF_CHUNKED
# beta-2 raw terms / w_partial of an f16 context (tc_supports_partial is false for beta 2: the fp32 contraction runs)
NMF_F16 = [(129, 64, 65), (4000, 1050, 20), (2112, 64, 100)]
# loss at beta 2: exact where 16 half-squares stay below 2^23
NMF_LOSS = NMF_EXACT


def nmf_bound(N, C, R, fmax, vmax):
    """Largest full sum / product of the beta-2 raw terms (and of S) of both factors."""
    smax = R * fmax * fmax
    return max(smax, vmax, max(N, C) * vmax * fmax, max(N, C) * smax * fmax)


def nmf_kl_bound(N, C, R):
    """beta 1, factors in {2, 3}, Q in {0..3}: V = Q S, numerators sum Q G, column sums."""
    smax = 9 * R
    return max(3 * smax, max(N, C) * 3 * 3)


def loss_bound(smax, vmax):
    """16 half-squares of one thread's tile sum."""
    return 16 * 0.5 * max(smax, vmax) ** 2


def pick_range(bound_of, loss_smax=None):
    """Largest factor value fmax in {3, 2, 1} (targets up to fmax^2) whose bound stays below 2^24 (and the loss's below
    2^23 when loss_smax(fmax) is given)."""
    for fmax in (3, 2, 1):
        if bound_of(fmax, fmax * fmax) < EXACT and (loss_smax is None or loss_bound(loss_smax(fmax), fmax * fmax) < EXACT_LOSS):
            return fmax
    raise AssertionError("no exact value range")


def nmf_range(N, C, R, loss=False):
    return pick_range(lambda f, v: nmf_bound(N, C, R, f, v), (lambda f: R * f * f) if loss else None)


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _ints(shape, lo, hi, g):
    return torch.randint(lo, hi + 1, shape, generator=g).float()


def nmf_eu_data(N, C, R, seed, loss=False):
    fmax = nmf_range(N, C, R, loss)
    g = _gen(seed)
    return _ints((N, C), 0, fmax * fmax, g), _ints((C, R), 0, fmax, g), _ints((N, R), 0, fmax, g)


def distinct_colsums(F):
    """Flip entries of F (in {2, 3}) until neighbouring components have different column sums, so that a ratio stage that
    reads the denominator of the wrong component shows."""
    moved = F.movedim(1, 0)
    x = moved.reshape(F.shape[1], -1).clone()                # (R, everything else)
    for r in range(1, x.shape[0]):
        i = 0
        while float(x[r].sum()) == float(x[r - 1].sum()):
            x[r, i] = 5 - x[r, i]
            i += 1
    return x.reshape(moved.shape).movedim(0, 1).contiguous()


def nmf_kl_data(N, C, R, seed):
    """(V, W, H, Q): V = Q * (H W^T) exactly, factors in {2, 3}."""
    g = _gen(seed)
    W, H = distinct_colsums(_ints((C, R), 2, 3, g)), distinct_colsums(_ints((N, R), 2, 3, g))
    Q = _ints((N, C), 0, 3, g)
    return (Q.double() * (H.double() @ W.double().t())).float(), W, H, Q


# ---- NMFD / NMF2D / NMF3D ------------------------------------------------------------------------------------------------
# (B, C, X, R, K): X the target's convolved sizes, K the kernel's; the last axis slides.  Recon MT from C in
# {1, 4, 5, 8, 9, 16, 17, 32, 33, 65, 129}, dgrad MT from R in {1, 4, 5, 9, 17, 33, 65, 129, 256}, T in {1, 2, 31, 32, 33,
# 63, 64, 65, 128, 129, 200}.
NMFD_EXACT = [
    (1, 1, (200,), 1, (200,)),         # L = T (Lin = 1), T > 128: 4 offset tiles (ntt > 1)
    (3, 4, (130,), 4, (129,)),         # T = 129, B = 3
    (1, 5, (191,), 5, (128,)),         # T = 128
    (3, 8, (97,), 9, (65,)),           # T = 65 (tp rounds up), L ragged
    (1, 9, (64,), 17, (64,)),          # L = T = 64
    (1, 16, (100,), 33, (63,)),
    (3, 17, (127,), 65, (33,)),
    (1, 32, (200,), 129, (32,)),
    (1, 33, (150,), 256, (31,)),       # rank 256
    (3, 65, (77,), 2, (2,)),           # dgrad: 64 splits of 2 channels over 65: the last 31 hold none
    (1, 129, (300,), 3, (1,)),         # T = 1
    (3, 7, (333,), 6, (6,)),           # W inner 6: 2 mod 4, even rank
    (1, 3, (4000,), 2, (8,)),          # long lines
    (2, 40, (515,), 4, (12,)),         # H inner 504 (vec4)
    (1, 20, (250,), 8, (2,)),
    (1, 129, (3400,), 3, (2,)),        # dgrad: 10 splits of 13 channels, the last one 12
    # NMF2D (X2, L) and NMF3D (X1, X2, L)
    (1, 3, (7, 70), 4, (3, 8)),        # T2 > 1; recon lines 7 and dgrad lines 5 not multiples of XT = 16
    (2, 20, (9, 66), 3, (4, 5)),       # recon MT 32 (XT 2): 9 lines
    (1, 2, (3, 6, 40), 3, (3, 2, 5)),  # T1 = X1 (J1 = 1), T2 = 2; several outer offsets per wgrad block
    (1, 4, (4, 5, 30), 2, (2, 3, 4)),  # 6 outer offsets in one wgrad block (no = 6), vec4 W
    (2, 5, (5, 6, 20), 3, (3, 4, 4)),  # 12 outer offsets over 2 block groups (nog > 1)
    (1, 2, (127, 20), 2, (1, 4)),      # wgrad: 64 splits of 2 lines over 127 lines, the last one 1
    (1, 1, (100, 9), 2, (1, 3)),       # wgrad: 64 splits of 2 lines over 100 lines: the last 14 hold none
]


def nmfd_dims(case):
    B, C, X, R, K = case
    J = tuple(x - k + 1 for x, k in zip(X, K))
    return B, C, X, R, K, J


def nmfd_terms(case):
    """(K_S, wgrad terms, dgrad terms): products per S, terms per W-gradient and per H-gradient entry."""
    B, C, X, R, K, J = nmfd_dims(case)
    return R * math.prod(K), B * math.prod(J), C * math.prod(K)


def nmfd_bound(case, fmax, vmax):
    ks, nw, nh = nmfd_terms(case)
    smax = ks * fmax * fmax
    return max(smax, vmax, max(nw, nh) * max(vmax, smax) * fmax)


def nmfd_kl_bound(case):
    ks, nw, nh = nmfd_terms(case)
    B, C, X, R, K, J = nmfd_dims(case)
    return max(27 * ks, max(nw, nh) * 9, max(B * math.prod(J), C * math.prod(K)) * 3)


def nmfd_range(case, loss=False):
    ks = nmfd_terms(case)[0]
    return pick_range(lambda f, v: nmfd_bound(case, f, v), (lambda f: ks * f * f) if loss else None)


def nmfd_loss_ok(case):
    try:
        nmfd_range(case, loss=True)
        return True
    except AssertionError:
        return False


NMFD_LOSS = [c for c in NMFD_EXACT if nmfd_loss_ok(c)]


def nmfd_eu_data(case, seed, loss=False):
    B, C, X, R, K, J = nmfd_dims(case)
    fmax = nmfd_range(case, loss)
    g = _gen(seed)
    return _ints((B, C, *X), 0, fmax * fmax, g), _ints((C, R, *K), 0, fmax, g), _ints((B, R, *J), 0, fmax, g)


def nmfd_kl_data(case, seed):
    B, C, X, R, K, J = nmfd_dims(case)
    g = _gen(seed)
    W, H = distinct_colsums(_ints((C, R, *K), 2, 3, g)), distinct_colsums(_ints((B, R, *J), 2, 3, g))
    Q = _ints((B, C, *X), 0, 3, g)
    return (Q.double() * recon(H.double(), W.double())).float(), W, H, Q


# ---- float64 references: plain shifted products (matmul / einsum), no convolution algorithm ---------------------------------
def _offsets(K):
    return itertools.product(*(range(k) for k in K))


def _window(t, J):
    return (slice(None), slice(None)) + tuple(slice(ti, ti + j) for ti, j in zip(t, J))


def recon(H, W):
    """S[b,c,j+t] = sum_r W[c,r,t] H[b,r,j] on H's device and dtype."""
    J, K = H.shape[2:], W.shape[2:]
    out = torch.zeros(H.shape[0], W.shape[0], *(j + k - 1 for j, k in zip(J, K)), dtype=H.dtype, device=H.device)
    for t in _offsets(K):
        out[_window(t, J)] += torch.einsum("cr,br...->bc...", W[(slice(None), slice(None)) + t], H)
    return out


def grad_w(G, H, K):
    J = H.shape[2:]
    out = torch.zeros(G.shape[1], H.shape[1], *K, dtype=H.dtype, device=H.device)
    for t in _offsets(K):
        out[(slice(None), slice(None)) + t] = torch.einsum("bc...,br...->cr", G[_window(t, J)], H)
    return out


def grad_h(G, W, J):
    K = W.shape[2:]
    out = torch.zeros(G.shape[0], W.shape[1], *J, dtype=W.dtype, device=W.device)
    for t in _offsets(K):
        out += torch.einsum("cr,bc...->br...", W[(slice(None), slice(None)) + t], G[_window(t, J)])
    return out


def colsum(F):
    return F.sum([d for d in range(F.dim()) if d != 1])


def nmf_terms64(which, Pn, Pp, W, H):
    """NMF raw terms from the phi outputs (Pp None: beta 1, the column sums of the other factor)."""
    if which == 0:
        return Pn.t() @ H, (H.sum(0) if Pp is None else Pp.t() @ H)
    return Pn @ W, (W.sum(0) if Pp is None else Pp @ W)


def nmfd_terms64(which, Pn, Pp, W, H):
    if which == 0:
        K = W.shape[2:]
        return grad_w(Pn, H, K), (colsum(H) if Pp is None else grad_w(Pp, H, K))
    J = H.shape[2:]
    return grad_h(Pn, W, J), (colsum(W) if Pp is None else grad_h(Pp, W, J))


# ---- float64-bar cases (random non-integer data): the mode arithmetic of beta 0, 0.5, 1.5, 3, -1 and every loss ---------
U = 2.0 ** -24
TWO_BETAS = [0, 0.5, 1.5, 3, -1]
LOSS_BETAS = [0, 0.5, 1, 1.5, 2, 3, -1]
NMF_BAR = [(65, 129, 17), (129, 191, 200), (1, 63, 1), (1050, 4000, 20), (64, 2112, 17)]
NMFD_BAR = [(3, 17, (127,), 65, (33,)), (1, 1, (200,), 1, (200,)), (2, 40, (515,), 4, (12,)), (1, 3, (7, 70), 4, (3, 8)),
            (2, 5, (5, 6, 20), 3, (3, 4, 4))]


def gam(n):
    """gamma_n = n u / (1 - n u): relative error bound of a sum of n non-negative fp32 terms (any order, fma included)."""
    return n * U / (1 - n * U)


def bar_data(shape_v, shape_w, shape_h, seed):
    g = _gen(seed)
    return (torch.rand(*shape_v, generator=g) + 0.5, torch.rand(*shape_w, generator=g) + 0.5,
            torch.rand(*shape_h, generator=g) + 0.5)


def terms_bar(beta, ks, n, nch):
    """Relative bars (numerator, denominator) of one raw-term entry: every term of the sum is computed to
    p (gamma_{K_S} + u) + 9u, with p the power S enters with (|beta - 2| and |beta - 1|, IS: 2 and 1): S to gamma_{K_S}, the
    eps add u; then the operations on it: 1/x and r r (IEEE, 0.5 ulp each) or powf (4 ulp, CUDA Math API single-precision
    table, "powf(x,y)"), and the product with v, within 9u.  The sum of the terms adds gamma_n, n >= its chunk's or split's
    length, and the chunk / split reduction gamma_{nch}.  x 1.01 for the second-order products."""
    out = []
    for p in (abs(beta - 2), abs(beta - 1)):
        out.append(1.01 * (p * (gam(ks) + U) + 9 * U + gam(n) + gam(nch)))
    return out


def loss_pieces(beta, s, v, eps):
    """(term, M): the float64 loss terms at (s, v) and the sum M of the absolute values of the pieces each is formed from.
    Every piece is computed to within rho = g (gamma_{K_S} + 2u) + 16u of M (see loss_bar)."""
    if beta == 2:
        d = s - v
        return 0.5 * d * d, 0.5 * d * d + d.abs() * s
    if beta == 1:
        lv, ls = (v + eps).log(), (s + eps).log()
        return v * (lv - ls) - v + s, v * lv.abs() + v * ls.abs() + v + s
    if beta == 0:
        te, xe = v + eps, s + eps
        return te / xe - te.log() + xe.log() - 1, te / xe + te.log().abs() + xe.log().abs() + 1
    x = s + eps
    t = v + eps if beta < 0 else v
    bm = beta - 1
    a, b, c = t.pow(beta), bm * x.pow(beta), beta * t * x.pow(bm)
    return (a + b - c) / (beta * bm), (a.abs() + b.abs() + c.abs()) / abs(beta * bm)


def loss_bar(beta, s, v, ks, eps):
    """Absolute bar of the loss: sum over the terms of M rho, rho = g (gamma_{K_S} + 2u) + 16u with g = max(1, |beta|,
    |beta - 1|) the largest power S enters with (its error through the power, the eps add), 16u for the powf (4 ulp) / logf
    (1 ulp, CUDA Math API single-precision table, "logf(x)") results and the roundings of the term's own arithmetic; plus
    gamma_16 of the sum of |terms| (one thread's `float local` over its 4 x 4 tile) and 1e-15 of it for the double sums."""
    term, M = loss_pieces(beta, s, v, eps)
    g = max(1.0, abs(beta), abs(beta - 1))
    rho = g * (gam(ks) + 2 * U) + 16 * U
    tot = term.abs().sum()
    return float(term.sum()), float(M.sum() * rho + (gam(16) + 1e-15) * tot)


# ---- ratio stage (nmf.py:78-92) --------------------------------------------------------------------------------------------
# (kind, case, label): one update of each factor from the exact raw terms of a case, with l1, l2 > 0 and gamma != 1
RATIO_L1, RATIO_L2 = 0.25, 0.125
RATIO_CASES = [
    ("nmf", (129, 64, 65)),
    ("nmf", (66555, 65, 17)),
    ("nmfd", (3, 7, (333,), 6, (6,))),          # W inner 6 (2 mod 4): scalar kernel, the H side too (Lin 328 -> vec4)
    ("nmfd", (2, 40, (515,), 4, (12,))),        # W inner 12 and H inner 504: vec4 on both
    ("nmfd", (3, 8, (97,), 9, (65,))),          # scalar on both
    ("nmfd", (1, 4, (4, 5, 30), 2, (2, 3, 4))),  # NMF3D: W inner 24 (vec4), H inner 81 (scalar)
]


def ratio64(p, num, den, gamma, l1, l2, kl):
    """nmf.py:78-92 in float64."""
    eps = 2.0 ** -23
    neg = num.clamp_min(0) + eps
    pos = den if kl else den.clamp_min(0) + eps
    pos = pos + l1
    pos = pos + l2 * p
    mult = neg / pos
    return p * mult.pow(gamma), mult


def ratio_bar(mult, gamma):
    """Relative bar of the ratio stage: eps add (u), the den + eps, + l1 and l2 fma (3u), the division (u): the ratio to
    5u; powf amplifies that by gamma and adds 4 ulp (8u) and gamma's own fp32 rounding (gamma u |ln mult|); the final
    product u.  x 1.01 for second-order products."""
    return 1.01 * U * (gamma * (5 + mult.log().abs()) + 10)
