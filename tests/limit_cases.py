"""Shapes at the size limits of the kernels: buffers past 2^31 elements and grids at the CUDA grid-dimension limits, with
the float64 references the GPU tests (tests/test_gpu_limits.py) compare against and the host checks of
tests/test_limit_plan.py.

TEST INFRASTRUCTURE ONLY.  Nothing here calls the library's kernels; the references are plain float64 torch on whichever
device the data lives on, in blocks of at most 2^24 target elements so that a 2^31-element target fits next to its
context on one card.

Every big case names the buffer and element index it crosses.  Its data is structured so that a wrapped 32-bit index reads
different values: the target and the factors are random, with a band of 8x hotter rows that straddles element 2^31 of the
target and hot last rows.  The exact beta-2 cases keep the contracted factor zero outside those rows, so that every sum
stays an integer below 2^24.
"""
import math

import torch

import f32_cases as fc
from oracle import mu_oracle as orc

ELEM = 2 ** 31                # the element index a 32-bit signed index cannot reach
GRID_X = 2 ** 31 - 1
GRID_YZ = 65535
INT_MAX = 2 ** 31 - 1
BAND = 32                     # hot rows on each side of the boundary row
LAST = 16                     # hot last rows
BLOCK = 2 ** 24               # target elements per reference block
F16_BAR = 1.25e-3             # tests/tc_model.py RTOL64["f16"]
KL_EXACT_BAR = 1e-9           # exact beta-1 data: the float64 reference divides by S + eps, the kernel's fp32 S + eps is S


def cdiv(a, b):
    return -(-a // b)


# ---- big cases ---------------------------------------------------------------------------------------------------------
# NMF (N, C, R): V (N, C).  "fac" is the factor whose rows the band marks (the rows of V it multiplies).
# prec -> betas run on it; beta 2 on f32 is exact (integer data, the contracted factor zero outside the hot rows).
NMF_BIG = {
    # the configs[3] shard for one card cut to just over 2^31: V row n >= 2^31 / C, and rows c >= 2^31 / ldn of the
    # transposed fp16 copy, lie past element 2^31
    "nmf_tall": dict(N=2 ** 18 + 64, C=8192, R=128, fac="H", runs={"f32": [2], "f16": [1]}),
    # 33 M rows of W: V column c of the last row is past 2^31 for c >= 2^31 - 63 C, and the transposed copy's last rows
    "nmf_wide": dict(N=64, C=2 ** 25 + 64, R=8, fac="W", runs={"f32": [2], "f16": [1]}),
    # H itself past 2^31 elements (rows n >= 2^31 / R): the W update's contraction reads all of it, and its beta-1
    # denominator is the column sum of H; past the tensor-core N limit, so fp32 only
    # Beta 1 on exact data: V = Q (H W^T), Q in {0..3}, H nonzero on the hot rows only, so the ratio is Q up to the eps
    # Its raw H terms hold three N R buffers at once (H, the split partials, the output): 26 GB is the library's floor there
    "nmf_tall_factor": dict(N=2 ** 24 + 64, C=8, R=128, fac="H", runs={"f32": [1]}, kl_exact=True),
}
# NMFD (B, C, L, R, T): V (B, C, L) past 2^31 at rows (b, c) >= 2^31 / L; P16 (B C rows of Lq) past it at rows >= 2^31 / Lq
NMFD_BIG = {
    "nmfd_long": dict(B=2, C=1025, L=ELEM // (2 * 1025) + 256, R=16, T=16, runs={"f32": [1], "f16": [1]}),
}


def nmf_boundary_row(case, boundary=ELEM):
    """The hot band's centre: the row of the banded factor whose V elements first reach `boundary`."""
    N, C, R = case["N"], case["C"], case["R"]
    if case["fac"] == "H":
        if N * C > boundary:
            return cdiv(boundary, C)
        return cdiv(boundary, R) if N * R > boundary else N // 2      # the factor itself crosses
    return boundary - (N - 1) * C if N * C > boundary else C // 2     # column of the last V row at the boundary


def nmf_hot_rows(case, boundary=ELEM):
    n = case["N"] if case["fac"] == "H" else case["C"]
    b = nmf_boundary_row(case, boundary)
    rows = set(range(max(0, b - BAND), min(n, b + BAND))) | set(range(n - LAST, n)) | {0}
    return torch.tensor(sorted(rows), dtype=torch.int64)


def nmf_elements(case):
    """Elements of each buffer the NMF kernels read: V, the fp16 copies (f16), the factors."""
    N, C, R = case["N"], case["C"], case["R"]
    return {"V": N * C, "W": C * R, "H": N * R}


def nmf_crossings(case):
    """{buffer: (factor, first row of that factor whose operand reaches element 2^31 of the buffer)} for every buffer of
    this case that passes 2^31 elements: V row n multiplies H row n, V column c (all of it in the transposed fp16 copy,
    of rows at least N long) W row c."""
    N, C, R = case["N"], case["C"], case["R"]
    out = {}
    if N * C > ELEM:
        out["V"] = ("H", ELEM // C) if case["fac"] == "H" else ("W", ELEM - (N - 1) * C)
        if "f16" in case["runs"]:
            out["Vt16"] = ("W", ELEM // N)
    if N * R > ELEM:
        out["H"] = ("H", ELEM // R)
    return out


def nmf_device_bytes(case, prec, beta, sms=132):
    """Device memory one run allocates, from the shape: V and the factors; the fp32 context's split partials (numerator at
    create, denominator for beta != 1: the larger factor's rows x R per chunk); the raw terms of the larger checked factor;
    on f16 the tensor-core context (V16, its transpose, the fp16 factors at the padded rank, its split partials, tc_create);
    the float64 reference (blocks of BLOCK elements, per-range terms of at most BLOCK elements)."""
    import tc_model as tcm
    from torchnmf_b200 import _capi
    N, C, R = case["N"], case["C"], case["R"]
    p = _capi.nmf_plan(N, C, R)
    b = 4 * N * C + 4 * (N + C) * R
    b += 4 * max(p["nch_w"] * C * R, p["nch_h"] * N * R) * (2 if beta != 1 else 1)
    rows = max((C, N)[w] for w in case.get("which", [0, 1]))
    b += 4 * (rows * R + (R if beta == 1 else rows * R))
    if prec == "f16":
        rp = 64 if R <= 64 else 128
        tn = tcm.tn(prec, R)
        b += 2 * N * cdiv(C, 8) * 8 + 2 * C * cdiv(N, 8) * 8 + 2 * (N + C) * rp
        b += 4 * max(tcm.plan(C, N, sms, tn)[2] * C * rp, tcm.plan(N, C, sms, tn)[2] * N * rp)
    return b + 8 * 8 * BLOCK + (2 << 30)                 # + the caching allocator's rounding of the blocks


def nmf_data(case, beta, device, seed=0):
    """(V, W, H) fp32 on `device`.  Beta 2: integers, the banded factor zero outside the hot rows.  Beta 1: positive
    reals, 8x hotter target in the hot rows."""
    N, C, R = case["N"], case["C"], case["R"]
    g = torch.Generator(device=device).manual_seed(seed)
    hot = nmf_hot_rows(case, case.get("boundary", ELEM)).to(device)
    if beta == 2:
        V = torch.randint(1, 5, (N, C), generator=g, device=device, dtype=torch.float32)
        W = torch.randint(1, 3, (C, R), generator=g, device=device, dtype=torch.float32)
        H = torch.randint(1, 3, (N, R), generator=g, device=device, dtype=torch.float32)
        F = H if case["fac"] == "H" else W
        keep = F[hot].clone()
        F.zero_()
        F[hot] = keep
        return V, W, H
    if case.get("kl_exact"):
        W = torch.randint(2, 4, (C, R), generator=g, device=device, dtype=torch.float32)
        H = torch.zeros(N, R, device=device)
        H[hot] = torch.randint(2, 4, (len(hot), R), generator=g, device=device, dtype=torch.float32)
        Q = torch.randint(0, 4, (N, C), generator=g, device=device, dtype=torch.float32)
        return Q.mul_(H @ W.t()), W, H
    V = torch.rand(N, C, generator=g, device=device).add_(0.5)
    W = torch.rand(C, R, generator=g, device=device).add_(0.5)
    H = torch.rand(N, R, generator=g, device=device).add_(0.5)
    if case["fac"] == "H":
        V[hot] *= 8
    else:
        V[:, hot] *= 8
    return V, W, H


def nmf_exact_bound(case):
    """Largest partial sum of the beta-2 terms of nmf_data (V <= 4, factors <= 2, the banded factor nonzero on the hot
    rows only): every fp32 sum is exact below 2^24."""
    N, C, R = case["N"], case["C"], case["R"]
    nhot = len(nmf_hot_rows(case, case.get("boundary", ELEM)))
    smax = R * 2 * 2
    full, banded = (C, nhot) if case["fac"] == "H" else (nhot, N)   # terms per H-row sum, per W-row sum
    return max(smax, full * max(4, smax) * 2, banded * max(4, smax) * 2)


def sum64(x, dim=None, rows=2 ** 20):
    """Float64 sum of fp32 `x` (over all elements, or over dim 0) in blocks of at most BLOCK elements: no float64 copy of
    x."""
    if dim is None:
        x = x.reshape(-1)
        rows = BLOCK
    else:
        rows = max(1, BLOCK // max(1, x[0].numel()))
    out = None
    for r0 in range(0, x.shape[0], rows):
        blk = x[r0:r0 + rows].double()
        part = blk.sum() if dim is None else blk.sum(dim)
        out = part if out is None else out + part
    return out


def nmf_terms_ref(V, W, H, beta, which, rows=None, blocks=BLOCK, F_rows=None):
    """Float64 raw terms (num, den) of the update of W (which 0) or H (which 1) for the factor rows `rows` (a range or an
    index tensor; None: all), den = the column sum of the other factor at beta 1.  `F_rows`: the values of those rows to use
    in place of the factor's current ones (the rows as they were before an update).  The contraction runs over blocks of
    the other factor's rows holding at most `blocks` elements of V or of that factor (None: one block)."""
    F, G = (W, H) if which == 0 else (H, W)
    rows = range(F.shape[0]) if rows is None else rows
    if isinstance(rows, range):
        idx, nr = slice(rows.start, rows.stop), len(rows)
    else:
        idx, nr = rows.to(V.device), rows.numel()
    F64 = (F[idx] if F_rows is None else F_rows).double()
    nG, R = G.shape
    kb = nG if blocks is None else max(1, blocks // max(nr, R))
    num = torch.zeros(nr, R, dtype=torch.float64, device=V.device)
    den = torch.zeros_like(num)
    for k0 in range(0, nG, kb):
        Gb = G[k0:k0 + kb].double()
        Vb = V[k0:k0 + kb, idx].t() if which == 0 else V[idx, k0:k0 + kb]       # copies the block only
        Pn, Pp = orc.phi(Vb.double(), F64 @ Gb.t(), beta)
        num += Pn @ Gb
        if Pp is not None:
            den += Pp @ Gb
    if beta == 1:
        den = sum64(G, 0)
    return num, den


def nmf_loss_ref(V, W, H, beta, blocks=BLOCK):
    """(sum of the float64 loss terms, sum of their pieces' magnitudes M, sum of |terms|) over blocks of V: the pieces of
    f32_cases.loss_bar, which adds over blocks."""
    N, C = V.shape
    cb = min(C, blocks)
    rb = max(1, blocks // cb)
    tot = [0.0, 0.0, 0.0]
    for r0 in range(0, N, rb):
        Hb = H[r0:r0 + rb].double()
        for c0 in range(0, C, cb):
            term, M = fc.loss_pieces(beta, Hb @ W[c0:c0 + cb].double().t(), V[r0:r0 + rb, c0:c0 + cb].double(), orc.EPS)
            tot[0] += float(term.sum()); tot[1] += float(M.sum()); tot[2] += float(term.abs().sum())
    return tot


def loss_bar_of(beta, pieces, ks, prec):
    """The absolute bar of f32_cases.loss_bar from summed pieces; on the tensor cores plus tests/test_gpu_tc_terms.py's
    f16 loss bar, (2^-11 g + 2^-12) of the sum of |terms|."""
    want, M, tot = pieces
    g = max(1.0, abs(beta), abs(beta - 1))
    bar = M * (g * (fc.gam(ks) + 2 * fc.U) + 16 * fc.U) + (fc.gam(16) + 1e-15) * tot
    if prec == "f16":
        bar += (2.0 ** -11 * g + 2.0 ** -12) * tot
    return want, bar


def update_rows(case, which, n_random=256, seed=1):
    """Rows of factor `which` whose update the GPU tests check: every row whose operand lies past element 2^31 of a buffer
    it is read from (V, the transposed fp16 copy, the factor itself), 2 BAND rows before the first such row, the hot rows,
    the first and the last row, and `n_random` others."""
    n = case["C"] if which == 0 else case["N"]
    fac = "W" if which == 0 else "H"
    rows = set(nmf_hot_rows(case, case.get("boundary", ELEM)).tolist()) if fac == case["fac"] else set()
    rows |= {0, n - 1}
    for buf, (f, first) in nmf_crossings(case).items():
        if f == fac:
            rows |= set(range(max(0, first - 2 * BAND), n))
    g = torch.Generator().manual_seed(seed)
    rows |= set(torch.randint(0, n, (n_random,), generator=g).tolist())
    return torch.tensor(sorted(rows), dtype=torch.int64)


def row_ranges(case, which, blocks=BLOCK):
    """The row ranges of factor `which` the GPU tests check one after another: together, every row."""
    n = case["C"] if which == 0 else case["N"]
    size = max(1, blocks // case["R"])
    return [range(r, min(n, r + size)) for r in range(0, n, size)]


def nmfd_dims(case):
    return case["B"], case["C"], case["L"], case["R"], case["T"]


def nmfd_crossings(case):
    B, C, L, R, T = nmfd_dims(case)
    out = {}
    if B * C * L > ELEM:
        out["V"] = ELEM // L                              # flattened row b C + c
        out["Pn"] = ELEM // L
        if "f16" in case["runs"]:
            lq = L + 1024                                 # P16's row pitch is at least L + 1024
            out["P16"] = ELEM // lq
    return out


def nmfd_device_bytes(case, prec):
    """Device memory one run allocates, from the shape: V and the context's Pn (fp32, every context); on f16 P16 (B C + 1
    rows of Lq halfs), Hp16 (B R rows of Lp) and the fp16 copies of W; the fp32 context's split partials (its numerator
    buffer, allocated at create); the factors, their copies before the updates, the raw terms; the float64 reference
    (channel blocks of BLOCK elements and the full-size terms of both factors)."""
    B, C, L, R, T = nmfd_dims(case)
    Lin = L - T + 1
    from torchnmf_b200 import _capi
    nw, nh = C * R * T, B * R * Lin
    p = _capi.nmfd_plan(B, C, [L], R, [T])
    b = 2 * 4 * B * C * L
    b += 4 * max(p["wgrad_nsplit"] * nw, p["dgrad_nsplit"] * nh)
    if prec == "f16":
        tp, q = _tc_pitches(L, T), _capi.nmfnd_tc_plan(B, C, [L], R, [T])
        b += 2 * (B * C + 1) * tp[1] + 2 * B * R * tp[0] + 2 * 2 * cdiv(C, 128) * 128 * R * cdiv(T, 64) * 64
        b += 4 * max(q["ws_w"] * nw, q["ws_h"] * nh)
    b += 4 * 3 * (2 * nw + 2 * nh)                        # factors, copies, raw terms
    b += 8 * 4 * (2 * nw + 2 * nh) + 8 * 8 * BLOCK         # float64 terms (num, den, |P - kappa| sums) and blocks
    return b


def _tc_pitches(L, T):
    """(Lp, Lq): the row pitches of Hp16 and P16 (tc_nmfd_plan)."""
    Tp = cdiv(T, 64) * 64
    padl = cdiv(Tp + 136, 8) * 8
    r2048 = cdiv(L, 2048) * 2048
    return cdiv(padl + r2048 + 256 + 256 + 136, 8) * 8, cdiv(r2048 + 1024 + Tp + 64 + 256 + 8, 8) * 8


def nmfd_data(case, device, seed=0):
    """Positive reals; the rows (b, c) around the boundary row and the last rows 8x hotter."""
    B, C, L, R, T = nmfd_dims(case)
    g = torch.Generator(device=device).manual_seed(seed)
    V = torch.rand(B, C, L, generator=g, device=device).add_(0.5)
    W = torch.rand(C, R, T, generator=g, device=device).add_(0.5)
    H = torch.rand(B, R, L - T + 1, generator=g, device=device).add_(0.5)
    rows = V.view(B * C, L)
    b = min(case.get("boundary", ELEM) // L, B * C - 1)
    rows[max(0, b - 2): b + 2] *= 8
    rows[-2:] *= 8
    return V, W, H


def nmfd_terms_ref(V, W, H, beta, blocks=BLOCK, kappa=None):
    """Float64 raw terms of both NMFD updates from channel blocks of at most `blocks` target elements (None: all).  With
    `kappa` (beta 1) also the sums of |P - kappa| times the other factor, ((A_W,), (A_H,)): what the tensor-core kernels
    accumulate, the scale of their fp32 accumulation error."""
    B, C, L = V.shape
    cb = C if blocks is None else max(1, min(C, blocks // (B * L)))
    W64, H64 = W.double(), H.double()
    K, J = W.shape[2:], H.shape[2:]
    gW = [torch.zeros(W.shape, dtype=torch.float64, device=V.device) for _ in range(3)]
    gH = [torch.zeros(H.shape, dtype=torch.float64, device=V.device) for _ in range(3)]
    for c0 in range(0, C, cb):
        Wb = W64[c0:c0 + cb]
        Pn, Pp = orc.phi(V[:, c0:c0 + cb].double(), fc.recon(H64, Wb), beta)
        gW[0][c0:c0 + cb] = fc.grad_w(Pn, H64, K)
        gH[0] += fc.grad_h(Pn, Wb, J)
        if kappa is not None:
            D = (Pn - kappa).abs_()
            gW[2][c0:c0 + cb] = fc.grad_w(D, H64, K)
            gH[2] += fc.grad_h(D, Wb, J)
        if Pp is not None:
            gW[1][c0:c0 + cb] = fc.grad_w(Pp, H64, K)
            gH[1] += fc.grad_h(Pp, Wb, J)
    if beta == 1:
        gW[1], gH[1] = fc.colsum(H64), fc.colsum(W64)
    if kappa is not None:
        return (gW[0], gW[1]), (gH[0], gH[1]), ((gW[2],), (gH[2],))
    return (gW[0], gW[1]), (gH[0], gH[1])


def nmfd_loss_ref(V, W, H, beta, blocks=BLOCK):
    """The pieces of f32_cases.loss_bar summed over channel blocks of at most `blocks` target elements."""
    B, C, L = V.shape
    cb = max(1, min(C, blocks // (B * L)))
    H64 = H.double()
    tot = [0.0, 0.0, 0.0]
    for c0 in range(0, C, cb):
        term, M = fc.loss_pieces(beta, fc.recon(H64, W[c0:c0 + cb].double()), V[:, c0:c0 + cb].double(), orc.EPS)
        tot[0] += float(term.sum()); tot[1] += float(M.sum()); tot[2] += float(term.abs().sum())
    return tot


def nmfd_kappa(V, W, H):
    """The tensor-core path's centring constant sum(V) / sum(W H), in float64."""
    return float(sum64(V) / (fc.colsum(W.double()) * fc.colsum(H.double())).sum())


def nmfd_tc_trunc(kblocks):
    """Relative (to A) bound of the tensor cores' truncating fp32 accumulation over one split of `kblocks` k-blocks of 64:
    tests/tc_model.py's KSTEP_ULP ulp per 16-term k-step."""
    return 8 * 2.0 ** -23 * kblocks * 4


def scaled(case, kind, factor):
    """A copy of a big case with the same structure and `factor` times fewer target elements: the long axis shrinks,
    and the boundary moves with it (boundary = 2^31 / factor)."""
    c = dict(case)
    if kind == "nmfd":
        c["L"] = max(c["T"] + 8, cdiv(c["L"], factor) + 1)
    else:
        k = "N" if c["fac"] == "H" else "C"
        c[k] = max(2 * BAND + LAST + 8, cdiv(c[k], factor) + 1)
    c["boundary"] = ELEM // factor
    return c


def wrap_target(V, boundary):
    """V as a 31-bit-masked index reads it: element i >= boundary replaced by element i mod boundary (boundary standing
    for 2^31 in a scaled case)."""
    flat = V.reshape(-1).clone()
    n = flat.numel()
    if n > boundary:
        idx = torch.arange(boundary, n, device=V.device) % boundary
        flat[boundary:] = flat[idx]
    return flat.view(V.shape)


# ---- grid-limit cases (tiny memory) --------------------------------------------------------------------------------------
# (name, kind, shape, precision, expected) with expected "runs", or ("rejected", words of the message) for create.
# NMF (N, C, R); NMFD (B, C, L, R, T).
NMF_TC_N = GRID_YZ * 64
GRID_CASES = [
    ("nmf_tc_n_limit", "nmf", (NMF_TC_N, 72, 8), "f16", "runs"),
    ("nmf_tc_n_over_auto", "nmf", (NMF_TC_N + 1, 72, 8), "auto", "runs"),           # resolves to f32
    ("nmf_tc_n_over_f16", "nmf", (NMF_TC_N + 1, 72, 8), "f16", ("rejected", "tensor-core")),
    # the f16 shapes keep every sum at 64 terms or more, as the f16 bar assumes (tests/test_gpu_tc_terms.py)
    ("nmfd_b65535_f32", "nmfd", (GRID_YZ, 2, 6, 2, 3), "f32", "runs"),
    ("nmfd_b65536_f32", "nmfd", (GRID_YZ + 1, 2, 6, 2, 3), "f32", "runs"),
    ("nmfd_b65535_f16", "nmfd", (GRID_YZ, 64, 6, 8, 3), "f16", "runs"),
    ("nmfd_b65536_f16", "nmfd", (GRID_YZ + 1, 64, 6, 8, 3), "f16", "runs"),
    ("nmfd_b131073_f16", "nmfd", (2 * GRID_YZ + 3, 32, 4, 8, 2), "f16", "runs"),      # three slices, the last of 3
    ("nmfd_br65535_f16", "nmfd", (257, 64, 6, 255, 2), "f16", "runs"),
    ("nmfd_br65536_f16", "nmfd", (256, 64, 6, 256, 2), "f16", "runs"),
    ("nmfd_br65600_f16", "nmfd", (1025, 64, 6, 64, 2), "f16", "runs"),
    ("nmfd_c_limit_f32", "nmfd", (1, GRID_YZ * 64, 2, 1, 1), "f32", "runs"),
    ("nmfd_c_over_f32", "nmfd", (1, GRID_YZ * 64 + 1, 2, 1, 1), "f32", ("rejected", "channels")),
    ("nmfd_rt65535_f16", "nmfd", (1, 1, 257 * 128 + 127, 255, 257 * 128), "f16", "runs"),
    ("nmfd_rt65536_f16", "nmfd", (1, 1, 256 * 128, 256, 256 * 128), "f16", ("rejected", "R ceil(T / 128)")),
    ("nmfd_rt65536_auto", "nmfd", (1, 1, 256 * 128, 256, 256 * 128), "auto", "runs"),   # resolves to f32
]

# shapes create must reject however much memory there is (the narrowing bounds of nmfd_shape_of / tc_nmfd_plan)
REJECT_CASES = [
    ("nmfd_b_2p31", (2 ** 31, 1, 1, 1, 1), "auto", "batch"),
    ("nmfd_c_2p31", (1, 2 ** 31, 1, 1, 1), "auto", "channels"),
    ("nmfd_bc_tma", (2 ** 20, 2048, 1, 1, 1), "f16", "B C"),
]


def grid_bytes(kind, shape, prec):
    """Upper estimate of the device memory of a grid case."""
    if kind == "nmf":
        N, C, R = shape
        return 16 * N * C + 64 * (N + C) * max(R, 64) + (1 << 28)
    B, C, L, R, T = shape
    Lin = L - T + 1
    tc = 2 * B * R * (L + 4096) + 2 * B * C * (L + 4096) + 8 * C * R * (T + 64) if prec != "f32" else 0
    return 4 * B * C * L * 4 + 4 * 70 * (C * R * T + B * R * Lin) + tc + (1 << 28)
