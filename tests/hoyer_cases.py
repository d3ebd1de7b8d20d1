"""Cases, float64 reference, a model of the kernel's arithmetic and the bars of the Hoyer projection tests
(tests/test_hoyer_cases.py on the CPU, tests/test_gpu_hoyer_terms.py on the GPU).

`nmfb200_hoyer_project` (csrc/project.cu) replaces every slice x[:, j, :] of a tensor viewed as (outer, D, inner) by the
projection of oracle/hoyer_oracle.proj_func (nmf.py:21-49).  Three references:

* proj64(x, k1, k2): the reference algorithm in float64 throughout, on the fp32 inputs; returns the output, the round count
  and the coordinates each round zeroes.
* kernel_model(x, k1, k2): the kernel's arithmetic restated.  fp32 element operations (`v = x + shift`, `fmaxf`, `w = v - m`,
  `fmaf(alphap, w, v)`), double reductions of exact fp32 products summed in the kernel's own order (1024 strided per-thread
  sums, then the xor butterflies of block_sum3), the fp32 quadratic for alphap, the same exits and `max_rounds`.  What the
  model cannot know is how the compiler contracts `bf*bf - 4.f*af*cf`; it compiles one of three forms (uncontracted, or
  either product fused), the same form every round.  model_bar() runs each form, and each with its shift one ulp off (a
  double sum rounded to fp32 next to a rounding boundary); per form, an output entry's bar is its spread over the shifted
  runs plus one ulp of the entry.  A kernel slice must match one form within that form's bar.  The sums a, b, c are exact
  products added in the kernel's order, so no wider set of alphap is admitted.  An entry that is zero in one run of the
  form and not in another is marked ambiguous: only there may the kernel's zero set differ.
* classify(): proj64 on seeded relative +-u perturbations (u = 2^-24) of x, k1 and k2, and of every element-wise step
  (where fp32 rounds: `x + shift` is relative to the shifted entry, not to x).  "stable": the zero sets of every
  round and the round count agree and 8x the output's spread stays below max|y| / 32; the case is then held to float64 at
  8x that spread plus 4 ulp of max|y|.  "unstable": they do not, and only the model and the invariants apply;
  "degenerate": float64 gives NaN (a = w.w = 0: the surviving support is uniform), zeroes every coordinate (the
  reference divides by zero), or the quadratic's b^2 or 4ac pass the fp32 range (gradient trials of 1e12 and more: the
  fp32 reference and the kernel both form inf - inf; only the model applies).

The catalogue names, per case, the branch or edge of the kernel it exists for; tests/test_hoyer_cases.py proves each case has
that property.
"""
import functools
import math
from dataclasses import dataclass, field

import numpy as np

U = 2.0 ** -24
FLT_MAX = float(np.finfo(np.float32).max)
THREADS = 1024                         # kProjThreads
F32 = np.float32


def max_rounds(n):
    """csrc/project.cu hoyer_project: every round that does not end the loop zeroes one more coordinate."""
    return n + 2 if n < 100000 else 100002


def slices(x, dim):
    """(D, n) float32 view of the slices along `dim`, each in the kernel's element order e = o * inner + i."""
    x = np.asarray(x, F32)
    return np.ascontiguousarray(np.moveaxis(x, dim, 0).reshape(x.shape[dim], -1))


def unslice(s, shape, dim):
    """Inverse of slices()."""
    moved = list(shape)
    d = moved.pop(dim)
    return np.moveaxis(np.asarray(s).reshape([d] + moved), 0, dim)


def layout(shape, dim):
    outer = int(np.prod(shape[:dim], dtype=np.int64))
    inner = int(np.prod(shape[dim + 1:], dtype=np.int64))
    return outer, int(shape[dim]), inner


# ------------------------------------------------------------------------------------------------------------------
# float64 reference
# ------------------------------------------------------------------------------------------------------------------
@dataclass
class Ref:
    y: np.ndarray                      # float64 output (NaN where the algorithm divides 0 by 0)
    rounds: int
    zeroed: list                       # per round: the coordinates that round zeroes
    outcome: str                       # "ok", "nan" (a = 0), "zero-division" (every coordinate zeroed) or "overflow"


def proj64(x, k1, k2, exact=False, noise=None):
    """proj_func in float64.  x, k1, k2 are rounded to fp32 first unless `exact` (the classifier's perturbed inputs).
    noise: a numpy Generator; both terms of every element-wise sum (`x + shift`, `v + alphap w`) are then scaled by 1 +- u:
    the fp32 rounding of a sum is relative to its larger term, and `x + shift` cancels when k2 does not match x's scale."""
    if exact:
        s = np.asarray(x, np.float64).ravel()
        k1, k2 = float(k1), float(k2)
    else:
        s = np.asarray(x, F32).astype(np.float64).ravel()
        k1, k2 = float(F32(k1)), float(F32(k2))
    n = s.size
    def add(p, q):
        if noise is None:
            return p + q
        return p * (1 + U * noise.choice([-1.0, 1.0], size=n)) + q * (1 + U * noise.choice([-1.0, 1.0], size=n))
    v = add(s, (k1 - s.sum()) / n)
    zero = np.zeros(n, bool)
    zeroed, rounds = [], 0
    with np.errstate(all="ignore"):
        while True:
            live = n - int(zero.sum())
            if live == 0:                                   # nmf.py:32, k1 / 0
                return Ref(np.zeros(n), rounds, zeroed, "zero-division")
            rounds += 1
            m = k1 / live
            w = np.where(~zero, v - m, v)
            a, b, c = w @ w, 2 * (w @ v), v @ v - k2
            if max(b * b, abs(4 * a * c)) > FLT_MAX:        # fp32 (the reference's and the kernel's) gets inf - inf
                return Ref(v, rounds, zeroed, "overflow")
            alphap = (-b + math.sqrt(max(b * b - 4 * a * c, 0.0))) * 0.5 / a if a != 0 else float("nan")
            v = add(v, alphap * w)
            neg = v < 0
            zeroed.append(np.flatnonzero(neg & ~zero))
            if not neg.any():
                return Ref(v, rounds, zeroed, "nan" if np.isnan(v).any() else "ok")
            zero |= neg
            v = np.maximum(v, 0)
            live = n - int(zero.sum())
            if live == 0:                                   # nmf.py:46 divides by 0 too; :32 then raises
                return Ref(np.zeros(n), rounds, zeroed, "zero-division")
            v = np.maximum(add(v, (k1 - v.sum()) / live), 0)


def classify(x, k1, k2, seed=0, nperturb=4):
    """(class, float64 Ref, bar on |y - y64| for a stable slice, else None)."""
    ref = proj64(x, k1, k2)
    if ref.outcome != "ok":
        return "degenerate", ref, None
    s = np.asarray(x, F32).astype(np.float64).ravel()
    k1d, k2d = float(F32(k1)), float(F32(k2))
    g = np.random.default_rng(seed)
    spread = 0.0
    for _ in range(nperturb):
        r = g.choice([-1.0, 1.0], size=s.size)
        p = proj64(s * (1 + U * r), k1d * (1 + U * g.choice([-1.0, 1.0])), k2d * (1 + U * g.choice([-1.0, 1.0])), exact=True,
                   noise=g)
        if (p.outcome != "ok" or p.rounds != ref.rounds
                or any(not np.array_equal(a, b) for a, b in zip(p.zeroed, ref.zeroed))):
            return "unstable", ref, None
        spread = max(spread, float(np.abs(p.y - ref.y).max()))
    ymax = float(np.abs(ref.y).max())
    if 8 * spread > ymax / 32:                    # same zero sets, but the output moves by percents: no fp32 answer is closer
        return "unstable", ref, None
    return "stable", ref, 8 * spread + 4 * U * ymax


# ------------------------------------------------------------------------------------------------------------------
# the kernel's arithmetic
# ------------------------------------------------------------------------------------------------------------------
_LANE = np.arange(32)


def _butterfly(a):
    """a (..., 32): the xor-shuffle sums of block_sum3; every lane ends with the same value, lane 0's is returned."""
    for o in (16, 8, 4, 2, 1):
        a = a + a[..., _LANE ^ o]
    return a[..., 0]


def block_sum(t):
    """Sum of the float64 terms t[e] in the kernel's order: thread e % 1024 adds its terms in e order, then block_sum3."""
    n = t.size
    pad = (-n) % THREADS
    if pad:
        t = np.concatenate([t, np.zeros(pad)])
    per_thread = t.reshape(-1, THREADS).sum(axis=0) if t.size > THREADS else t      # row by row: sequential per column
    return float(_butterfly(_butterfly(per_thread.reshape(32, 32))[None, :])[0])


def _f(x):
    return F32(x)


def _fmaf(a, b, c):
    """fmaf on float32 arrays: the product is exact in double; the sum is rounded to double, then to fp32."""
    return (np.float64(a) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(F32)


def alphap_forms(af, bf, cf):
    """alphap from fp32 a, b, c as the kernel writes it, uncontracted and with each FMA contraction of the discriminant."""
    t1, t2 = _f(bf * bf), _f(_f(F32(4) * af) * cf)
    discs = (_f(t1 - t2), _fmaf(bf, bf, -t2)[()], _fmaf(-_f(F32(4) * af), cf, t1)[()])
    out = []
    for d in discs:
        d = np.fmax(d, F32(0))                       # fmaxf: a NaN discriminant (inf - inf, inf * 0) becomes 0
        out.append(_f(_f(_f(-bf + np.sqrt(F32(d))) * F32(0.5)) / af))
    return out


@dataclass
class Model:
    y: np.ndarray                      # fp32 output
    rounds: int
    exit: str                          # "converged" (anyneg == 0), "all-zeroed" (nzero >= n) or "max-rounds"
    zeroed: np.ndarray                 # the kernel's zeroed[] at exit
    alphas: list = field(default_factory=list)
    final: dict = field(default_factory=dict)      # last round: v, w, alphap (for the invariant bars)


def kernel_model(x, k1, k2, pick="plain", shift_ulp=0):
    """hoyer_project_kernel on one slice.  pick: which admissible alphap every round takes ("plain" = uncontracted at the
    rounded a, b, c; "fma1" / "fma2" = the contracted discriminants); shift_ulp moves every shift one ulp."""
    x = np.asarray(x, F32).ravel().copy()
    n = x.size
    k1d, k2d = float(F32(k1)), float(F32(k2))
    s0 = block_sum(x.astype(np.float64))

    def _shift(val):
        s = _f(val)
        for _ in range(abs(shift_ulp)):
            s = np.nextafter(s, F32(np.inf) if shift_ulp > 0 else F32(-np.inf))
        return s
    shift = _shift((k1d - s0) / n)
    clamp, nzero = False, 0
    zeroed = np.zeros(n, bool)
    alphas, final = [], {}
    with np.errstate(all="ignore"):
        for rnd in range(max_rounds(n)):
            m = _f(k1d / (n - nzero))
            v = (x + shift).astype(F32)
            if clamp:
                v = np.fmax(v, F32(0))               # fmaxf: NaN -> 0
            w = np.where(zeroed, v, (v - m).astype(F32)).astype(F32) if rnd > 0 else (v - m).astype(F32)
            w64, v64 = w.astype(np.float64), v.astype(np.float64)
            a, b, c = block_sum(w64 * w64), block_sum(w64 * v64), block_sum(v64 * v64)
            af, bf, cf = _f(a), _f(2.0 * b), _f(c - k2d)
            alphap = alphap_forms(af, bf, cf)[("plain", "fma1", "fma2").index(pick)]
            alphas.append(alphap)
            nv = _fmaf(alphap, w, v)
            neg = nv < 0
            zeroed |= neg
            nv[neg] = 0
            x = nv
            final = dict(v=v, w=w, alphap=alphap)
            if not neg.any():
                return Model(x, rnd + 1, "converged", zeroed, alphas, final)
            nzero = int(zeroed.sum())
            if nzero >= n:
                return Model(x, rnd + 1, "all-zeroed", zeroed, alphas, final)
            shift = _shift((k1d - block_sum(x.astype(np.float64))) / (n - nzero))
            clamp = True
    return Model(x, max_rounds(n), "max-rounds", zeroed, alphas, final)


FORMS = ("plain", "fma1", "fma2")


@dataclass
class FormBar:
    y: np.ndarray                      # fp32 output of this form
    bar: np.ndarray                    # per entry: spread over the shift-moved runs + 1 ulp of the entry
    ambiguous: np.ndarray              # entries zero in one run and not in another


@dataclass
class ModelBar:
    model: Model                       # the uncontracted form (the invariant bars' final round)
    forms: dict                        # form -> FormBar
    contraction_spread: float          # max |fma1/fma2 - plain|: what the compiler's choice alone moves

    @property
    def bar(self):
        return self.forms["plain"].bar

    def rel(self):
        """max over forms of max bar / max |y| on the finite entries: how much of the slice's scale a check leaves open."""
        out = 0.0
        for f in self.forms.values():
            fin = np.isfinite(f.y)
            if fin.any():
                out = max(out, float(f.bar[fin].max() / max(float(np.abs(f.y[fin]).max()), 1e-30)))
        return out


def model_bar(x, k1, k2):
    forms, cspread = {}, 0.0
    with np.errstate(invalid="ignore"):
        for pick in FORMS:
            nom = kernel_model(x, k1, k2, pick)
            y = nom.y.astype(np.float64)
            spread = np.zeros_like(y)
            amb = np.zeros(y.shape, bool)
            for sh in (-1, 1):
                t = kernel_model(x, k1, k2, pick, sh).y.astype(np.float64)
                d = np.abs(t - y)
                d[np.isnan(t) & np.isnan(y)] = 0
                spread = np.fmax(spread, d)
                amb |= (t == 0) != (y == 0)
            forms[pick] = FormBar(nom.y, spread + np.spacing(np.abs(nom.y)).astype(np.float64), amb)
            if pick == "plain":
                plain = nom
            else:
                d = np.abs(y - plain.y.astype(np.float64))
                d[np.isnan(y) & np.isnan(plain.y)] = 0
                cspread = max(cspread, float(np.nan_to_num(d, nan=np.inf).max()))
    return ModelBar(plain, forms, cspread)


def invariant_bars(mb, k1, k2):
    """Bars on |sum y - k1| and |sum y^2 - k2| from the model's final round: fp32 rounding of `v = x + shift` and of the
    fmaf update (u per element each, against sum|v| + |alphap| sum|w|), the spread over the forms, and
    the model's own distance from k1, k2 (the discriminant is clamped at 0 when no real root exists)."""
    f = mb.model.final
    v, w = f["v"].astype(np.float64), f["w"].astype(np.float64)
    al = abs(float(f["alphap"]))
    y = mb.model.y.astype(np.float64)
    mag = np.abs(v) + al * np.abs(w)
    k1d, k2d = float(F32(k1)), float(F32(k2))
    bar = mb.bar
    for f in mb.forms.values():
        bar = np.fmax(bar, np.abs(f.y.astype(np.float64) - y) + f.bar)
    b1 = 8 * U * mag.sum() + bar.sum() + abs(y.sum() - k1d) + 4 * U * abs(k1d)
    b2 = 16 * U * (mag * mag).sum() + 2 * (np.abs(y) * bar).sum() + abs((y * y).sum() - k2d) + 4 * U * abs(k2d)
    return b1, b2


# ------------------------------------------------------------------------------------------------------------------
# the catalogue
# ------------------------------------------------------------------------------------------------------------------
def l1_of(n, s):
    """nmf.py:461 / trainer.py:175: the L1 norm of a unit-L2 vector of n entries with Hoyer sparseness s."""
    return math.sqrt(n) * (1 - s) + s


def _data(kind, D, n, seed):
    g = np.random.default_rng(seed)
    i = np.arange(n, dtype=np.float64)
    if kind == "rand":
        s = g.random((D, n))
    elif kind == "abs_normal":
        s = np.abs(g.standard_normal((D, n))) + 1e-3
    elif kind == "lognormal":
        s = np.exp(3.0 * g.standard_normal((D, n)))
    elif kind == "normal":                     # a gradient-step trial: mixed signs
        s = g.standard_normal((D, n))
    elif kind == "negative":                   # a trial that overshot: every entry negative
        s = -(g.random((D, n)) + 0.1)
    elif kind == "decays":                     # slow structured decays: one coordinate (or a few) leaves per round
        forms = [1 - i / n, np.sqrt(1 - i / n), np.log(n + 1 - i), np.exp(-i / (n / 8)), (1 - i / n) ** 2]
        s = np.stack([forms[j % len(forms)] for j in range(D)])
    elif kind == "ties":                       # 8 levels, each n / 8 times: the threshold falls between two tied groups
        s = np.stack([np.floor(g.permutation(n) * 8 / n) + 1 for _ in range(D)])
    elif kind == "n1":                         # n = 1 with k1 - x exact: v = m, a = 0
        s = np.full((D, n), 0.5)
    elif kind == "const":                      # uniform support from round 0: a = 0
        s = np.full((D, n), 1.0)
    elif kind == "two_valued":                 # the low values are zeroed, the survivors are uniform: a = 0 in round 2
        s = np.where(i < n // 2, 1.0, 4.0)[None, :].repeat(D, 0)
    elif kind == "all_zeroed":                 # three entries 2^-18 above the fourth: fp32 sends all four below 0
        s = np.array([[1 + 2.0 ** -18] * 3 + [1.0]] * D)
    elif kind == "zero_division":              # float64 zeroes every coordinate in round 2; fp32 keeps some
        s = np.array([[1 + 2.0 ** -15, 1 + 2.0 ** -16] * 3] * D)
    else:
        raise ValueError(kind)
    return s.astype(F32)


@dataclass(frozen=True)
class Case:
    name: str
    why: str                            # the branch or edge of the kernel this case exists for
    shape: tuple
    dim: int
    data: str
    k: str                              # "norm": k2 = |x|^2, k1 = L1(s) |x|; "unit": k2 = 1, k1 = L1(s); "feasible": x's own
    sp: tuple = (0.5,)                  # sparseness per slice (cycled)
    cls: str = "stable"                 # the conditioning classes its slices may take, "|"-separated
    seed: int = 0
    k_override: tuple = None            # explicit (k1, k2) per slice (degenerate cases)

    @property
    def D(self):
        return self.shape[self.dim]

    @property
    def n(self):
        return int(np.prod(self.shape, dtype=np.int64)) // self.D

    @property
    def layout(self):
        return layout(self.shape, self.dim)


def _slice_data(c):
    """(D, n) fp32 slices and the D fp32 k1, k2 of case c."""
    s = _data(c.data, c.D, c.n, c.seed)
    if c.k_override is not None:
        k1 = np.array([c.k_override[0]] * c.D, F32)
        k2 = np.array([c.k_override[1]] * c.D, F32)
        return s, k1, k2
    sp = np.array([c.sp[j % len(c.sp)] for j in range(c.D)])
    s64 = s.astype(np.float64)
    if c.k == "feasible":
        return s, s64.sum(1).astype(F32), (s64 * s64).sum(1).astype(F32)
    l1 = np.array([l1_of(c.n, q) for q in sp])
    if c.k == "unit":
        return s, l1.astype(F32), np.ones(c.D, F32)
    nrm = np.sqrt((s64 * s64).sum(1))
    return s, (l1 * nrm).astype(F32), (nrm * nrm).astype(F32)


def case_tensor(c):
    """(x of c.shape, k1, k2) as fp32 numpy arrays."""
    s, k1, k2 = _slice_data(c)
    return np.ascontiguousarray(unslice(s, c.shape, c.dim)).astype(F32), k1, k2


SP_SPREAD = (0.1, 0.5, 0.8, 0.9, 0.95)

CASES = [
    # slice lengths around the 1024-thread stride, one per residue class of interest
    Case("n1", "n = 1: the survivor is uniform, a = 0 -> NaN", (4, 1), 0, "n1", "norm", cls="degenerate",
         k_override=(1.0, 1.0)),
    Case("n2", "n = 2: one thread per element, one zeroing round", (3, 2), 0, "rand", "norm", (0.3, 0.6, 0.9), seed=2),
    Case("n3", "n = 3", (3, 2), 1, "abs_normal", "norm", (0.4, 0.8), seed=3),
    Case("n31", "n = 31: one partial warp", (31, 5), 1, "abs_normal", "norm", SP_SPREAD, seed=31),
    Case("n32", "n = 32: one full warp", (6, 32), 0, "abs_normal", "norm", SP_SPREAD, seed=32),
    Case("n1023", "n = 1023: every thread but the last", (1023, 4), 1, "abs_normal", "norm", SP_SPREAD, seed=1023),
    Case("n1024", "n = 1024: exactly one element per thread", (1024, 5), 1, "abs_normal", "norm", SP_SPREAD, seed=1024),
    Case("n1025", "n = 1025: thread 0 takes a second element", (3, 1025), 0, "rand", "norm", (0.6, 0.9, 0.3), seed=1025),
    Case("n2047", "n = 2047: the second stride pass one short", (2047, 3), 1, "abs_normal", "norm", (0.7, 0.2, 0.9),
         seed=2047),
    Case("n4097", "n = 4097: the fifth stride pass holds one element", (17, 4, 241), 1, "abs_normal", "norm", SP_SPREAD,
         seed=4097),
    Case("n65537", "n = 65537: 65 elements on thread 0, 64 on the rest", (65537, 3), 1, "abs_normal", "norm",
         (0.85, 0.5, 0.95), seed=7),
    Case("n100001", "n = 100001: max_rounds takes its 100002 cap", (2, 100001), 0, "abs_normal", "norm", (0.9, 0.6),
         seed=100001),
    Case("n2p20", "n = 2^20: 1024 elements per thread", (2, 1 << 20), 0, "abs_normal", "norm", (0.8, 0.97), cls="unstable",
         seed=20),
    # layouts: (outer, D, inner) from 2-D to 5-D tensors along dim 0..3
    Case("h_cfg1", "the H of BASELINE configs[1]: inner = 1, stride 64", (65536, 64), 1, "abs_normal", "norm",
         (0.85, 0.3, 0.6, 0.95), cls="stable|unstable", seed=11),
    Case("nmfd_w", "NMFD W (C, R, T) along dim 1", (257, 8, 16), 1, "abs_normal", "norm", SP_SPREAD, seed=41),
    Case("nmfd_h", "NMFD H (B, R, L) along dim 1", (3, 5, 1365), 1, "rand", "norm", SP_SPREAD, seed=42),
    Case("nmf3d_w", "NMF3D W (C, R, K1, K2, K3) along dim 1", (9, 4, 5, 6, 7), 1, "abs_normal", "norm", SP_SPREAD,
         seed=43),
    Case("dim2_4d", "4-D along dim 2: outer = 6, inner = 7", (2, 3, 5, 7), 2, "abs_normal", "norm", SP_SPREAD, seed=44),
    Case("dim3_4d", "4-D along dim 3: inner = 1, outer = 105", (3, 5, 7, 6), 3, "abs_normal", "norm", SP_SPREAD, seed=45),
    Case("dim0_3d", "3-D along dim 0: outer = 1, inner = 600", (5, 20, 30), 0, "rand", "norm", SP_SPREAD, seed=46),
    Case("dim2_5d", "5-D along dim 2", (3, 4, 6, 5, 11), 2, "abs_normal", "norm", SP_SPREAD, seed=47),
    Case("dim3_5d", "5-D along dim 3", (2, 3, 4, 9, 13), 3, "abs_normal", "norm", SP_SPREAD, seed=48),
    # targets
    Case("sp_low", "sparseness 0.001: alphap near -1, the discriminant near 0", (4096, 3), 1, "rand", "norm",
         (1e-3, 5e-3, 2e-2), seed=50),
    Case("sp_high", "sparseness 0.999: few survivors", (3, 4096), 0, "abs_normal", "norm", (0.999, 0.99, 0.995),
         seed=51),
    Case("negative", "gradient-step trials with negative entries", (2000, 4), 1, "normal", "norm", (0.3, 0.6, 0.8, 0.9),
         seed=52),
    Case("all_negative", "an all-negative trial", (3, 1500), 0, "negative", "norm", (0.2, 0.5, 0.8), seed=53),
    Case("feasible", "already feasible: one round, the output is the input", (3, 2500), 0, "rand", "feasible", seed=54),
    Case("ties", "8 tied levels: whole groups reach the zeroing threshold together", (4, 4096), 0, "ties", "norm",
         (0.3, 0.4, 0.5, 0.6), seed=55),
    Case("tie_top", "8 tied levels, only the top group survives: uniform support, a = 0", (2, 4096), 0, "ties", "norm",
         (0.7,), cls="degenerate", seed=56),
    Case("decays", "structured decays: 12 to 14 rounds", (5, 4096), 0, "decays", "norm", (0.95, 0.97, 0.99, 0.97, 0.98)),
    Case("many_rounds", "the most rounds found (16): linear and sqrt decays, n = 16384, sparseness 0.999 / 0.995; a search "
         "over power, exponential, log and harmonic decays, n in {1024, 4096, 16384} and sparseness 0.8-0.999 found no more",
         (2, 16384), 0, "decays", "norm", (0.999, 0.995)),
    # sparse_fit's initial projection: k2 = 1 on an unnormalised W0 / H0
    Case("init_rand", "sparse_fit's first projection, k2 = 1 on torch.rand-like W0", (500, 6), 1, "rand", "unit",
         (0.5, 0.7), cls="stable|unstable", seed=60),
    Case("init_lognormal", "sparse_fit's first projection, k2 = 1 on a lognormal (sigma 3) H0", (3, 4096), 0, "lognormal",
         "unit", (0.5, 0.8, 0.3), cls="unstable", seed=61),
    # degenerate slices
    Case("const", "a constant slice: a = w.w = 0 in round 1", (3, 64), 0, "const", "norm", cls="degenerate",
         k_override=(32.0, 16.0)),
    Case("two_valued", "the low half is zeroed, the survivors are uniform: a = 0 in round 2", (2, 64), 0, "two_valued",
         "norm", (0.5,), cls="degenerate", k_override=(8.0, 64.0)),
    Case("all_zeroed", "near-uniform: the fp32 round zeroes every coordinate, the nzero >= n exit", (2, 4), 0,
         "all_zeroed", "norm", cls="unstable", k_override=(1.0, 1.0)),
    Case("zero_division", "near-uniform: the reference divides by zero in round 2", (2, 6), 0, "zero_division", "norm",
         cls="degenerate", k_override=(1.2235201265201974, 1.0)),
]
BY_NAME = {c.name: c for c in CASES}

# One slice length per residue class mod 1024 the kernel's stride loop distinguishes.
N_COVER = (1, 2, 3, 31, 32, 1023, 1024, 1025, 2047, 4097, 65537, 100001, 1 << 20)

# The many-slice case: D * n, (o * D + j) * inner and j * n past 2^31.  Slices repeat 8 patterns (8 distinct k1, k2) so the
# CPU references stay 8 slices; identical slices must give bit-identical outputs.
HUGE = Case("huge", "D n > 2^31: j n in zeroed_ws and (o D + j) inner past int32", (4096, 8 * 65537), 1, "abs_normal",
            "norm", (0.5, 0.6, 0.7, 0.8, 0.9, 0.95, 0.3, 0.85), seed=77)
HUGE_PATTERNS = 8


def huge_patterns():
    """(4096, 8) pattern columns and their 8 k1, k2: column j of the huge case is pattern j % 8."""
    c = Case("huge_p", HUGE.why, (4096, HUGE_PATTERNS), 1, HUGE.data, HUGE.k, HUGE.sp, seed=HUGE.seed)
    return case_tensor(c)


@functools.lru_cache(maxsize=None)
def analyse(name):
    """Per slice of case `name`: class, float64 Ref, float64 bar, ModelBar.  Cached: the CPU and GPU tests share it."""
    c = BY_NAME[name] if name != "huge" else None
    if c is None:
        x, k1, k2 = huge_patterns()
        s = slices(x, 1)
    else:
        s, k1, k2 = _slice_data(c)
    out = []
    for j in range(s.shape[0]):
        cls, ref, bar64 = classify(s[j], k1[j], k2[j], seed=j)
        out.append(dict(cls=cls, ref=ref, bar64=bar64, mb=model_bar(s[j], k1[j], k2[j]), x=s[j], k1=k1[j], k2=k2[j]))
    return out
