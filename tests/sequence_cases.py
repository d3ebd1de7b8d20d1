"""Scripted call sequences on ONE long-lived engine context, checked call by call against float64.

TEST INFRASTRUCTURE ONLY.  `fit()`, `BetaMu.step`, PLCA and the sharded fit keep a context alive for hundreds of calls, and
the workspace cache hands contexts from one fit to the next, so every call after the first runs on state left behind by
earlier ones: the fp16 operand copies and their exponents, kappa, the dirty flags, the prefetched W numerators, the cached
V-only loss term, the AUTO mode's tensor-core switch.  A harness run drives one context through a
sequence of steps; before every step it reads the factors back, and it checks that step's output against a float64
evaluation of that one step FROM THOSE FACTORS.  Errors do not build up, so the per-call bars of the term tests apply
unchanged (tests/tc_model.py, tests/f32_cases.py).

A step is a tuple (op, *args):
    ("update_w" | "update_h", beta, gamma, l1, l2)     one factor update
    ("raw", which, beta)                              the raw terms of one update (`raw_terms`)
    ("loss", beta) / ("prefetch", beta)               the loss pass / the loss folded into the next W update's contraction
    ("iterate", beta, gamma, l1, l2)                  iterate(1): one W and one H update in one call
    ("rescale", f)                                    W *= f and H /= f in place (W H unchanged), then sync()
    ("shard", beta, gamma, l1, l2)                    w_partial, that buffer as the "all-reduced" sum into w_apply
    ("target", name)                                  set_target of another target of the sequence on the same context

`simulate` restates, on the host, the state machine of the library (csrc/capi.cu, csrc/tc_nmf.cu, csrc/tc_nmfd.cu) that
decides which path a call takes and which cached state it may reuse.  It yields per step the path that must run, whether a W
update must reuse the prefetched numerators, and the state transitions the step exercises; tests/test_sequence_harness.py
checks on the CPU that the sequences below reach every transition in TRANSITIONS.
"""
from dataclasses import dataclass, field

import torch

TRANSITIONS = [
    "prefetch reused", "prefetch dropped", "dirty from the fp32 path", "beta change without refresh",
    "tc_off flipped", "sparse to dense",
    "NMFD refresh after an fp32 update",
]
SCALES = [-16, -12, 0, 12, 20]


@dataclass
class Seq:
    name: str
    kind: str                     # "nmf" | "nmfd" | "sparse" (a sparse engine, then a dense f32 engine on its context)
    shape: tuple                  # nmf: (N, C, R); nmfd: (B, C, L, R, T)
    precision: str
    steps: list
    targets: dict = field(default_factory=dict)      # name -> (scale exponent, heavy-tailed)
    tc: bool = True               # runs on the tensor cores at all (the scale sweep applies)


def _upd(w, beta, gamma=1.0, l1=0.0, l2=0.0):
    return ("update_w" if w else "update_h", beta, gamma, l1, l2)


UW = lambda beta, *a: _upd(True, beta, *a)           # noqa: E731
UH = lambda beta, *a: _upd(False, beta, *a)          # noqa: E731
G8 = 0.8

FIT_STEPS = [
    UW(1), UH(1), ("loss", 1), ("prefetch", 1), UW(1),                 # prefetch reused
    ("prefetch", 1), UH(1), UW(1),                                     # dropped: the H contraction overwrote it
    ("raw", 0, 1), ("raw", 1, 1), ("prefetch", 1), ("raw", 0, 1), UW(1),
    # iterations across both absmax parities, then with a new gamma and new l1
    ("iterate", 1, 1.0, 0.0, 0.0), ("iterate", 1, 1.0, 0.0, 0.0), ("iterate", 1, 1.0, 0.0, 0.0), ("iterate", 1, 1.0, 0.0, 0.0),
    ("iterate", 1, G8, 0.0, 0.0), ("iterate", 1, G8, 0.0, 0.0), ("iterate", 1, G8, 0.0, 0.0), ("iterate", 1, G8, 0.0, 0.0),
    ("iterate", 1, G8, 1e-3, 0.0), ("iterate", 1, G8, 1e-3, 0.0),
    ("prefetch", 1), ("rescale", 2.0 ** -12), UW(1),                  # in-place edit after a prefetch: no reuse
    ("loss", 1), UH(1, G8, 1e-3, 1e-3), ("prefetch", 1), UW(1, G8, 1e-3, 1e-3), ("loss", 1),
]

MIXED_STEPS = [
    UW(1), UH(2), UW(1), ("raw", 1, 0.5), UH(0.5), ("loss", 0.5), UW(0), ("raw", 0, 3), UH(3), ("loss", 3),
    UW(2), ("raw", 1, 0), ("loss", 0), UH(1), ("raw", 0, 0.5), UW(0.5), UH(2), ("loss", 2), ("raw", 1, 1),
    ("iterate", 2, 1.0, 0.0, 0.0), ("raw", 0, 3), ("iterate", 0.5, 1.0, 0.0, 0.0), UH(0), ("loss", 1),
]

PATH_STEPS = [                                       # R in 65..128: two-output betas run on the fp32 kernels
    UW(1), UH(0.5), UW(2), ("raw", 0, 0.5), UH(1), UW(1), UW(3), ("loss", 2), UH(2), ("raw", 1, 1), ("prefetch", 1),
    UH(0), UW(1), ("raw", 0, 2), ("loss", 0.5), UH(1),
]

TARGET_STEPS = [
    UW(1), ("loss", 0.5), UH(2), ("target", "rescaled"), ("loss", 0.5), UW(2), UH(1), ("raw", 0, 0.5),
    ("target", "heavy"), UW(1), ("loss", 0.5), UH(2), ("target", "base"), ("loss", 0.5), UW(2), UH(1), ("loss", 1),
]

SHARD_STEPS = [
    ("shard", 1, 1.0, 0.0, 0.0), UH(1), ("shard", 1, 1.0, 0.0, 0.0), UH(1),
    ("shard", 0.5, 1.0, 0.0, 0.0), UH(0.5), ("shard", 0.5, 1.0, 0.0, 0.0), UH(0.5),
    ("shard", 2, 1.0, 0.0, 0.0), UH(2), ("shard", 2, 1.0, 0.0, 0.0), UH(2), ("loss", 2),
]

NMFD_STEPS = [
    UW(1), UH(1), ("raw", 0, 1), ("loss", 1), UW(2), UH(1), ("raw", 1, 1), UH(2), UW(1), ("loss", 2),
    ("rescale", 2.0 ** -12), ("raw", 0, 1), UH(1), UW(1), ("loss", 1),
]

SPARSE_STEPS = [                                     # a sparse target, then a dense one on the same (cached) context
    UW(1), UH(2), ("raw", 0, 1), ("raw", 1, 2), ("loss", 2), ("loss", 1), ("target", "dense"),
    UW(1), UH(2), ("raw", 0, 2), ("loss", 1), ("loss", 0.5), UW(0.5),
]


def sequences():
    """Every sequence of the suite (the tensor-core ones at one scale; the sweep multiplies them)."""
    return [
        Seq("fit-f16", "nmf", (300, 260, 40), "f16", FIT_STEPS),
        Seq("fit-split", "nmf", (300, 260, 40), "f16_split", FIT_STEPS),
        Seq("mixed-f16", "nmf", (300, 260, 40), "f16", MIXED_STEPS),
        Seq("mixed-split", "nmf", (300, 260, 40), "f16_split", MIXED_STEPS),
        Seq("paths-r100", "nmf", (300, 260, 100), "f16", PATH_STEPS),
        Seq("target", "nmf", (300, 260, 40), "auto", TARGET_STEPS,
            targets={"base": (0, False), "rescaled": (16, False), "heavy": (0, True)}),
        Seq("shard", "nmf", (300, 260, 40), "f16", SHARD_STEPS),
        Seq("nmfd", "nmfd", (1, 20, 300, 4, 200), "f16", NMFD_STEPS),
        Seq("sparse", "sparse", (300, 260, 40), "f32", SPARSE_STEPS, targets={"dense": (0, False)}, tc=False),
    ]


def scale_tag(s):
    return f"s{s:+d}"


def by_name(name):
    return next(s for s in sequences() if s.name == name)


# ---- the host-side state machine -------------------------------------------------------------------------------------------
def tc_supports(seq, beta):
    """tc_supports_beta (csrc/tc_nmf.cu) / tc_nmfd_supported (csrc/tc_nmfd.cu)."""
    if seq.kind == "nmfd":
        return beta == 1
    return beta in (1, 2) or seq.shape[2] <= 64


@dataclass
class StepPlan:
    step: tuple
    path: str                     # "tc" | "f32": the kernels of the call's contraction ("shard": of w_partial)
    reported: str = "f32"         # what precision_for(beta) reports: "tc" wherever the context serves beta at all
    reuse: bool = False           # update_w: skips its contraction (prefetched numerators)
    refresh: bool = False         # a tensor-core step that first rebuilds dirty operand copies
    events: list = field(default_factory=list)


def simulate(seq):
    """[StepPlan] of the sequence: the path of every call, prefetch reuse, and the state transitions it exercises."""
    has_tc = seq.precision != "f32" and seq.kind != "sparse"
    sparse = seq.kind == "sparse"
    tc_off = False
    w_pending = False
    dirty = {"w": True, "h": True}
    exps_beta = None
    nmfd_fp32_since_tc = False
    out = []

    def use_tc(beta):
        return has_tc and not tc_off and not sparse and tc_supports(seq, beta)

    def contraction(beta, ev, factors_read=True):
        """A tensor-core contraction at beta: refresh what is dirty (publishing at beta), then the kernel."""
        nonlocal exps_beta, nmfd_fp32_since_tc
        if seq.kind == "nmfd":
            if nmfd_fp32_since_tc:
                ev.append("NMFD refresh after an fp32 update")
            nmfd_fp32_since_tc = False
            return
        if dirty["w"] or dirty["h"]:
            exps_beta = beta
            dirty["w"] = dirty["h"] = False
        elif beta != 1 and exps_beta != beta:
            ev.append("beta change without refresh")
            exps_beta = beta

    for st in seq.steps:
        op = st[0]
        ev = []
        plan = StepPlan(st, "f32")
        beta = st[2] if op == "raw" else (st[1] if op in ("update_w", "update_h", "iterate", "shard", "loss", "prefetch") else None)
        if beta is not None:
            plan.path = plan.reported = "tc" if use_tc(beta) else "f32"
            if op in ("shard", "raw") and beta == 2 and seq.kind == "nmf":
                plan.path = "f32"                   # no tensor-core beta-2 raw terms: the fp32 kernels (w_apply stays tc)
        reuse = (op == "update_w" and plan.path == "tc" and beta == 1 and w_pending and not (dirty["w"] or dirty["h"]))
        plan.refresh = plan.path == "tc" and seq.kind == "nmf" and (dirty["w"] or dirty["h"])
        # every update contraction (not the loss pass) overwrites the prefetched numerators, and so does a new target
        clears = op == "target" or (plan.path == "tc" and op in ("update_w", "update_h", "iterate", "shard", "raw", "prefetch"))
        if w_pending and clears and not reuse:
            ev.append("prefetch dropped")
        if clears:
            w_pending = False
        if op == "rescale":                         # in-place edit + sync(): both operand copies are stale
            if has_tc and seq.kind == "nmf":
                dirty["w"] = dirty["h"] = True
            nmfd_fp32_since_tc = False              # (NMFD: a full refresh follows anyway)
        elif op == "target":
            heavy = seq.targets[st[1]][1]
            if sparse:
                ev.append("sparse to dense")
                sparse = False
            new_off = has_tc and seq.precision == "auto" and heavy
            if new_off != tc_off:
                ev.append("tc_off flipped")
            tc_off = new_off
            dirty["w"] = dirty["h"] = True
        elif plan.path == "f32":
            writes = op in ("update_w", "update_h", "iterate") or (op == "raw" and seq.kind == "nmfd")
            if writes and has_tc and not tc_off and not sparse:
                ev.append("dirty from the fp32 path")
                if seq.kind == "nmfd":
                    nmfd_fp32_since_tc = True
                else:
                    dirty["w" if op == "update_w" else "h"] = True
                    if op == "iterate":
                        dirty["w"] = True
            if op == "shard" and use_tc(beta):      # beta 2: w_apply's ratio stage republishes W at this beta
                dirty["w"] = False
                exps_beta = beta
        elif op in ("update_w", "update_h"):
            if reuse:
                plan.reuse = True
                ev.append("prefetch reused")
            else:
                contraction(beta, ev)
            exps_beta = beta
        elif op == "iterate":
            contraction(beta, ev)
            exps_beta = beta
        elif op == "shard":
            contraction(beta, ev)
            dirty["w"] = False
            exps_beta = beta
        elif op == "raw" or seq.kind == "nmfd":
            contraction(beta, ev)
        else:                                       # the loss pass: refreshes what is dirty, reads no beta exponent
            if dirty["w"] or dirty["h"]:
                exps_beta = beta
                dirty["w"] = dirty["h"] = False
            if op == "prefetch" and beta == 1 and seq.precision != "f16_split":
                w_pending = True
        plan.events = ev
        out.append(plan)
    return out


def transitions_reached(seqs):
    """{transition: [sequence names reaching it]}"""
    got = {t: [] for t in TRANSITIONS}
    for s in seqs:
        for p in simulate(s):
            for e in p.events:
                if s.name not in got[e]:
                    got[e].append(s.name)
    return got


# ---- data ------------------------------------------------------------------------------------------------------------------
def fitted_data(seq, scale=0, unbalanced=0, seed=0):
    """(targets {name: V}, W, H) with W H ~ V: V = (H W^T)(1 + 0.1 noise) 2^scale and the factors matched to it, each by
    2^(scale / 2) (W further by 2^unbalanced, H by 2^-unbalanced).  A roughly fitted model is what long-lived contexts see,
    and the residual V - W H is then ~10% of V: the tile the beta-2 kernel scales by exps[4]."""
    g = torch.Generator().manual_seed(seed + 1000 * (seq.shape[-1] % 97))
    if seq.kind == "nmfd":
        B, C, L, R, T = seq.shape
        W = torch.rand(C, R, T, generator=g) + 0.1
        H = torch.rand(B, R, L - T + 1, generator=g) + 0.1
        from tc_model import nmfd_reconstruct
        S = nmfd_reconstruct(H.double(), W.double())
    else:
        N, C, R = seq.shape
        W = torch.rand(C, R, generator=g) + 0.1
        H = torch.rand(N, R, generator=g) + 0.1
        S = H.double() @ W.double().t()
    m = float(S.mean())
    W = W / m
    S = S / m
    half = 2.0 ** (scale / 2)
    W = (W * half * 2.0 ** unbalanced).float()
    H = (H * half * 2.0 ** -unbalanced).float()

    def target(s, heavy, salt):
        gg = torch.Generator().manual_seed(seed + salt)
        V = S * (1 + 0.1 * (2 * torch.rand(S.shape, generator=gg, dtype=torch.float64) - 1))
        if heavy:                                    # max / mean > 64: AUTO moves to the fp32 kernels
            V.view(-1)[torch.randperm(V.numel(), generator=gg)[:5]] *= 400
        return (V * 2.0 ** (scale + s)).float()
    targets = {"V": target(0, False, 1)}
    for i, (name, (s, heavy)) in enumerate(sorted(seq.targets.items())):
        targets[name] = target(s, heavy, 2 + i)
    if seq.kind == "sparse":
        V = targets["V"]
        keep = torch.rand(V.shape, generator=g) < 0.3
        targets["V"] = (V * keep).to_sparse().coalesce()
    return targets, W, H



# ---- the runner --------------------------------------------------------------------------------------------------------------
def call(eng, st):
    """Run one step on an engine; returns what the step outputs besides the factors."""
    op = st[0]
    if op in ("update_w", "update_h"):
        getattr(eng, op)(*st[1:])
    elif op == "raw":
        return tuple(t.clone() for t in eng.raw_terms(st[1], st[2]))
    elif op == "loss":
        return eng.loss(st[1])
    elif op == "prefetch":
        return eng.loss_prefetch_w(st[1]) if hasattr(eng, "loss_prefetch_w") else eng.loss(st[1])
    elif op == "iterate":
        if hasattr(eng, "iterate"):
            eng.iterate(1, *st[1:])
        else:
            eng.update_w(*st[1:])
            eng.update_h(*st[1:])
    elif op == "rescale":
        eng.W.mul_(st[1])
        eng.H.div_(st[1])
        eng.sync()
    elif op == "shard":
        buf = eng.w_partial(st[1]).clone()
        eng.w_apply(buf, *st[1:])
        return buf
    return None


def run(seq, eng, check, set_target=None, measure=None):
    """Drive `eng` through the steps of `seq`.  Before each step the factors are read back; `check(i, plan, eng, before,
    out)` then compares the step's output with float64 from `before` and returns its worst err / bar.  A ("target", name)
    step calls `set_target(eng, name)`, which returns the engine to go on with.  `measure(plan, run_step)`, if given, runs
    each step (run_step()) and may observe it: launch counts, a profile.  Returns [(step index, op, err / bar)]."""
    res = []
    for i, plan in enumerate(simulate(seq)):
        st = plan.step
        if st[0] == "target":
            eng = set_target(eng, st[1])
            continue
        before = (eng.W.detach().clone(), eng.H.detach().clone())
        out = measure(plan, lambda: call(eng, st)) if measure else call(eng, st)
        res.append((i, st[0], check(i, plan, eng, before, out)))
    return eng, res


def terms64(kind, V, W, H, which, beta):
    """(numerator, denominator) of one update in float64 (the oracle's phi and contractions)."""
    from oracle_engine import OracleNmfdEngine, OracleNmfEngine
    cls = OracleNmfEngine if kind != "nmfd" else OracleNmfdEngine
    return cls(V.double().cpu(), W.double().cpu(), H.double().cpu()).raw_terms(which, beta)


def recon64(kind, W, H):
    from oracle import mu_oracle as orc
    H, W = H.double().cpu(), W.double().cpu()
    return orc.nmfd_reconstruct(H, W) if kind == "nmfd" else orc.nmf_reconstruct(H, W)


def two_output(beta):
    return beta not in (1, 2)


def rtol_terms(beta, rtol):
    """Float64 bars of a numerator / denominator (tests/test_gpu_tc_terms.py: two-output tiles carry |beta - 2|, |beta - 1|
    times the relative error of S)."""
    if not two_output(beta):
        return rtol, rtol
    return rtol * max(1, abs(beta - 2)), rtol * max(1, abs(beta - 1))


def update64(kind, V, W, H, which, st):
    """The factor one update step must produce from (W, H), float64, and its multiplier."""
    import f32_cases as fc
    beta, gamma, l1, l2 = st[1:]
    num, den = terms64(kind, V, W, H, which, beta)
    p = (W if which == 0 else H).double().cpu()
    if beta == 1:
        den = den.reshape((1, -1) + (1,) * (p.dim() - 2))
    return fc.ratio64(p, num, den, gamma, l1, l2, beta == 1)


def loss64(kind, V, W, H, beta):
    """(float64 loss, the sum of the absolute values of its pieces)."""
    import f32_cases as fc
    term, M = fc.loss_pieces(beta, recon64(kind, W, H).reshape(-1), V.double().cpu().reshape(-1), 2.0 ** -23)
    return float(term.sum()), float(M.sum())


def rel_err(got, want):
    got, want = got.double().cpu(), want.double().cpu()
    return float(((got - want).abs() / want.abs()).max())


def float64_check(seq, V, rtol=1.25e-3, loss_rel=2.0 ** -11):
    """The float64 check of every step at the f16 bars (no rounding model): what tests/test_sequence_harness.py runs on
    the CPU.  Returns check(i, plan, eng, before, out) for `run`."""
    def check(i, plan, eng, before, out):
        W0, H0 = before
        st = plan.step
        op, tag = st[0], f"{seq.name}[{i}] {st}"
        if op == "raw":
            which, beta = st[1:]
            num, den = terms64(seq.kind, V, W0, H0, which, beta)
            rn, rd = rtol_terms(beta, rtol)
            e = rel_err(out[0], num) / rn
            e = max(e, rel_err(out[1], den.reshape(-1) if beta == 1 else den) / (1e-5 if beta == 1 else rd))
        elif op in ("loss", "prefetch"):
            beta = st[1]
            val, M = loss64(seq.kind, V, W0, H0, beta)
            g = max(1.0, abs(beta), abs(beta - 1))
            e = abs(out - val) / ((loss_rel * g + 2.0 ** -12) * M)
        elif op in ("update_w", "update_h", "iterate", "shard"):
            beta, gamma = st[1], st[2]
            rn, rd = rtol_terms(beta, rtol)
            bar = gamma * (rn + (rd if beta != 1 else 1e-5)) + 1e-5
            if op == "shard":
                num, den = terms64(seq.kind, V, W0, H0, 0, beta)
                e = rel_err(out[:num.numel()], num.reshape(-1)) / rn
            else:
                e = 0.0
            whiches = (0, 1) if op == "iterate" else ((0,) if op in ("update_w", "shard") else (1,))
            for which in whiches:
                Wb = W0 if which == 0 else eng.W          # iterate: the H update starts from the new W
                want, _ = update64(seq.kind, V, Wb, H0, which, (None,) + tuple(st[1:]))
                e = max(e, rel_err(eng.W if which == 0 else eng.H, want) / bar)
        else:
            return 0.0
        assert e <= 1.0, f"{tag}: {e:.2f} x the float64 bar"
        return e
    return check
