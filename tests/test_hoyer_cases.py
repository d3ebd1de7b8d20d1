"""CPU tests of the Hoyer projection cases (tests/hoyer_cases.py): every case has the property it is listed for, the model of
the kernel's arithmetic and the fp32 oracle are each within the conditioning bar of float64 on the stable cases, the three
references agree with the reference's own outputs (tests/golden/reference_hoyer.npz), and the bars are not loose."""
import os

import numpy as np
import pytest
import torch

import hoyer_cases as hc
from conftest import GOLDEN
from oracle import hoyer_oracle as hoy

NAMES = [c.name for c in hc.CASES]


@pytest.mark.parametrize("name", NAMES)
def test_case_has_its_property(name):
    c = hc.BY_NAME[name]
    A = hc.analyse(name)
    classes = {a["cls"] for a in A}
    assert classes <= set(c.cls.split("|")), (name, classes)
    outer, D, inner = c.layout
    assert outer * D * inner == int(np.prod(c.shape)) and D == len(A) and c.n == outer * inner
    for a in A:
        m = a["mb"].model
        assert m.exit != "max-rounds" and m.rounds <= hc.max_rounds(c.n)
        if a["cls"] != "degenerate":
            assert a["ref"].outcome == "ok"
    if name == "all_zeroed":
        assert all(a["mb"].model.exit == "all-zeroed" and not a["mb"].model.y.any() for a in A)
    if name in ("n1", "const", "two_valued", "tie_top"):
        assert all(a["ref"].outcome == "nan" and np.isnan(a["mb"].model.y).all() for a in A)
    if name == "zero_division":                 # float64 divides by zero; the kernel's fp32 rounds keep a support
        assert all(a["ref"].outcome == "zero-division" and a["mb"].model.exit == "converged" for a in A)
    if name == "feasible":
        assert all(a["ref"].rounds == 1 for a in A)
    if name == "ties":                          # a tied group is zeroed whole, in the same round
        for a in A:
            for z in a["ref"].zeroed:
                lv = np.unique(a["x"][z])
                assert all(np.isin(np.flatnonzero(a["x"] == q), z).all() for q in lv)
        assert any(len(z) for a in A for z in a["ref"].zeroed)
    if name in ("negative", "all_negative"):
        assert all((a["x"] < 0).any() for a in A)
        if name == "all_negative":
            assert all((a["x"] < 0).all() for a in A)
    if name == "sp_low":                        # alphap near -1: the projection barely moves the shifted slice
        assert all(abs(float(a["mb"].model.alphas[0]) + 1) < 0.5 for a in A)
    if name == "sp_high":
        assert all(np.count_nonzero(a["ref"].y) <= 0.02 * c.n for a in A)
    if c.k == "norm" and c.k_override is None and len(c.sp) > 1:                  # per-slice k1, k2 (tied levels: one k2)
        assert len({float(a["k1"]) for a in A}) > 1 and (c.data == "ties" or len({float(a["k2"]) for a in A}) > 1)


def test_slice_lengths_and_layouts_are_covered():
    ns = {c.n for c in hc.CASES}
    assert set(hc.N_COVER) <= ns
    assert {n % hc.THREADS for n in hc.N_COVER} >= {0, 1, 2, 3, 31, 32, 1023}
    dims = {(len(c.shape), c.dim) for c in hc.CASES}
    assert {(2, 0), (2, 1), (3, 0), (3, 1), (4, 2), (4, 3), (5, 1), (5, 2), (5, 3)} <= dims
    assert any(c.layout[2] == 1 and c.layout[1] >= 64 and c.n == 65536 for c in hc.CASES)     # H of configs[1]
    assert any(c.layout[0] > 1 and c.layout[2] > 1 for c in hc.CASES)
    assert hc.max_rounds(100001) == 100002 and hc.max_rounds(99999) == 100001


def test_round_counts():
    """The many-round case takes the most rounds of the catalogue (16, the most a search over decay shapes found), and on
    stable slices the model takes proj64's round count."""
    best = max(a["ref"].rounds for c in hc.CASES for a in hc.analyse(c.name))
    assert best == 16 and min(a["ref"].rounds for a in hc.analyse("many_rounds")) == best
    for c in hc.CASES:
        for a in hc.analyse(c.name):
            if a["cls"] == "stable":
                assert a["mb"].model.rounds == a["ref"].rounds, (c.name, a["mb"].model.rounds, a["ref"].rounds)


def test_huge_case_crosses_int32():
    c = hc.HUGE
    outer, D, inner = c.layout
    n = outer * inner
    assert D * n > 2 ** 31 and (D - 1) * n > 2 ** 31 - n            # j n + e past int32 in zeroed_ws
    assert ((outer - 1) * D + D - 1) * inner >= 2 ** 31               # (o D + j) inner in at()
    assert D % hc.HUGE_PATTERNS == 0
    assert {a["cls"] for a in hc.analyse("huge")} == {"stable"}


@pytest.mark.parametrize("name", NAMES)
def test_model_and_oracle_within_the_conditioning_bar(name):
    """On stable slices the kernel model and the fp32 oracle are each within the float64 bar (not within each other's
    distance: they round differently)."""
    for j, a in enumerate(hc.analyse(name)):
        if a["cls"] != "stable":
            continue
        y64 = a["ref"].y
        em = float(np.abs(a["mb"].model.y - y64).max()) / a["bar64"]
        orc = hoy.proj_func(torch.from_numpy(a["x"].copy()), float(a["k1"]), float(a["k2"])).double().numpy()
        eo = float(np.abs(orc - y64).max()) / a["bar64"]
        assert em <= 1.0 and eo <= 1.0, (name, j, em, eo)


MODEL_BAR_CAP = 2.0 ** -12


@pytest.mark.parametrize("name", NAMES)
def test_bars_are_tight(name):
    """Per case: on every non-degenerate slice each model form's bar stays below 2^-12 of max|y| (ill-conditioned slices
    included: a form is one fixed arithmetic, only the shift's last bit moves it), and on every stable slice it is below
    the float64 bar, so the model check is the stricter one.  The float64 bar (8x the perturbation spread) is within 128x
    of the model's distance from float64 on at least one stable slice of the case."""
    A = hc.analyse(name)
    for j, a in enumerate(A):
        if a["cls"] == "degenerate":
            continue
        assert a["mb"].rel() <= MODEL_BAR_CAP, (name, j, a["mb"].rel())
        if a["cls"] == "stable":
            assert max(float(f.bar.max()) for f in a["mb"].forms.values()) <= a["bar64"], (name, j)
    e64 = [float(np.abs(a["mb"].model.y - a["ref"].y).max()) / a["bar64"] for a in A if a["cls"] == "stable"]
    if e64:
        assert max(e64) >= 1 / 128, (name, max(e64))


def test_references_match_the_fixtures():
    z = np.load(os.path.join(GOLDEN, "reference_hoyer.npz"), allow_pickle=False)
    names = sorted({k.split("/")[0] for k in z.files if k.startswith("proj_")})
    assert names
    for nm in names:
        X, Y, dim = z[nm + "/X"], z[nm + "/Y"].astype(np.float64), int(z[nm + "/dim"])
        k1, k2 = z[nm + "/k1"], z[nm + "/k2"]
        xs, ys = hc.slices(X, dim), hc.slices(Y, dim)
        for j in range(xs.shape[0]):
            want = ys[j]
            atol = 5e-6 * float(np.abs(want).max())
            for got in (hc.proj64(xs[j], k1[j], k2[j]).y, hc.kernel_model(xs[j], k1[j], k2[j]).y.astype(np.float64),
                        hoy.proj_func(torch.from_numpy(xs[j].copy()), float(k1[j]), float(k2[j])).double().numpy()):
                assert float((np.abs(got - want) / (1e-4 * np.abs(want) + atol)).max()) <= 1.0, (nm, j)


def test_degenerate_outcomes_are_recorded():
    """What the reference does on each degenerate slice: NaN (a = 0) or ZeroDivisionError (every coordinate zeroed)."""
    seen = set()
    for c in hc.CASES:
        for a in hc.analyse(c.name):
            if a["cls"] != "degenerate":
                continue
            x = torch.from_numpy(a["x"].copy())
            try:                                # the fp32 oracle lands on one of the two, not always float64's
                oracle = "nan" if torch.isnan(hoy.proj_func(x, float(a["k1"]), float(a["k2"]))).all() else "finite"
            except ZeroDivisionError:
                oracle = "zero-division"
            assert a["ref"].outcome in ("nan", "zero-division") and oracle in ("nan", "zero-division", "finite"), (c.name, oracle)
            seen.add(a["ref"].outcome)
    assert seen == {"nan", "zero-division"}
