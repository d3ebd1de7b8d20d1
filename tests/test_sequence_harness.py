"""CPU checks of the call-sequence harness (tests/sequence_cases.py): the sequences reach every state transition they are
there for, and the harness's float64 checks pass an exact engine and fail one that lags a call behind."""
import pytest
import torch

import sequence_cases as sc
from oracle_engine import OracleNmfEngine


def test_sequences_reach_every_transition():
    reached = sc.transitions_reached(sc.sequences())
    missing = [t for t, names in reached.items() if not names]
    assert not missing, f"no sequence reaches: {missing}"


def test_every_listed_tensor_core_step_has_a_path():
    """The simulated paths are what the sequences are built around: the mixed-beta and target sequences stay on the tensor
    cores where they must, the R > 64 sequence runs its two-output betas on the fp32 kernels."""
    paths = {s.name: [(p.step, p.reported) for p in sc.simulate(s)] for s in sc.sequences()}
    assert all(path == "tc" for st, path in paths["mixed-f16"] if st[0] != "rescale")
    r100 = [(st, path) for st, path in paths["paths-r100"] if st[0] in ("update_w", "update_h", "raw")]
    assert all((path == "f32") == sc.two_output(st[-1] if st[0] == "raw" else st[1]) for st, path in r100)


class LaggingEngine(OracleNmfEngine):
    """Contracts with the factors of one call earlier (what a stale operand copy amounts to)."""

    def __init__(self, V, W, H):
        super().__init__(V, W, H)
        self._prev = (W.clone(), H.clone())

    def _stale(self, fn, *args):
        now = (self.W.clone(), self.H.clone())
        self.W.copy_(self._prev[0])
        self.H.copy_(self._prev[1])
        out = fn(*args)
        moved = (self.W.clone(), self.H.clone())
        self.W.copy_(now[0])
        self.H.copy_(now[1])
        if not torch.equal(moved[0], self._prev[0]):
            self.W.copy_(moved[0])
        if not torch.equal(moved[1], self._prev[1]):
            self.H.copy_(moved[1])
        self._prev = now
        return out

    def update_w(self, *a):
        return self._stale(super().update_w, *a)

    def update_h(self, *a):
        return self._stale(super().update_h, *a)

    def raw_terms(self, *a):
        return self._stale(super().raw_terms, *a)

    def loss(self, *a):
        return self._stale(super().loss, *a)


CPU_SEQS = ["fit-f16", "mixed-f16", "shard"]


def _cpu_run(name, cls):
    seq = sc.by_name(name)
    seq.shape = (96, 80, 12)                # the same steps, small enough for float64 on the CPU
    targets, W, H = sc.fitted_data(seq)
    V = targets["V"].double()
    eng = cls(V, W.double(), H.double())
    return sc.run(seq, eng, sc.float64_check(seq, V))


@pytest.mark.parametrize("name", CPU_SEQS)
def test_harness_passes_the_exact_engine(name):
    _, res = _cpu_run(name, OracleNmfEngine)
    assert len(res) >= 10 and max(e for _, _, e in res) < 1e-6


@pytest.mark.parametrize("name", CPU_SEQS)
def test_harness_fails_an_engine_one_call_behind(name):
    with pytest.raises(AssertionError, match="x the float64 bar"):
        _cpu_run(name, LaggingEngine)
