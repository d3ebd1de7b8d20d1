"""Test-only batched engine: the interface of engine.CudaBatchedNmfEngine / CudaBatchedNmfdEngine over one single oracle
engine (tests/oracle_engine.py, tests/test_cd.py) per problem, so the batched fits' host logic runs without a GPU.  It is
never imported by the product."""
import torch


class BatchedOracleEngine:
    """P problems, problem p on `single(V[p], W[p], H[p])`, a stopped problem (`set_active`) left untouched.  A target
    without the problem axis is shared by every problem.  `lengths` (one int per problem): a ragged batch, each problem's
    engine built on its real cells only -- rows [:L] of V[p] and H[p] for an NMF engine, positions [:L] of V[p]'s last axis
    and [:L - T + 1] of H[p]'s for a convolutive one (T: W's last size); H's padding is never touched.

    Counts the W and H updates each problem receives (`updates_w`, `updates_h`) and logs every update call (`calls`).
    `iterate` exists for NMF engines only, as on the CUDA engines; `cd_update` / `cd_iterate` where `single` has them."""
    device = torch.device("cpu")
    precision = "oracle"

    def __init__(self, V, W, H, single, lengths=None):
        P = W.shape[0]
        if V.dim() == W.dim() - 1:
            V = V.expand(P, *V.shape)
        nmf = single.kind == "nmf"
        self.kind = single.kind + "_batched"
        self.V, self.W, self.H = V, W, H
        if lengths is None:
            self.cuts = [(Ellipsis,)] * P
            vcuts = self.cuts
        elif nmf:
            self.cuts = vcuts = [(slice(None, L),) for L in lengths]
        else:
            vcuts = [(Ellipsis, slice(None, L)) for L in lengths]
            self.cuts = [(Ellipsis, slice(None, L - W.shape[-1] + 1)) for L in lengths]
        # H's real cells as a contiguous tensor (a view where they are one already), written back after each H update
        self.engines = [single(self.V[p][vc].contiguous(), W[p], H[p][hc].contiguous())
                        for p, (vc, hc) in enumerate(zip(vcuts, self.cuts))]
        self.active = [True] * P
        self.updates_w = [0] * P
        self.updates_h = [0] * P
        self.calls = []
        self._last = torch.full((P,), float("nan"), dtype=torch.float64)
        if nmf:
            self.iterate = self._iterate
        if hasattr(single, "cd_update"):
            self.cd_update, self.cd_iterate = self._cd_update, self._cd_iterate

    def close(self):
        pass

    def minmax(self):
        real = torch.cat([e.V.reshape(-1) for e in self.engines])
        return float(real.min()), float(real.max())

    def set_active(self, active):
        self.active = [bool(a) for a in active]

    def _each(self, fn, which):
        for p, e in enumerate(self.engines):
            if self.active[p]:
                fn(e)
                if which == 0:
                    self.updates_w[p] += 1
                else:
                    self.H[p][self.cuts[p]] = e.H
                    self.updates_h[p] += 1

    def update_w(self, *a):
        self.calls.append(("update_w",) + a)
        self._each(lambda e: e.update_w(*a), 0)

    def update_h(self, *a):
        self.calls.append(("update_h",) + a)
        self._each(lambda e: e.update_h(*a), 1)

    def _iterate(self, k, *a):
        self.calls.append(("iterate", k) + a)
        for _ in range(k):
            self._each(lambda e: e.update_w(*a), 0)
            self._each(lambda e: e.update_h(*a), 1)

    def _cd_update(self, which, l1, l2):
        self.calls.append(("cd_update", which, l1, l2))
        self._each(lambda e: e.cd_update(which, l1, l2), which)

    def _cd_iterate(self, k, l1, l2):
        self.calls.append(("cd_iterate", k, l1, l2))
        for _ in range(k):
            self._each(lambda e: e.cd_update(0, l1, l2), 0)
            self._each(lambda e: e.cd_update(1, l1, l2), 1)

    def losses(self, beta):
        for p, e in enumerate(self.engines):
            if self.active[p]:
                self._last[p] = e.loss(beta)
        return self._last.clone()

    @classmethod
    def factory(cls, single, log):
        """A three-argument `_engine_factory` that appends every engine it makes to `log`."""
        def make(V, W, H):
            eng = cls(V, W, H, single)
            log.append(eng)
            return eng
        return make
