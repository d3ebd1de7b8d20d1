"""Helpers of the sharded PLCA tests (tests/test_sharded_gloo_plca.py on the CPU, tests/test_gpu_sharded_plca.py on the GPU).

`recorded_losses` captures the divergence a fit's stop rule sees at every check: on a sharded fit that is the all-reduced
sum over the ranks, so comparing it with the unsharded fit's checks the loss all-reduce directly, constant factors
included.  `interior_tol` picks, from an unsharded fit's divergences at tol = -inf, a tol at which that fit stops at an
interior check with a margin on both sides, so that a rank stopping on its own shard's loss would take another decision.
`spawn` is mp.spawn with a deadline: a rank that has not finished by then is killed and the test fails instead of hanging.
"""
import contextlib
import math
import time

import pytest
import torch.multiprocessing as mp


@contextlib.contextmanager
def recorded_losses():
    """Within the block, every PLCA-family fit appends the raw divergence of each of its stop-rule checks to the yielded
    list, in order."""
    import torchnmf_b200.plca as plca
    inner = plca._fit_single
    losses = []

    def fit_single(step, divergence, max_iter, tol, verbose):
        def recorded(follows):
            d = divergence(follows)
            losses.append(d)
            return d
        return inner(step, recorded, max_iter, tol, verbose)

    plca._fit_single = fit_single
    try:
        yield losses
    finally:
        plca._fit_single = inner


def interior_tol(divergences, margin=1.2):
    """A tol at which a fit with these divergences at its checks (tol = -inf, so one per check up to max_iter) stops at an
    interior check after at least one that does not stop: the geometric mean of the smallest relative decrease before that
    check and the decrease at it, at least `margin` apart.  The stop rule is nmf._fit_single's."""
    loss = [math.sqrt(2.0 * d) for d in divergences]
    dec = [(loss[i - 1] - loss[i]) / loss[0] for i in range(1, len(loss))]
    for k in range(1, len(dec) - 1):
        before = min(dec[:k])
        if dec[k] > 0 and before > margin * dec[k]:
            return math.sqrt(before * dec[k])
    raise AssertionError(f"no interior stop with margin {margin} in the relative decreases {dec}")


def spawn(worker, args, world=2, timeout=240):
    """mp.spawn(worker, args, nprocs=world) that kills every rank still running after `timeout` s and fails the test."""
    ctx = mp.spawn(worker, args=args, nprocs=world, join=False)
    deadline = time.monotonic() + timeout
    while not ctx.join(timeout=5):
        if time.monotonic() > deadline:
            for p in ctx.processes:
                if p.is_alive():
                    p.kill()
            for p in ctx.processes:
                p.join()
            pytest.fail(f"a rank did not finish within {timeout} s")
