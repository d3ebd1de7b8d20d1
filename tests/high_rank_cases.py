"""Cases of the rank-blocked fp32 kernels (ranks above 256) for tests/test_gpu_high_rank.py, and what they must cover
(checked against the library's own planner on the CPU by tests/test_high_rank_plan.py).

Above rank 256 the fused contraction runs one CTA per output block of 256 components (grid z), each summing S over every
rank chunk of 256 with its own chunk last; the loss kernel sums S over the same chunks; the KL column sums run one block of
256 components per grid y.  The exactness argument of tests/f32_cases.py holds unchanged: integer data whose every partial
sum is an integer below 2^24 makes every order exact.
"""
import math

import f32_cases as fc

BLOCK = 256

# (N, C, R): rows and contracted columns at residues {1, 63, 0} mod 64, one to four rank blocks, short and full last blocks
HIGH_EDGE = [
    (1, 1, 257),           # two blocks, the last holding one component
    (63, 129, 300),        # R % 16 != 0
    (128, 191, 512),       # two full blocks
    (129, 64, 513),        # three blocks, one component in the last
    (65, 127, 1000),       # four blocks, the last 232 components
    (191, 63, 256),        # one block: the single-chunk kernel
]
HIGH_CHUNKED = [
    (64, 4000, 512),       # H update: 32 chunks (the cap) of 2 tiles over 63 tiles
    (4000, 64, 300),       # the same for the W update
    (1000, 2000, 1000),    # both updates several chunks (9 and 5) over four rank blocks
]
HIGH_EXACT = HIGH_EDGE + HIGH_CHUNKED
HIGH_LOSS = HIGH_EXACT
# float64-bar cases (beta 0, 0.5, 1.5, 3 and their losses)
HIGH_BAR = [(65, 129, 300), (129, 1000, 513), (64, 2112, 512)]
# the ratio stage on exact raw terms
HIGH_RATIO = [(129, 64, 513), (1000, 2000, 1000)]


def cdiv(a, b):
    return -(-a // b)


def rank_blocks(R):
    return cdiv(R, BLOCK)


def parent_plan(N, C, R):
    """nmfb200_nmf_plan of a rank <= 256 context, restated: nothing of it depends on the rank blocks."""
    def chunks(rows, cols):
        return max(1, min(cdiv(528, cdiv(rows, 64)), cdiv(cols, 64), 32))

    def loss_chunks(rows, cols):
        return max(1, min(cdiv(528, cdiv(rows, 64)), cdiv(cols, 64)))

    nch_w, nch_h = chunks(C, N), chunks(N, C)
    lc = loss_chunks(N, C)
    rb = 1 if R <= 16 else 2 if R <= 32 else 4 if R <= 64 else 8 if R <= 128 else 16
    return {"nch_w": nch_w, "nch_h": nch_h, "tpc_w": cdiv(cdiv(N, 64), nch_w), "tpc_h": cdiv(cdiv(C, 64), nch_h),
            "rb": rb, "loss_chunks": lc, "loss_tpc": cdiv(cdiv(C, 64), lc),
            "colsum_blocks_n": max(1, min(1024, cdiv(N, 64))), "colsum_blocks_c": max(1, min(1024, cdiv(C, 64)))}


def exact_ok(case):
    N, C, R = case
    fc.nmf_range(N, C, R)
    fc.nmf_range(N, C, R, loss=True)
    return fc.nmf_kl_bound(N, C, R) < fc.EXACT


def flops(N, C, R, beta):
    """Algorithmic FLOPs of one iteration (both updates) of the fused contraction: S = F G^T (2 N C R) and the numerator
    (2 N C R) per update, plus the denominator (2 N C R) for beta != 1."""
    per = (4 if beta == 1 else 6) * N * C * R
    return 2 * per


def recompute_factor(R, beta):
    """Executed over minimal FLOPs of the rank-blocked contraction: S is recomputed for each of the nb output blocks."""
    nb = rank_blocks(R)
    return (nb + 1) / 2 if beta == 1 else (nb + 2) / 3


assert all(exact_ok(c) for c in HIGH_EXACT)
assert math.isfinite(recompute_factor(512, 1))
