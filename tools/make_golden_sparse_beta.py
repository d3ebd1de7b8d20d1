"""Generate tests/golden/reference_sparse_beta.npz: NMF fits of sparse COO targets at beta 0.5, 1.5 and 3 through the REAL
reference's sparse path (torchnmf 0.3.5 `_nmf_sp_recon_beta_pos_neg`, nmf.py:603-638, importable from oracle/_ref:
oracle/build_ref.py), on the CPU.

    python tools/make_golden_sparse_beta.py

Targets follow oracle/make_golden.py:sparse_cases: rand(N, C) from seed 0 with the entries above 0.93 kept (about 7 %
stored), one row and one column emptied; W0 / H0 = |randn| from seed 1.  The cases: every beta with and without the
penalties, a stop-rule fit per beta that ends before max_iter, one at rank 200 (8 rank floats per lane of the gather
kernels) and one at a rank that is not a multiple of 32.  Stored in oracle/make_golden.py's layout (dense V).
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.make_golden import ref_nmf, run_reference, save_cases  # noqa: E402  (imports the reference)


def target(N, C):
    torch.manual_seed(0)
    D = torch.rand(N, C)
    D = torch.where(D > 0.93, D, torch.zeros(()))
    D[N // 17] = 0                              # an empty row and an empty column
    D[:, 5] = 0
    return D


def factors(N, C, R):
    torch.manual_seed(1)
    return torch.randn(C, R).abs(), torch.randn(N, R).abs()


#     name suffix      (N, C)      R    betas             iters  tol   alpha l1_ratio
SPECS = [
    ("a0_l0",       (300, 200), 8,   (0.5, 1.5, 3), 12,  None, 0.0, 0.0),
    ("a0.1_l0.5",   (300, 200), 8,   (0.5, 1.5, 3), 12,  None, 0.1, 0.5),
    ("stoprule",    (300, 200), 8,   (0.5, 1.5, 3), 200, 3e-2, 0.0, 0.0),
    ("r200",        (40, 36),   200, (1.5,),        10,  None, 0.0, 0.0),
    ("r40",         (120, 100), 40,  (3,),          15,  None, 0.1, 0.5),
]


def main():
    torch.set_num_threads(1)          # deterministic reduction order
    cases = {}
    for tag, (N, C), R, betas, iters, tol, alpha, l1r in SPECS:
        D = target(N, C)
        W0, H0 = factors(N, C, R)
        for beta in betas:
            tol_v = float("-inf") if tol is None else tol
            W, H, n_iter, losses = run_reference(ref_nmf.NMF, D.to_sparse(), W0, H0, beta, tol_v, iters, alpha, l1r)
            if tol is not None:
                assert n_iter < iters, f"the stop rule must end the fit early (beta {beta}: {n_iter})"
            name = f"spbeta_b{beta}_{tag}"
            cases[name] = dict(kind="nmf", V=D, W0=W0, H0=H0, W=W, H=H, n_iter=n_iter, losses=losses, beta=beta,
                               tol=tol_v, max_iter=iters, alpha=alpha, l1_ratio=l1r)
            print(name, "n_iter", n_iter)
    save_cases(cases, "reference_sparse_beta.npz")


if __name__ == "__main__":
    main()
