"""Cases on which every CTA of the tensor-core NMF contraction (csrc/tc_nmf.cu: tc_contract_kernel) walks several work items.

TEST INFRASTRUCTURE ONLY (no library calls).  The contraction is persistent: grid = min(items, SMs) CTAs, CTA b walks items
b, b + grid, b + 2 grid, ... (item = chunk x row_blocks + row block), and what carries over from one item to the next -- the
F slot (it % NF) and its barrier parity ((it / NF) & 1), the stage counter of the NS-stage ring, the ping-pong token of the
two consumer warpgroups, the loss accumulators -- only matters from a CTA's second item on.  Every case here is derived
from an SM count S, so it reaches the same walk state on any card:

  tall     N = 128 (4 S + 4) + 65 rows, C = 600: the H update (F = H) has 4 S + 5 items on S CTAs, so some CTAs walk 5
           items (it = 0..4: each slot of NF = 2 back at phase 0) and the others 4; the last row block holds 65 rows.
           C = 600 is 5 tiles of 128 columns (10 of 64 at TN = 64), neither a multiple of NS = 4 nor of NS = 3, the last
           tile short: item boundaries fall inside the stage ring and inside a ring phase.
  wide     the same sizes, axes swapped: the W update (F = W) and the loss folded into it walk.
  chunked  ~141 row blocks over C = 4161 (33 tiles): the H update splits the columns into chunks with a short last one, so
           a CTA walks up to 8 items of alternating lengths.  Fast mode only, like tests/test_gpu_tc_terms.py's CHUNK_CASES:
           the split mode's model bar is not tight over 4000-term sums.

Periodic data: the walked factor's rows, and the matching rows (tall) or columns (wide) of V, repeat a random block of
128 P rows, P the smallest prime >= 5 that does not divide the grid.  Consecutive items of a CTA then read F blocks from
different residues mod P (so a stale or wrong F slot moves the model and float64 bars), and every output row must equal its
representative in the first period bit for bit, whichever CTA, walk position, F slot, barrier phase and stage offset
produced it (each row is summed in one fixed order that depends on its row within the 128-row block only).
"""
import torch

import tc_model as tcm

# (precision, rank) of the four kernel configurations <RP, SPLIT, TN>, and their shared-memory layouts (TN, NS, NF) as
# SmemLayout<KW, TN> works them out from the 227 KB budget
CONFIGS = [("f16", 64), ("f16_split", 40), ("f16", 128), ("f16_split", 100)]
LAYOUTS = {("f16", 64): (128, 4, 2), ("f16_split", 64): (128, 3, 1), ("f16", 128): (128, 3, 1),
           ("f16_split", 128): (64, 3, 1)}
SM_COUNTS = (132, 114)                 # H100 SXM, H100 PCIe
TALL_C = 600
CHUNK_C = 4161
CHUNK_RANKS = (64, 128)


def layout(prec, R):
    """(TN, NS, NF) of the configuration serving (prec, R)."""
    return LAYOUTS[(prec, 64 if R <= 64 else 128)]


def period_prime(grid):
    """The smallest prime >= 5 that does not divide `grid`."""
    p = 5
    while any(p % d == 0 for d in range(2, p)) or grid % p == 0:
        p += 1
    return p


def tall_rows(S):
    return 128 * (4 * S + 4) + 65


def side(p, which):
    """The W (0) or H (1) half of a plan dict of _capi.nmf_tc_plan (or of `mirror_plan`)."""
    k = "w" if which == 0 else "h"
    return {f: p[f"{f}_{k}"] for f in ("row_blocks", "tiles", "nchunks", "tpc", "items", "grid")}


def mirror_plan(N, C, R, prec, S):
    """What nmfb200_nmf_tc_plan reports, from tc_model's mirror of make_plan and the layouts above."""
    TN, NS, NF = layout(prec, R)
    out = {"tn": TN, "ns": NS, "nf": NF}
    for k, (rows, cols) in (("w", (C, N)), ("h", (N, C))):
        rb, tiles, nch, tpc = tcm.plan(rows, cols, S, TN)
        items = rb * nch
        out.update({f"row_blocks_{k}": rb, f"tiles_{k}": tiles, f"nchunks_{k}": nch, f"tpc_{k}": tpc,
                    f"items_{k}": items, f"grid_{k}": min(items, S)})
    return out


def walk(pl, NS, NF):
    """Per CTA of one orientation's launch (pl: `side`), the items it walks in order, each as a dict: item, row block,
    chunk, tiles, F slot, F barrier parity, stage slot of its first tile (t % NS) and that stage's ring phase."""
    rb, tiles, tpc, items, grid = pl["row_blocks"], pl["tiles"], pl["tpc"], pl["items"], pl["grid"]
    ctas = []
    for b in range(grid):
        t, seq = 0, []
        for it, item in enumerate(range(b, items, grid)):
            chunk = item // rb
            n = min(tiles, (chunk + 1) * tpc) - chunk * tpc
            seq.append({"item": item, "row_block": item % rb, "chunk": chunk, "tiles": n, "slot": it % NF,
                        "parity": (it // NF) & 1, "stage": t % NS, "ring_phase": (t // NS) & 1})
            t += n
        ctas.append(seq)
    return ctas


def walk_state(pl, NS, NF, P, TN, cols):
    """What the walk of one orientation reaches (pl: `side`; cols: the contracted length), as a dict of facts the tests
    assert: most / fewest items of a CTA, whether an F slot gets back to phase 0 after its flip, whether an item starts
    inside the stage ring, whether a CTA alternates chunk lengths, and whether consecutive items of every CTA read F blocks
    of different residues mod P."""
    ctas = walk(pl, NS, NF)
    counts = [len(c) for c in ctas]
    last_tiles = pl["tiles"] - (pl["nchunks"] - 1) * pl["tpc"]
    return {
        "max_items": max(counts), "min_items": min(counts),
        # slot f at parity 0, then 1, then 0 again: item it = 2 NF + f for some f < NF
        "slot_back_to_phase0": max(counts) >= 2 * NF + 1,
        "uneven": pl["items"] % pl["grid"] != 0,
        "item_inside_ring": any(s["stage"] != 0 for c in ctas for s in c[1:]),
        "item_inside_ring_phase": any(s["stage"] != 0 and s["ring_phase"] == 1 for c in ctas for s in c[1:]),
        "tiles_per_item_mod_ns": pl["tpc"] % NS,
        "short_last_tile": cols % TN != 0,
        "short_last_chunk": pl["nchunks"] > 1 and last_tiles < pl["tpc"],
        "alternating_chunk_lengths": any(len({s["tiles"] for s in c}) > 1 for c in ctas),
        "distinct_consecutive_f": all((a["row_block"] - b["row_block"]) % P != 0
                                      for c in ctas for a, b in zip(c, c[1:])),
    }


def _chunk_rows(S, R):
    """Rows of the chunked case: the first row-block count from 141 up whose H-update plan at S SMs has more than one
    chunk, a short last chunk, an item count that is not a multiple of the grid, at least 2 NF + 1 items on the busiest
    CTA and consecutive items on distinct F residues; the last row block holds 65 rows."""
    TN, NS, NF = layout("f16", R)
    for rb in range(141, 400):
        N = 128 * (rb - 1) + 65
        pl = side(mirror_plan(N, CHUNK_C, R, "f16", S), 1)
        w = walk_state(pl, NS, NF, period_prime(pl["grid"]), TN, CHUNK_C)
        if (w["short_last_chunk"] and w["uneven"] and w["slot_back_to_phase0"] and w["distinct_consecutive_f"]
                and w["alternating_chunk_lengths"] and pl["tpc"] % NS != 0):
            return N
    raise AssertionError(f"no chunked case at {S} SMs, rank {R}")


def cases(S):
    """Every case at S SMs: dicts with name, kind, prec, N, C, R, which (the walked update: 0 = W, 1 = H), P."""
    out = []
    n = tall_rows(S)
    for prec, R in CONFIGS:
        out.append({"kind": "tall", "prec": prec, "N": n, "C": TALL_C, "R": R, "which": 1})
        out.append({"kind": "wide", "prec": prec, "N": TALL_C, "C": n, "R": R, "which": 0})
    for R in CHUNK_RANKS:
        out.append({"kind": "chunked", "prec": "f16", "N": _chunk_rows(S, R), "C": CHUNK_C, "R": R, "which": 1})
    for c in out:
        c["P"] = period_prime(S)
        c["name"] = f"{c['kind']}-{c['prec']}-{c['N']}x{c['C']}-r{c['R']}"
    return out


def case(S, kind, prec, R):
    return next(c for c in cases(S) if (c["kind"], c["prec"], c["R"]) == (kind, prec, R))


def periodic_data(c, seed, two_output=False):
    """(V, W, H) fp32 on the CPU for case c: the walked factor's rows and the matching rows / columns of V repeat a random
    block of 128 P rows.  Targets rand + 0.05 and factors rand + 0.1; for the two-output kernels factors in [0.5, 1.5)
    and targets rand + 0.01 (tests/test_gpu_tc_terms.py: test_nmf_two_output_terms_and_loss)."""
    N, C, R, which, per = c["N"], c["C"], c["R"], c["which"], 128 * c["P"]
    vmin, fmin = (0.01, 0.5) if two_output else (0.05, 0.1)
    g = torch.Generator().manual_seed(seed)
    rows, cols = (C, N) if which == 0 else (N, C)        # rows of F, rows of G
    reps = -(-rows // per)
    F = (torch.rand(per, R, generator=g) + fmin).repeat(reps, 1)[:rows].contiguous()
    G = torch.rand(cols, R, generator=g) + fmin
    Vm = (torch.rand(per, cols, generator=g) + vmin).repeat(reps, 1)[:rows]
    V = (Vm.t() if which == 0 else Vm).contiguous()
    W, H = (F, G) if which == 0 else (G, F)
    return V, W, H


def period_breaks(X, period, pl, limit=4):
    """Rows of X (rows of F first) that are not bitwise equal to their representative row % period, at most `limit`, each
    with the items that produced it (one per chunk), their CTAs (item % grid) and walk positions (item // grid)."""
    X = X.detach().reshape(X.shape[0], -1).contiguous()
    bits = X.view(torch.int32) if X.dtype == torch.float32 else X.view(torch.int64)
    idx = torch.arange(X.shape[0], device=X.device) % period
    bad = (bits != bits[idx]).any(1).nonzero().flatten()[:limit].tolist()
    out = []
    for r in bad:
        items = [ch * pl["row_blocks"] + r // 128 for ch in range(pl["nchunks"])]
        out.append({"row": r, "representative": r % period, "items": items,
                    "ctas": [i % pl["grid"] for i in items], "walk_positions": [i // pl["grid"] for i in items],
                    "got": X[r][(bits[r] != bits[r % period])][:1].tolist(),
                    "want": X[r % period][(bits[r] != bits[r % period])][:1].tolist()})
    return out


def assert_periodic(tag, X, period, pl):
    bad = period_breaks(X, period, pl)
    assert not bad, f"{tag}: rows differ from their representative in the first period: {bad}"
