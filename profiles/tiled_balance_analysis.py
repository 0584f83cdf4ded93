"""How evenly do the tiled SpMM kernel's warps share a band's work?  (spmm.cu, spmm_csr_tiled_kernel)

A CTA owns a band of 128 rows: NW warps of W rows each.  Every warp must release a staged operand tile before it is
refilled, so each tile runs at the pace of the warp with the most entries in it.  With entries spread evenly over the
columns, a warp's share of every tile follows its rows' total length, and the band runs at

    balance = mean over the band's warps of the warp's total length / the largest warp's total length

of the rate it would with perfectly even warps.  This script measures that on the benchmark generator
(``make_tables(200000, 0.03, 64, 1)``) for two ways of giving rows to warps: consecutive rows (warp w takes rows
w*W .. w*W + W - 1 of the band), and the band's rows sorted by length and dealt snake-wise (the kernel's order).

- Rows of A (cells): the real row lengths of the first ``cells`` rows the generator makes.
- Rows of Aᵀ (peaks): each peak's expected entry count over 500k cells, from the generator's own probabilities.

CPU only:

    python profiles/tiled_balance_analysis.py [cells=12800]
"""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from muon_b200._synth import generate_host, make_tables  # noqa: E402

R = 128
D, dens, T, seed, N = 200_000, 0.03, 64, 1, 500_000


def warp_rows(lengths, NW, W, snake):
    """[NW, W] band-local row ids per warp: consecutive, or ranked longest first (ties: lower row) and dealt
    snake-wise, rank p to warp p mod NW in even rounds and NW - 1 - p mod NW in odd ones"""
    if not snake:
        return np.arange(R).reshape(NW, W)
    order = np.lexsort((np.arange(R), -lengths))
    rows = np.empty((NW, W), dtype=np.int64)
    for p, r in enumerate(order):
        w, k = p % NW, p // NW
        rows[NW - 1 - w if k & 1 else w, k] = r
    return rows


def balance(lengths, NW, W, snake):
    """mean over the full bands of (mean warp total / largest warp total)"""
    out = []
    for b0 in range(0, lengths.size - R + 1, R):
        band = lengths[b0:b0 + R]
        tot = band[warp_rows(band, NW, W, snake)].sum(1)
        if tot.max() > 0:
            out.append(tot.mean() / tot.max())
    return float(np.mean(out))


cells = int(sys.argv[1]) if len(sys.argv) > 1 else 12800
tb = make_tables(D, dens, T, seed)
X = generate_host(cells, D, dens, tables=tb)
cell_len = np.diff(X.indptr).astype(np.float64)
# expected entries of peak j: the sum over cells of p(cell, j) = scale(cell) * (beta_j / 2 + topic[t(cell), j]) (the
# generator's 0.9 clip is never reached at this density)
t, s = tb.rows(0, N)
S = np.bincount(t, weights=s.astype(np.float64), minlength=T)
peak_len = S.sum() * 0.5 * tb.beta.astype(np.float64) + S @ tb.topic.astype(np.float64)

out = {"cells": cells, "peaks": D, "density": dens}
for name, L in (("cells (rows of A)", cell_len), ("peaks (rows of At)", peak_len)):
    out[name] = {"length_cv": round(float(L.std() / L.mean()), 2), "max_over_mean": round(float(L.max() / L.mean()), 1)}
    for NW, W in ((16, 8), (32, 4)):
        for snake in (False, True):
            key = f"{NW}x{W} " + ("sorted, snake" if snake else "consecutive")
            out[name][key] = round(balance(L, NW, W, snake), 2)
print(json.dumps(out, indent=1))
