"""How much of the dense-operand gather could a row-window SpMM share?  (round-2 VERDICT item 2)

The row-warp SpMM gathers 4*P bytes of the dense operand per non-zero (DESIGN.md section 4).  A row-window
kernel -- W rows processed in lock-step so that a gathered operand row is reused by every window row holding that
column -- cuts the gather by  reuse(W) = nnz(window) / |union of the window's columns|.  This script measures
reuse(W) on the benchmark generator's own matrix (BASELINE configs[1] column count and density), with windows of
(a) cells of the SAME planted topic, i.e. a perfect clustering, and (b) consecutive cells in generation order,
and the same for windows of peaks (rows of A^T).  CPU only:

    python profiles/spmm_reuse_analysis.py [cells=6000] > profiles/spmm_reuse_analysis_r2.json
"""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from muon_b200._synth import generate_host, make_tables  # noqa: E402

n = int(sys.argv[1]) if len(sys.argv) > 1 else 6000
D, dens, T, seed = 200_000, 0.03, 64, 1
tb = make_tables(D, dens, T, seed)
X = generate_host(n, D, dens, tables=tb)
rt, _ = tb.rows(0, n)


def reuse(M, order, W, same_key=None):
    tot = uni = 0
    for s in range(0, M.shape[0] - W + 1, W):
        rows = order[s:s + W]
        if same_key is not None and same_key[rows[0]] != same_key[rows[-1]]:
            continue
        cols = np.concatenate([M.indices[M.indptr[r]:M.indptr[r + 1]] for r in rows])
        tot += cols.size
        uni += np.unique(cols).size
    return tot / max(uni, 1)


by_topic = np.argsort(rt, kind="stable")
out = {"cells": n, "peaks": D, "density": dens, "nnz_per_cell": X.nnz / n, "cells_rows": {}, "peaks_rows": {}}
for W in (2, 4, 8, 16, 32, 64, 128):
    out["cells_rows"][W] = {"same_topic": round(reuse(X, by_topic, W, rt), 3),
                            "generation_order": round(reuse(X, np.arange(n), W), 3)}
# rows of A^T: peaks; "clustering" = peaks ordered by the topic in which they are strongest
Xt = X.T.tocsr()
peak_topic = np.argmax(tb.topic, axis=0)
live = np.nonzero(np.diff(Xt.indptr) > 0)[0]
order_p = live[np.argsort(peak_topic[live], kind="stable")]
for W in (8, 32, 128):
    out["peaks_rows"][W] = {"by_strongest_topic": round(reuse(Xt[order_p], np.arange(order_p.size), W), 3),
                            "index_order": round(reuse(Xt[live], np.arange(live.size), W), 3)}
out["reading"] = ("83 % of the non-zeros come from the per-peak baseline, which has no cluster structure, and per-peak "
                  "probabilities are a few percent, as in real scATAC: two cells of the same topic share ~4 % of their peaks. "
                  "A window of 8 perfectly clustered cells shares 1.26x (21 % fewer gathered bytes) while every gathered "
                  "operand row would have to be applied to 8 accumulator rows under predication (8x the FMA issue for 1.26x "
                  "fewer loads); generation order gives 1.21x, so clustering buys almost nothing.  Reuse only becomes large "
                  "(>2x) at W >= 32-64, where the window is simply dense in its columns -- the regime where the operand is "
                  "staged in shared memory, which is bound by the same 128 B/clk L1/shared data pipe.  Hence the "
                  "round-2 lever taken instead: fewer BYTES per gathered element (IEEE-half operand in the early block-"
                  "Lanczos steps, spmm.cu::spmm_row with T = __half).")
print(json.dumps(out, indent=1))
