"""mu.atac.tl.rank_peaks_groups on the benchmark's ATAC matrix, one H100.

    python profiles/bench_rank.py [cells=500000] [peaks=200000] [cpu_peaks=20000]

The configs[1] matrix (3 % density) is generated on the device (``_synth.generate_device``) and TF-IDF-transformed; the
groups are the generator's planted topic ids (64 topics of skewed sizes).  Not timed.  Each of t-test, wilcoxon (rest),
wilcoxon with ``tie_correct`` and wilcoxon against group "0" runs once as warm-up and once timed, with the phases of
``muon_b200._rank`` bracketed by device synchronisation: the transposition, the sort-and-sweep (``rank.stats``), the
scoring with the correction and top-n selection (``rank.score``) and the host assembly.  Also printed: the share of
stored entries on the long-row path, the peak device memory, and the card's name and power limit.

CPU figure: the numpy / scipy restatement (``oracle/rank_ref.py``, not scanpy) on the first 10 000 cells and the first
``cpu_peaks`` peaks, with the GPU timed on that same matrix.  Prints one JSON line.
"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import pandas as pd
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import muon_b200 as mu  # noqa: E402
from muon_b200 import _device, _lib, _rank, _synth  # noqa: E402
from oracle import rank_ref  # noqa: E402

N = int(sys.argv[1]) if len(sys.argv) > 1 else 500_000
D = int(sys.argv[2]) if len(sys.argv) > 2 else 200_000
CPU_PEAKS = int(sys.argv[3]) if len(sys.argv) > 3 else 20_000
CONFIGS = {"t-test": {}, "wilcoxon": {"method": "wilcoxon"},
           "wilcoxon_tie": {"method": "wilcoxon", "tie_correct": True},
           "wilcoxon_vs_0": {"method": "wilcoxon", "reference": "0"}}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def run(ad, kw):
    _lib.PHASES = {}
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    _rank.rank_genes_groups(ad, "topic", **kw)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    ph, _lib.PHASES = _lib.PHASES, None
    return {"wall_s": round(wall, 3), **{k.split(".")[1] + "_s": round(v, 3) for k, v in ph.items()}}


def main():
    torch.cuda.set_device(0)
    tb = _synth.make_tables(D, 0.03, 64, 0)
    A = _synth.generate_device(N, D, 0.03, tables=tb)
    X = _device.tfidf_csr(A, inplace_values=True) or A
    topics = tb.rows(0, N)[0]
    obs = pd.DataFrame({"topic": pd.Categorical([str(t) for t in topics], categories=[str(t) for t in range(64)])})
    obs = obs.loc[:, ["topic"]]
    ad = mu.SimpleAnnData(shape=(N, D), obs=obs)
    ad.X = X
    counts = torch.bincount(X.indices, minlength=D)
    cap = int(_lib.load().mub_rank_shared_capacity(4))
    out = {"cells": N, "peaks": D, "nnz": X.nnz, "groups": int(len(np.unique(topics))), "card": card(),
           "long_row_share": round(float(counts[counts > cap].sum()) / X.nnz, 4),
           "long_rows": int((counts > cap).sum())}
    torch.cuda.reset_peak_memory_stats()
    for name, kw in CONFIGS.items():
        run(ad, kw)
        out[name] = run(ad, kw)
        print(name, out[name], file=sys.stderr, flush=True)
    out["peak_device_gb"] = round(torch.cuda.max_memory_allocated() / 1e9, 2)

    # CPU leg: the numpy restatement on a 10 000-cell slice, the GPU on the same host matrix
    n_cpu = min(10_000, N)
    k = int(X.indptr[n_cpu])
    head = _device.DeviceCSR(X.indptr[:n_cpu + 1], X.indices[:k], X.data[:k], (n_cpu, D))
    sub = head.get()[:, :CPU_PEAKS]
    small = mu.SimpleAnnData(sub, obs=obs.iloc[:n_cpu])
    cpu = {"cells": n_cpu, "peaks": sub.shape[1], "impl": "oracle/rank_ref.py (numpy/scipy restatement, not scanpy)"}
    for name in ("t-test", "wilcoxon"):
        kw = CONFIGS[name]
        t0 = time.perf_counter()
        rank_ref.rank_genes_groups(small, "topic", **kw)
        cpu[f"{name}_cpu_s"] = round(time.perf_counter() - t0, 3)
        _rank.rank_genes_groups(small, "topic", **kw)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        _rank.rank_genes_groups(small, "topic", **kw)
        torch.cuda.synchronize()
        cpu[f"{name}_gpu_s"] = round(time.perf_counter() - t0, 3)
    out["cpu_baseline"] = cpu
    print(json.dumps(out))


if __name__ == "__main__":
    main()
