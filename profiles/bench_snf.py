"""mu.tl.snf on planted-cluster kNN distance graphs, one H100.

    python profiles/bench_snf.py [cells=20000] [modalities=2] [--cpu-baseline N]

Each modality is 30 planted Gaussian clusters in 30 dimensions with its exact 15-NN distance graph (built on the
device as in bench_umap.py), NOT timed.  One warm-up call, then one timed call of mu.tl.snf with default arguments
(n_neighbors=20, 20 iterations), bracketed by device synchronisation.  Prints one JSON line: wall time, ms per
diffusion iteration (CUDA events around each iteration), the bytes the diffusion kernels gather per second against
the H100 SXM's 3.35 TB/s HBM3 peak, peak device memory, the card name and its power limit.

The gathered bytes count one float64 operand load per stored entry of S and output column: N k N for the
transposed product and, for the mirrored one, N k times the columns of the upper-triangle tiles of each row (S has
k entries per column, so N k per product; the per-row split is taken as k per row).  Most of these loads are served
from L2, so the rate can exceed the HBM peak; it is the kernels' operand throughput, not HBM traffic.

With ``--cpu-baseline N`` it also times, on the host at N cells and the same modality count (dense distances),
oracle/snf_ref.py (sparse S products) and its dense ``np.dot`` variant, which is the reference's arithmetic.
"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import scipy.sparse as sp
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import muon_b200 as mu  # noqa: E402
from muon_b200 import _device, _snf  # noqa: E402

args = [a for a in sys.argv[1:] if not a.startswith("--")]
cpu_n = None
if "--cpu-baseline" in sys.argv:
    cpu_n = int(sys.argv[sys.argv.index("--cpu-baseline") + 1])
    args = [a for a in args if a != str(cpu_n)]
N = int(args[0]) if len(args) > 0 else 20000
M = int(args[1]) if len(args) > 1 else 2
K, KG, ITERS, TILE = 20, 15, 20, 64

rng = np.random.default_rng(0)
c = rng.integers(0, 30, N)
mods = {}
for m in range(M):
    X = rng.normal(size=(N, 30)).astype(np.float32) + 3.0 * rng.normal(size=(30, 30)).astype(np.float32)[c]
    idx, dist = _device.knn_l2(torch.from_numpy(X).cuda(), KG + 1)
    g = sp.csr_matrix((dist[:, 1:].cpu().numpy().ravel().astype(np.float64),
                       idx[:, 1:].cpu().numpy().ravel().astype(np.int64), np.arange(0, N * KG + 1, KG)), shape=(N, N))
    del idx, dist
    ad = mu.SimpleAnnData(np.zeros((N, 1), dtype=np.float32))
    ad.obsp["distances"] = g
    ad.uns["neighbors"] = {"params": {"n_neighbors": KG}, "distances_key": "distances"}
    mods[f"m{m}"] = ad
md = mu.SimpleMuData(mods)
torch.cuda.empty_cache()

mu.tl.snf(md)                                        # warm-up
torch.cuda.synchronize()
torch.cuda.reset_peak_memory_stats()
base = torch.cuda.memory_allocated()
t0 = time.perf_counter()
mu.tl.snf(md)
torch.cuda.synchronize()
dt = time.perf_counter() - t0
peak = torch.cuda.max_memory_allocated() - base

# the diffusion alone, per iteration (CUDA events)
ev = []
_snf.fuse([md.mod[m].obsp["distances"] for m in md.mod], n_neighbors=K, n_iterations=ITERS, timings=ev)
torch.cuda.synchronize()
it_ms = [a.elapsed_time(b) for a, b in ev]
cols = N - TILE * (np.arange(N) // TILE)             # columns of the upper-triangle tiles of each row
gathered = M * 8.0 * (N * K * N + K * float(cols.sum()))
ms = float(np.median(it_ms))
try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, timeout=30).stdout.strip().splitlines()[0]
except Exception:
    q = torch.cuda.get_device_name(0) + ", power limit unknown"
out = {"metric": "mu.tl.snf on planted-cluster 15-NN distance graphs", "cells": N, "modalities": M,
       "n_neighbors": K, "iterations": ITERS, "seconds": dt, "ms_per_iteration": ms,
       "ms_per_iteration_min_max": [float(min(it_ms)), float(max(it_ms))],
       "gathered_bytes_per_iteration": gathered, "gathered_TB_per_s": gathered / (ms / 1e3) / 1e12,
       "gathered_over_hbm_peak": gathered / (ms / 1e3) / 3.35e12,
       "peak_device_GiB": peak / 2**30, "budget_GiB": (2 * M + 2) * N * N * 8 / 2**30, "gpu": q}

if cpu_n:
    from oracle import snf_ref as R
    dists, _ = R.planted_distances(cpu_n, M, seed=0)
    t0 = time.perf_counter()
    R.snf_ref(dists, n_neighbors=K, n_iterations=ITERS)
    t_sparse = time.perf_counter() - t0
    t0 = time.perf_counter()
    R.snf_dense_dot(dists, n_neighbors=K, n_iterations=ITERS)
    t_dense = time.perf_counter() - t0
    md_small = mu.SimpleMuData({f"m{m}": mu.SimpleAnnData(np.zeros((cpu_n, 1))) for m in range(M)})
    for m, a in zip(range(M), md_small.mod.values()):
        a.obsp["distances"] = dists[m]
        a.uns["neighbors"] = {"params": {}, "distances_key": "distances"}
    mu.tl.snf(md_small)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    mu.tl.snf(md_small)
    torch.cuda.synchronize()
    out["cpu_baseline"] = {"cells": cpu_n, "host_sparse_products_s": t_sparse, "host_dense_np_dot_s": t_dense,
                           "gpu_same_input_s": time.perf_counter() - t0, "host_threads": os.cpu_count()}
print(json.dumps(out))
