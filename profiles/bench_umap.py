"""mu.tl.umap on a WNN graph: the layout after mu.pp.neighbors, one H100.

    python profiles/bench_umap.py [cells=1000000]

The graph is built as in bench_wnn.py (two L2-normalised embeddings, 50 + 30 dims, 30 planted clusters, per-modality
exact 15-NN, then mu.pp.neighbors) and is NOT timed.  One warm-up call, then one timed call of mu.tl.umap with
default arguments (200 epochs above 10 000 cells), bracketed by device synchronisation.  Spectral init needs at most
2 * n_components connected components; on a graph with more the script falls back to init_pos="random" and says so.
Prints one JSON line: wall time, ms per epoch (epoch kernels alone, CUDA events), sampled edges per second, the card
name and its power limit.
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
from muon_b200 import _device, _lib, _umap  # noqa: E402

N = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
k = 15
rng = np.random.default_rng(0)
c = rng.integers(0, 30, N)
mods = {}
for name, d in (("rna", 50), ("atac", 30)):
    R = rng.normal(size=(N, d)).astype(np.float32) + 3.0 * (np.eye(30, dtype=np.float32)[c] @ rng.normal(size=(30, d)).astype(np.float32))
    R /= np.linalg.norm(R, axis=1, keepdims=True)
    idx, dist = _device.knn_l2(torch.from_numpy(R).cuda(), k)
    g = sp.csr_matrix((dist[:, 1:].cpu().numpy().ravel().astype(np.float64), idx[:, 1:].cpu().numpy().ravel().astype(np.int64),
                       np.arange(0, N * (k - 1) + 1, k - 1)), shape=(N, N))
    ad = mu.SimpleAnnData(np.zeros((N, 1), dtype=np.float32))
    ad.obsm["X_emb"] = R
    ad.obsp["distances"] = g
    ad.uns["neighbors"] = {"params": {"n_neighbors": k, "use_rep": "X_emb"}, "distances_key": "distances"}
    mods[name] = ad
md = mu.SimpleMuData(mods)
mu.pp.neighbors(md)
W = md.obsp["connectivities"]
n_comp = _umap.components(W)[0]
init = "spectral" if n_comp <= 4 else "random"

mu.tl.umap(md, init_pos=init)                     # warm-up
torch.cuda.synchronize()
_lib.PROFILE = {}
t0 = time.perf_counter()
mu.tl.umap(md, init_pos=init)
torch.cuda.synchronize()
dt = time.perf_counter() - t0
prof, _lib.PROFILE = _lib.PROFILE, None
ev = prof["mub_umap_epoch_f32"]
epoch_ms = float(sum(a.elapsed_time(b) for a, b in ev))
G, n_epochs = _umap.prune(W, 0)
eps = _umap.epochs_per_sample(G.data).astype(np.float64)
sampled = float(np.floor((n_epochs - 1) / eps).sum())      # each entry is sampled once per multiple of eps_e in [1, n_epochs)
try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, timeout=30).stdout.strip().splitlines()[0]
except Exception:
    q = torch.cuda.get_device_name(0) + ", power limit unknown"
print(json.dumps({"metric": "mu.tl.umap on a WNN graph (2 modalities, 50+30 dims)", "cells": N, "stored_edges": int(W.nnz),
                  "kept_edges": int(G.nnz), "components": int(n_comp), "init_pos": init, "epochs": n_epochs,
                  "seconds": dt, "ms_per_epoch": epoch_ms / len(ev),
                  "sampled_edges_per_s": sampled / (epoch_ms / 1e3), "gpu": q}))
