"""mu.tl.leiden / mu.tl.louvain on the graphs mu.pp.neighbors builds, one H100.

    python profiles/bench_leiden.py [cells=1000000]

The two modality graphs and the WNN graph are built as in bench_umap.py (two L2-normalised embeddings, 50 + 30 dims,
30 planted clusters, per-modality exact 15-NN, then mu.pp.neighbors) and are NOT timed.  Then one warm-up call and
one timed call, each bracketed by device synchronisation, of
  * multiplex mu.tl.leiden(md) and mu.tl.louvain(md) on the two modality graphs (the MuData branch: unit weights,
    leiden with n_iterations=2, louvain until nothing changes);
  * the single-graph branch, mu.tl.leiden / mu.tl.louvain on the WNN graph (scanpy's defaults: weighted leiden with
    n_iterations=-1, unweighted louvain).
For each: wall time, levels, sweeps, refinement rounds, kernel time (sum of CUDA events around the leiden.cu entry
points), clusters and the quality sum_l w_l Q_l.  If networkx is importable it also runs networkx's
louvain_communities (a different, sequential Python Louvain -- not leidenalg) and mu.tl.louvain on the WNN subgraph of
the first 50 000 cells, and reports both qualities and times.  Prints one JSON line with the card name and its power
limit.
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
from muon_b200 import _device, _leiden, _lib  # noqa: E402
from muon_b200.pp import _umap_connectivities  # noqa: E402

N = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
k = 15
rng = np.random.default_rng(0)
c = rng.integers(0, 30, N)
mods, conns = {}, {}
for name, d in (("rna", 50), ("atac", 30)):
    R = rng.normal(size=(N, d)).astype(np.float32) + 3.0 * (np.eye(30, dtype=np.float32)[c] @ rng.normal(size=(30, d)).astype(np.float32))
    R /= np.linalg.norm(R, axis=1, keepdims=True)
    idx, dist = _device.knn_l2(torch.from_numpy(R).cuda(), k)
    conn = _umap_connectivities(idx.to(torch.int64), dist, N)     # the modality's own graph, as scanpy builds it
    g = sp.csr_matrix((dist[:, 1:].cpu().numpy().ravel().astype(np.float64), idx[:, 1:].cpu().numpy().ravel().astype(np.int64),
                       np.arange(0, N * (k - 1) + 1, k - 1)), shape=(N, N))
    ad = mu.SimpleAnnData(np.zeros((N, 1), dtype=np.float32))
    ad.obsm["X_emb"] = R
    ad.obsp["distances"] = g
    ad.uns["neighbors"] = {"params": {"n_neighbors": k, "use_rep": "X_emb"}, "distances_key": "distances"}
    mods[name] = ad
    conns[name] = conn
md = mu.SimpleMuData(mods)
mu.pp.neighbors(md)
for name, ad in mods.items():
    ad.obsp["connectivities"] = conns[name]
    ad.uns["neighbors"]["connectivities_key"] = "connectivities"
W = md.obsp["connectivities"]
wnn = mu.SimpleAnnData(np.zeros((N, 1), dtype=np.float32))
wnn.obsp["connectivities"] = W
wnn.uns["neighbors"] = {"connectivities_key": "connectivities", "params": {}}


def layers_of(target, alg):
    if target is md:
        return [_leiden.layer_matrix(mods[m].obsp["connectivities"], False) for m in mods], [1.0] * len(mods)
    return [_leiden.layer_matrix(W, alg == "leiden")], [1.0]


def quality(labels, layers, weights):
    P = _leiden.Problem(layers, weights, [1.0] * len(layers))
    return _leiden.Level.from_problem(P).quality(torch.from_numpy(labels.astype(np.int32)).cuda())


def timed(fn, target, alg):
    fn(target)                                         # warm-up
    torch.cuda.synchronize()
    stats = {}
    real = _leiden.optimise

    def counting(*a, **kw):
        kw["stats"] = stats
        return real(*a, **kw)
    _leiden.optimise = counting
    _lib.PROFILE = {}
    t0 = time.perf_counter()
    fn(target)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    prof, _lib.PROFILE = _lib.PROFILE, None
    _leiden.optimise = real
    kernel_ms = sum(a.elapsed_time(b) for name, ev in prof.items() if name.startswith("mub_leiden") for a, b in ev)
    key = "leiden" if alg == "leiden" else "louvain"
    labels = np.asarray(target.obs[key].astype(int))
    layers, weights = layers_of(target, alg)
    return {"seconds": dt, "kernel_ms": kernel_ms, "clusters": int(labels.max()) + 1,
            "quality": quality(labels, layers, weights), **stats}


out = {"metric": "mu.tl.leiden / louvain on neighbour graphs (2 modalities, 50+30 dims, 15-NN)", "cells": N,
       "edges": {m: int(mods[m].obsp["connectivities"].nnz) for m in mods} | {"wnn": int(W.nnz)}}
out["multiplex_leiden"] = timed(mu.tl.leiden, md, "leiden")
out["multiplex_louvain"] = timed(mu.tl.louvain, md, "louvain")
out["wnn_leiden"] = timed(mu.tl.leiden, wnn, "leiden")
out["wnn_louvain"] = timed(mu.tl.louvain, wnn, "louvain")

try:
    import networkx as nx
except ImportError:
    nx = None
if nx is not None:
    n_sub = min(50_000, N)
    S = sp.csr_matrix(W[:n_sub][:, :n_sub])
    sub = mu.SimpleAnnData(np.zeros((n_sub, 1), dtype=np.float32))
    sub.obsp["connectivities"] = S
    sub.uns["neighbors"] = {"connectivities_key": "connectivities", "params": {}}
    mu.tl.louvain(sub, use_weights=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    mu.tl.louvain(sub, use_weights=True)
    torch.cuda.synchronize()
    t_gpu = time.perf_counter() - t0
    gpu_labels = np.asarray(sub.obs["louvain"].astype(int))
    A = _leiden.layer_matrix(S, True)
    t0 = time.perf_counter()
    parts = nx.community.louvain_communities(nx.from_scipy_sparse_array(A), weight="weight", seed=0)
    t_nx = time.perf_counter() - t0
    nx_labels = np.empty(n_sub, dtype=np.int64)
    for i, p in enumerate(parts):
        nx_labels[list(p)] = i
    out["same_graph_vs_networkx_louvain"] = {
        "cells": n_sub, "edges": int(S.nnz), "gpu_seconds": t_gpu, "networkx_seconds": t_nx,
        "gpu_quality": quality(gpu_labels, [A], [1.0]), "networkx_quality": quality(nx_labels, [A], [1.0]),
        "gpu_clusters": int(gpu_labels.max()) + 1, "networkx_clusters": len(parts)}
else:
    out["same_graph_vs_networkx_louvain"] = "not measured: networkx is not importable"
try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, timeout=30).stdout.strip().splitlines()[0]
except Exception:
    q = torch.cuda.get_device_name(0) + ", power limit unknown"
out["gpu"] = q
print(json.dumps(out))
