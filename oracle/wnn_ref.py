"""TEST INFRASTRUCTURE ONLY (CPU oracle) -- WNN (``muon.pp.neighbors``) restated in numpy with exact searches.

Follows the reference driver step by step (muon/_core/preproc.py:264-640):
  :399-407  nndistances_i = smallest stored distance of cell i in its modality's kNN graph
  :425      bbox_norm = ||max - min|| of the representation
  :452-460  n_bandwidth_neighbors cells minimising the tie-breaking metric of :51-76
            (N - jd N) + (bbox - e)/bbox for cells whose kNN sets overlap (jd = Jaccard distance < 1), N + 1 otherwise
            -- found here by exhaustive evaluation + stable sort (the reference asks NN-descent)
  :462-470  sigma_i = mean Euclidean distance to those cells
  :478-506  theta per pair of modalities (neighbour means over the non-zero stored distances), ratios, softmax ->
            cell-modality weights
  :509-567  candidates = union over modalities of the n_multineighbors nearest cells (exact)
  :569-602  affinity sum_m w_im exp(-d_m(i,j)/sigma_im), distance sqrt(0.5 (1 - affinity))
  :604      n_neighbors + 1 smallest per cell (numba helper :114-135)
  :607-614  UMAP connectivities (oracle/_third_party.py::umap_connectivities)

Pinned against the reference's own control flow executed with exact-search stand-ins
(tests/golden/wnn_small.npz, tests/test_oracle_wnn.py): weights to 4e-16, distances to 2e-16.
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp
from scipy.spatial.distance import cdist
from scipy.special import softmax

from ._third_party import umap_connectivities


def _nonzero_neighbours(g, i):
    """Neighbours of cell i with a non-zero stored distance: the reference takes ``graph[i, :].nonzero()``
    (preproc.py:480-483), which skips explicitly stored zeros such as a duplicate cell."""
    a, b = g.indptr[i], g.indptr[i + 1]
    return g.indices[a:b][g.data[a:b] != 0]


def wnn_ref(reps, graphs, n_neighbors, n_bandwidth_neighbors=20, n_multineighbors=200, eps=1e-4):
    """``reps``: list of n x d_m arrays; ``graphs``: list of n x n CSR kNN distance graphs (one per modality).
    Returns dict(weights n x M, sigma list, distances CSR (n_neighbors+1 per row, ascending), connectivities CSR)."""
    M = len(reps)
    N = reps[0].shape[0]
    reps = [np.asarray(r, dtype=np.float64) for r in reps]
    graphs = [sp.csr_matrix(g) for g in graphs]
    sig, nnd = [], []
    for x, g in zip(reps, graphs):
        nnd.append(np.minimum.reduceat(g.data, g.indptr[:-1]))
        bbox = np.linalg.norm(np.ptp(x, axis=0))
        S = [set(g.indices[g.indptr[i]:g.indptr[i + 1]].tolist()) for i in range(N)]
        E = cdist(x, x)
        s = np.zeros(N)
        for i in range(N):
            vals = np.full(N, N + 1.0)
            for j in range(N):
                if j == i:
                    continue
                c = len(S[i] & S[j])
                if c:
                    u = len(S[i]) + len(S[j]) - c
                    vals[j] = (N - (u - c) / u * N) + (bbox - E[i, j]) / bbox
            s[i] = E[i, np.argsort(vals, kind="stable")[:n_bandwidth_neighbors]].mean()
        sig.append(s)
    ratios = np.full((N, M), -np.inf)
    for i1 in range(M):
        th = []
        for i2 in range(M):
            g = graphs[i2]
            r = np.stack([reps[i1][_nonzero_neighbours(g, i)].mean(0) for i in range(N)])
            th.append(np.exp(-np.maximum(np.linalg.norm(reps[i1] - r, axis=1) - nnd[i1], 0) / (sig[i1] - nnd[i1])))
        other = np.max([t for i2, t in enumerate(th) if i2 != i1], axis=0) if M > 1 else -np.inf
        ratios[:, i1] = th[i1] / (other + eps)
    w = softmax(ratios, axis=1)
    kc = min(n_multineighbors + 1, N)
    cand = [np.argsort(cdist(x, x), axis=1, kind="stable")[:, 1:kc] for x in reps]
    k1 = n_neighbors + 1
    idx = np.zeros((N, k1), dtype=np.int64)
    dist = np.zeros((N, k1))
    for i in range(N):
        u = np.unique(np.concatenate([c[i] for c in cand]))
        u = u[u != i]
        aff = sum(w[i, m] * np.exp(-np.linalg.norm(reps[m][i] - reps[m][u], axis=1) / sig[m][i]) for m in range(M))
        d = np.sqrt(0.5 * (1 - aff))
        o = np.argsort(d, kind="stable")[:k1]
        idx[i], dist[i] = u[o], d[o]
    D = sp.csr_matrix((dist.ravel(), idx.ravel(), np.arange(0, (N + 1) * k1, k1)), shape=(N, N))
    C = umap_connectivities(idx, dist, n_obs=N, n_neighbors=k1)
    return {"weights": w, "sigma": sig, "distances": D, "connectivities": C, "knn_indices": idx, "knn_dists": dist}


def wnn_cells_ref(cells, reps, graphs, n_neighbors, n_bandwidth_neighbors=20, n_multineighbors=200, eps=1e-4):
    """``wnn_ref`` restated for the cells ``cells`` alone, so that it scales to large N: everything cell i needs is
    local to it -- sigma_i from the overlap counts ``B[i] @ B.T`` of the boolean kNN graph and the exact distances
    from i, theta and the weights from i's neighbour means, the candidates from the float64 kNN of i, and the
    affinities.  Returns dict(weights len(cells) x M, sigma list, knn_indices, knn_dists) in the order of ``cells``."""
    cells = np.asarray(cells, dtype=np.int64)
    M = len(reps)
    N = reps[0].shape[0]
    reps = [np.asarray(r, dtype=np.float64) for r in reps]
    graphs = [sp.csr_matrix(g) for g in graphs]
    bboxes = [np.linalg.norm(np.ptp(x, axis=0)) for x in reps]
    Bs = [sp.csr_matrix((np.ones_like(g.data), g.indices, g.indptr), shape=g.shape) for g in graphs]
    BTs = [B.T.tocsr() for B in Bs]
    sig = np.empty((M, len(cells)))
    nnd = np.empty((M, len(cells)))
    E = []                                           # per modality: distances from each cell to every cell
    for m, (x, g, B, BT) in enumerate(zip(reps, graphs, Bs, BTs)):
        size = np.diff(g.indptr).astype(np.float64)
        Em = cdist(x[cells], x)
        E.append(Em)
        for c, i in enumerate(cells):
            nnd[m, c] = g.data[g.indptr[i]:g.indptr[i + 1]].min()
            cnt = np.asarray((B[i] @ BT).todense()).ravel()
            cnt[i] = 0
            vals = np.full(N, N + 1.0)
            j = np.nonzero(cnt)[0]
            u = size[i] + size[j] - cnt[j]
            vals[j] = (N - (u - cnt[j]) / u * N) + (bboxes[m] - Em[c, j]) / bboxes[m]
            sig[m, c] = Em[c, np.argsort(vals, kind="stable")[:n_bandwidth_neighbors]].mean()
    ratios = np.full((len(cells), M), -np.inf)
    for i1 in range(M):
        th = []
        for i2 in range(M):
            r = np.stack([reps[i1][_nonzero_neighbours(graphs[i2], i)].mean(0) for i in cells])
            th.append(np.exp(-np.maximum(np.linalg.norm(reps[i1][cells] - r, axis=1) - nnd[i1], 0) / (sig[i1] - nnd[i1])))
        other = np.max([t for i2, t in enumerate(th) if i2 != i1], axis=0) if M > 1 else -np.inf
        ratios[:, i1] = th[i1] / (other + eps)
    w = softmax(ratios, axis=1)
    kc = min(n_multineighbors + 1, N)
    k1 = n_neighbors + 1
    idx = np.zeros((len(cells), k1), dtype=np.int64)
    dist = np.zeros((len(cells), k1))
    for c, i in enumerate(cells):
        u = np.unique(np.concatenate([np.argsort(E[m][c], kind="stable")[1:kc] for m in range(M)]))
        u = u[u != i]
        aff = sum(w[c, m] * np.exp(-E[m][c, u] / sig[m, c]) for m in range(M))
        d = np.sqrt(0.5 * (1 - aff))
        o = np.argsort(d, kind="stable")[:k1]
        idx[c], dist[c] = u[o], d[o]
    return {"weights": w, "sigma": list(sig), "knn_indices": idx, "knn_dists": dist}
