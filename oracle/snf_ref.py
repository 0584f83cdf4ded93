"""Float64 numpy / scipy restatement of ``mu.tl.snf`` (muon_b200/_snf.py), for the tests and the benchmark.

It states the semantics of DESIGN.md section 8 once, in the reference's own arithmetic (muon/_core/tools.py:716-920):
the affinity, ``_normalize``, ``_dominateset`` with its broadcasting quirk, the diffusion and the two final row
selections.  Where the reference is unusable or unspecified it takes the project's rules:
  * sparse distances: (D + D^T) / 2, ``setdiag(0)``, ``eliminate_zeros()`` as scipy does them, then every unstored
    off-diagonal entry is +inf with affinity 0;
  * every top-k selection breaks ties by ascending column (stable sorts).
The dominate sets are scipy sparse matrices, so S P S^T costs O(N^2 k) and N = 4000 runs in seconds.
``snf_dense_dot`` is the same computation with the reference's dense ``np.dot`` products, for timing.
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp
import scipy.stats as stats

EPS = np.finfo(np.float64).eps


def symmetrised(dist) -> np.ndarray:
    """The dense symmetrised distance matrix the affinity starts from (diagonal 0, unstored sparse entries +inf)."""
    if sp.issparse(dist):
        D = sp.csr_matrix(dist, dtype=np.float64)
        D = sp.csr_matrix((D + D.T) / 2)
        D.setdiag(0)
        D.eliminate_zeros()
        F = np.full(D.shape, np.inf)
        Q = D.tocoo()
        F[Q.row, Q.col] = Q.data
        np.fill_diagonal(F, 0.0)
        return F
    D = np.asarray(dist, dtype=np.float64)
    D = (D + D.T) / 2
    np.fill_diagonal(D, 0)
    return D


def affinity(D: np.ndarray, k: int, sigma: float, eps: float = EPS) -> np.ndarray:
    """The reference's ``_affinity_matrix`` on a symmetrised dense D; +inf distances get affinity 0."""
    srt = np.sort(D, axis=1)[:, 1:k + 1]
    fin = ~np.isinf(srt)
    with np.errstate(invalid="ignore", divide="ignore"):
        means = np.where(fin, srt, 0.0).sum(axis=1) / fin.sum(axis=1) + eps
        sig = np.add.outer(means, means) / 3 + D / 3 + eps
        dens = stats.norm(0, sigma * sig).pdf(D)
    dens = np.where(np.isinf(D), 0.0, dens)
    return (dens + dens.T) / 2


def normalize(x: np.ndarray) -> np.ndarray:
    """The reference's ``_normalize``."""
    row_sum_mdiag = x.sum(axis=1) - x.diagonal()
    row_sum_mdiag[row_sum_mdiag == 0] = 1
    x = x / (2 * row_sum_mdiag[:, None])
    np.fill_diagonal(x, 0.5)
    return (x + x.T) / 2


def dominate_set(W: np.ndarray, k: int):
    """The reference's ``_dominateset``: keep the top k of each column (ties: lower row first), then divide entry
    [i, j] by row sum j (numpy's broadcast of ``x / x.sum(axis=1)``).  Returned as a CSR matrix."""
    n = W.shape[0]
    if k >= n:
        raise ValueError("'n_neighbors' seems to be too high.")
    order = np.argsort(-W, axis=0, kind="stable")[:k]            # [k x n]: row indices kept in each column
    cols = np.broadcast_to(np.arange(n), order.shape)
    X = sp.csr_matrix((W[order, cols].ravel(), (order.ravel(), cols.ravel())), shape=(n, n))
    rs = np.asarray(X.sum(axis=1)).ravel()
    return sp.csr_matrix(X.multiply(1.0 / rs[None, :]))


def row_smallest(x: np.ndarray, k: int):
    """``_sparse_csr_fast_knn(csr_matrix(x), k)``: per row the k smallest non-zero entries, ascending (ties: lower
    column first), as a ``csr_array``."""
    n = x.shape[0]
    idx = np.empty((n, k), dtype=np.int64)
    val = np.empty((n, k))
    for i in range(n):
        nz = np.flatnonzero(x[i])
        if nz.size < k:
            raise ValueError(f"row {i} has only {nz.size} non-zero entries")
        o = nz[np.argsort(x[i, nz], kind="stable")[:k]]
        idx[i], val[i] = o, x[i, o]
    return sp.csr_array((val.ravel(), idx.ravel(), np.arange(0, n * k + 1, k)), shape=(n, n))


def _fuse(distances, n_neighbors, n_iterations, sigma, eps, product, steps=None):
    wall = [normalize(affinity(symmetrised(d), n_neighbors, sigma, eps)) for d in distances]
    new = [dominate_set(w, n_neighbors) for w in wall]
    m = len(wall)
    for it in range(n_iterations):
        nxt = []
        for j in range(m):
            sumWJ = np.zeros_like(wall[j])
            for q in range(m):
                if q != j:
                    sumWJ = sumWJ + wall[q]
            nxt.append(product(new[j], sumWJ / (m - 1)))
        wall = [normalize(x) for x in nxt]
        if steps is not None:
            steps.append(normalize(np.sum(wall, axis=0) / m))
    w = normalize(np.sum(wall, axis=0) / m)
    return w, wall


def _sparse_product(S, P):
    return np.asarray((S @ np.asarray((S @ P).T)).T)     # S P S^T = (S (S P)^T)^T with two sparse x dense products


def _dense_product(S, P):
    Sd = S.toarray()
    return np.dot(np.dot(Sd, P), Sd.T)


def snf_ref(distances, n_neighbors=20, n_iterations=20, sigma=0.5, eps=EPS, *, steps=None):
    """SNF of the per-modality distances -> dict(distances, connectivities, w, modalities).  ``steps``, a list,
    receives the fused matrix after every iteration."""
    w, wall = _fuse(distances, n_neighbors, n_iterations, sigma, eps, _sparse_product, steps)
    return {"distances": row_smallest(0.5 - w, n_neighbors), "connectivities": row_smallest(w, n_neighbors),
            "w": w, "modalities": wall}


def snf_dense_dot(distances, n_neighbors=20, n_iterations=20, sigma=0.5, eps=EPS):
    """The fused matrix with the reference's dense ``np.dot`` products (for host timing)."""
    return _fuse(distances, n_neighbors, n_iterations, sigma, eps, _dense_product)[0]


def planted_distances(n, n_mod, *, n_clusters=3, dim=10, k_graph=None, seed=0):
    """Per-modality Euclidean distances of ``n`` points in ``n_clusters`` planted Gaussian clusters (labels i *
    n_clusters // n).  ``k_graph``: the exact ``k_graph``-nearest-neighbour distance graph (CSR, one direction per
    stored edge, as ``sc.pp.neighbors`` stores it) instead of the dense matrix."""
    from scipy.spatial.distance import cdist
    rng = np.random.default_rng(seed)
    labels = np.arange(n) * n_clusters // n
    out = []
    for _ in range(n_mod):
        X = rng.normal(size=(n, dim)) + rng.normal(size=(n_clusters, dim))[labels] * 3
        D = cdist(X, X)
        if k_graph is None:
            out.append(D)
            continue
        np.fill_diagonal(D, np.inf)
        nb = np.argpartition(D, k_graph, axis=1)[:, :k_graph]
        rows = np.repeat(np.arange(n), k_graph)
        out.append(sp.csr_matrix((D[rows, nb.ravel()], (rows, nb.ravel())), shape=(n, n)))
    return out, labels
