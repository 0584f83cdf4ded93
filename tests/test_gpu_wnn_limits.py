"""GPU: mu.pp.neighbors (WNN, csrc/wnn.cu) at its limits against the float64 restatements in oracle/wnn_ref.py --
three and four modalities, cells that share kNN neighbours with fewer than n_bandwidth_neighbors cells, duplicate
cells, and 150 000 cells with the query blocks of low_memory."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

import muon_b200 as mu
from muon_b200 import _device
from muon_b200._containers import SimpleAnnData, SimpleMuData
from oracle import _third_party as tp
from oracle.wnn_ref import wnn_cells_ref, wnn_ref

pytestmark = pytest.mark.gpu


def _graph(idx, dist, n):
    k = idx.shape[1]
    return sp.csr_matrix((dist.ravel().astype(np.float64), idx.ravel().astype(np.int64), np.arange(0, n * k + 1, k)),
                         shape=(n, n))


def _exact_graphs(reps, k):
    """Exact kNN graphs (k - 1 stored neighbours, self dropped wherever it sits, so a duplicate cell keeps its twin
    at an explicit zero distance)."""
    graphs = []
    for R in reps:
        idx, dist, _ = tp.nearest_neighbors(R, k + 1, "euclidean")
        n = R.shape[0]
        keep = [np.where(r != i)[0][:k - 1] for i, r in enumerate(idx)]
        graphs.append(_graph(np.stack([idx[i, c] for i, c in enumerate(keep)]),
                             np.stack([dist[i, c] for i, c in enumerate(keep)]), n))
    return graphs


def _mudata(reps, graphs, k):
    mods = {}
    for m, (R, g) in enumerate(zip(reps, graphs)):
        ad = SimpleAnnData(np.zeros((R.shape[0], 1), dtype=np.float32))
        ad.obsm["X_emb"] = np.asarray(R, dtype=np.float32)
        ad.obsp["d"] = g
        ad.uns["nn"] = {"params": {"n_neighbors": k, "use_rep": "X_emb"}, "distances_key": "d"}
        mods[f"m{m}"] = ad
    return SimpleMuData(mods), {f"m{m}": "nn" for m in range(len(reps))}


def _run(reps, graphs, k, **kw):
    md, keys = _mudata(reps, graphs, k)
    mu.pp.neighbors(md, neighbor_keys=keys, **kw)
    W = np.stack([md.obs[f"m{m}:mod_weight"].to_numpy() for m in range(len(reps))], 1)
    D = sp.csr_matrix(md.obsp["distances"])
    n = D.shape[0]
    k1 = k + 1
    assert np.all(np.diff(D.indptr) == k1)
    return W, D.indices.reshape(n, k1), D.data.reshape(n, k1), sp.csr_matrix(md.obsp["connectivities"])


def _compare_rows(cells, idx, dist, ref, reps, min_same=0.98, must_match=()):
    """Rows ``cells`` of the product's distance graph (idx / dist, stored order) against the float64 reference's
    rows (aligned with ``cells``).  Nearly every row must hold the same neighbours in the same order with the same
    distances.  A row that differs may only differ by a tie: the distances of the cells it returns, recomputed in
    float64 with the reference's weights and bandwidths, must be its stored distances and must equal the
    reference's distances place by place.  The cells in ``must_match`` must match exactly."""
    ridx, rdist, w = ref["knn_indices"], ref["knn_dists"], ref["weights"]
    assert np.all(np.diff(dist, axis=1) >= 0)
    same = np.all(idx == ridx, axis=1)
    assert same.mean() >= min_same, same.mean()
    assert same[list(must_match)].all()
    np.testing.assert_allclose(dist[same], rdist[same], rtol=1e-5, atol=1e-7)
    for r in np.where(~same)[0]:
        i, js = cells[r], idx[r]
        assert i not in js and len(set(js.tolist())) == len(js)
        aff = sum(w[r, m] * np.exp(-np.linalg.norm(reps[m][i] - reps[m][js], axis=1) / ref["sigma"][m][r])
                  for m in range(len(reps)))
        np.testing.assert_allclose(dist[r], np.sqrt(0.5 * (1 - aff)), rtol=1e-5, atol=1e-7)
        np.testing.assert_allclose(dist[r], rdist[r], rtol=1e-5, atol=1e-7)
    return same


def _compare(reps, graphs, k, n_multineighbors, **kw):
    W, idx, dist, C = _run(reps, graphs, k, n_multineighbors=n_multineighbors, **kw)
    ref = wnn_ref(reps, graphs, k, n_multineighbors=n_multineighbors, **kw)
    np.testing.assert_allclose(W, ref["weights"], rtol=2e-5, atol=1e-7)
    same = _compare_rows(np.arange(len(idx)), idx, dist, ref, reps)
    # connectivities: the fuzzy union of row i involves the rows of i's neighbours -- compare where all of them agree,
    # including which distances are exactly zero: a duplicate cell sits at sqrt(0.5 (1 - sum_m w_m)), 0 or ~7e-9
    # depending on the last bit of the weights, and UMAP's rho is the smallest non-zero distance of the row
    same &= np.array([np.array_equal(np.sort(a) > 0, np.sort(b) > 0) for a, b in zip(dist, ref["knn_dists"])])
    Cr = ref["connectivities"].tocsr()
    assert (C != C.T).nnz == 0
    for i in np.where(same)[0]:
        nb = np.union1d(C[i].indices, Cr[i].indices)
        if same[nb].all():
            np.testing.assert_allclose(C[i].toarray(), Cr[i].toarray(), atol=1e-4)
    return ref


def _modalities(n, dims, seed, n_clusters=4):
    rng = np.random.default_rng(seed)
    c = rng.integers(0, n_clusters, n)
    reps = []
    for d in dims:
        R = rng.normal(size=(n, d)) + 2.5 * np.eye(n_clusters)[c] @ rng.normal(size=(n_clusters, d))
        reps.append((R / np.linalg.norm(R, axis=1, keepdims=True)).astype(np.float32).astype(np.float64))
    return reps


# ---- 7. three and four modalities ---------------------------------------------------------------------------------
@pytest.mark.parametrize("dims,n_multi", [((12, 5, 8), 40), ((12, 5, 8, 20), 40), ((12, 5, 8, 20), 300)])
def test_three_and_four_modalities(cuda, dims, n_multi):
    """kWnnMaxMod = 4.  4 x 300 puts up to 1 200 candidates per cell into the 2 048-slot table of
    wnn_affinity_topk_kernel."""
    N, k = 400, 10
    reps = _modalities(N, dims, seed=len(dims) + n_multi)
    graphs = _exact_graphs(reps, k)
    _compare(reps, graphs, k, n_multi)


# ---- 8. the bandwidth search's fill-up path ------------------------------------------------------------------------
def _isolated(seed=8, n_main=300, sizes=(5, 8, 12, 15)):
    rng = np.random.default_rng(seed)
    reps = []
    for d in (10, 6):
        parts = [rng.normal(size=(n_main, d))]
        for s in sizes:
            u = rng.normal(size=d)
            parts.append(40.0 * u / np.linalg.norm(u) + 0.3 * rng.normal(size=(s, d)))
        reps.append(np.concatenate(parts).astype(np.float32).astype(np.float64))
    return reps


def test_cells_with_few_overlapping_cells_fill_the_bandwidth_set(cuda):
    """Small clusters far from the rest: their cells share kNN neighbours with fewer than 20 cells, and step 4 of
    wnn_bandwidth_kernel completes the set with ties at N + 1, lowest index first, the cell itself included."""
    k = 8
    reps = _isolated()
    graphs = _exact_graphs(reps, k)
    for g in graphs:
        B = sp.csr_matrix((np.ones_like(g.data), g.indices, g.indptr), shape=g.shape)
        overlap = np.diff((B @ B.T).tocsr().indptr) - 1              # cells sharing a neighbour, self excluded
        assert (overlap < 20).sum() >= 20
    _compare(reps, graphs, k, 30)


# ---- 9. duplicate cells -------------------------------------------------------------------------------------------
def test_duplicate_cells(cuda):
    """Repeated rows: the kNN graphs store explicit zero distances (the reference's neighbour means skip them),
    and the candidate lists meet exact ties at distance 0, where dropping the first column of the kNN result is
    not the same as dropping the cell itself."""
    N0, k = 300, 10
    rng = np.random.default_rng(9)
    base = _modalities(N0, (12, 6), seed=9)
    rows = np.concatenate([np.arange(N0), rng.choice(N0, 40, replace=False), rng.choice(N0, 10, replace=False)])
    perm = rng.permutation(len(rows))
    reps = [np.ascontiguousarray(R[rows[perm]]) for R in base]
    graphs = _exact_graphs(reps, k)
    assert all((g.data == 0).sum() >= 40 for g in graphs)
    _compare(reps, graphs, k, 30)


# ---- 10. 150 000 cells, low_memory query blocks ----------------------------------------------------------------------
def test_wnn_at_150k_cells_against_the_per_cell_restatement(cuda):
    """Two modalities (50 and 30 dims) generated as in profiles/bench_wnn.py, input graphs from knn_l2,
    n_multineighbors = 200, low_memory at its default (on above 50 000 cells: two query blocks of the candidate
    search).  About 200 cells against oracle/wnn_ref.py::wnn_cells_ref."""
    N, k = 150_000, 15
    rng = np.random.default_rng(0)
    c = rng.integers(0, 30, N)
    reps, graphs = [], []
    for d in (50, 30):
        R = rng.normal(size=(N, d)).astype(np.float32) + \
            3.0 * (np.eye(30, dtype=np.float32)[c] @ rng.normal(size=(30, d)).astype(np.float32))
        R /= np.linalg.norm(R, axis=1, keepdims=True)
        idx, dist = _device.knn_l2(torch.from_numpy(R).to(cuda), k)
        graphs.append(_graph(idx[:, 1:].cpu().numpy(), dist[:, 1:].cpu().numpy(), N))
        reps.append(R.astype(np.float64))
    W, idx, dist, _ = _run(reps, graphs, k)
    cells = np.unique(np.concatenate([[0, N - 1, 131071, 131072], rng.choice(N, 196, replace=False)]))
    ref = wnn_cells_ref(cells, reps, graphs, k)
    np.testing.assert_allclose(W[cells], ref["weights"], rtol=2e-5, atol=1e-7)
    edges = np.searchsorted(cells, [0, N - 1, 131071, 131072])   # first / last cell, the two query blocks' seam
    _compare_rows(cells, idx[cells], dist[cells], ref, reps, min_same=0.97, must_match=edges)
