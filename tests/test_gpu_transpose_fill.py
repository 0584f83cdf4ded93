"""The tiled transposition fill (transpose.cu, mub_csr_transpose_fill_tiled) at its edges.  Every transposed row panel
must equal scipy's transpose of the same rows byte for byte: transposed rows in ascending cell order, the TF-IDF value
bits unchanged.  The matrices hold empty rows, rows whose run inside one column tile is longer than the loads a warp
issues up front, peaks with no entry in a row block, empty peaks, a row count that is not a multiple of the 512-row
block, several panels, and column slabs of one and of several tiles.  A pattern that no longer matches the counts of
the TF-IDF pass sends the panels to the atomic-cursor fill."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

import muon_b200 as mu
from muon_b200 import _device

pytestmark = pytest.mark.gpu

EMPTY_ROWS = (3, 600, 601, 4999)


def _edge_matrix(n, d, density, seed):
    rng = np.random.default_rng(seed)
    m = int(density * n * d)
    r, c = rng.integers(0, n, m), rng.integers(0, d, m)
    keep = ~np.isin(r, EMPTY_ROWS)
    keep &= ~((r < 512) & (c >= 5000) & (c < 5200))            # peaks without entries in row block 0 only
    keep &= ~((c >= 7000) & (c < 7010))                         # peaks without any entry
    r, c = r[keep], c[keep]
    long_rows = [(np.full(3000, 10), np.arange(3000)),          # 1024 entries in each of three column tiles
                 (np.full(d // 2, 700), np.arange(0, d, 2)),    # 512 entries in every tile
                 (np.full(d // 3, 1500), np.arange(0, d, 3))]
    r = np.concatenate([r] + [lr for lr, _ in long_rows])
    c = np.concatenate([c] + [lc for _, lc in long_rows])
    data = rng.integers(1, 6, r.size).astype(np.float32)
    C = sp.csr_matrix((data, (r, c)), shape=(n, d))
    C.sum_duplicates()
    C.sort_indices()
    return C


def _assert_panels_are_the_transpose(T, X):
    """T: TransposedPanels; X: host CSR with the values the panels were built from."""
    for a0, a1, P in T.panels:
        want = X[a0:a1].T.tocsr()
        want.sort_indices()
        assert np.array_equal(P.indptr.cpu().numpy(), want.indptr.astype(np.int64)), (a0, a1)
        pairs = P.pairs.cpu().numpy()
        assert np.array_equal(pairs[:, 0], want.indices), (a0, a1)
        assert np.array_equal(pairs[:, 1], want.data.astype(np.float32).view(np.int32)), (a0, a1)


@pytest.mark.parametrize("n, d, density, budget", [
    (5000, 30000, 0.02, 1 << 18),           # 1024 cells per panel -> 5 panels of 1-2 row blocks, one tile per slab
    (70000, 30000, 0.004, None),            # 2 panels of 69 row blocks, two tiles per slab
])
def test_tiled_fill_is_the_transpose(cuda, monkeypatch, n, d, density, budget):
    C = _edge_matrix(n, d, density, seed=n)
    got = _device.tfidf_csr(mu.DeviceCSR.from_scipy(C))
    assert "rb_counts" in got._aux
    X = sp.csr_matrix((got.data.cpu().numpy(), C.indices, C.indptr), shape=C.shape)
    if budget is not None:
        monkeypatch.setattr(_device.TransposedPanels, "L2_BUDGET", budget)
    T = _device.TransposedPanels(got, 64)
    assert T.counts_reused and T.tiled_fill and len(T.panels) >= 2
    _assert_panels_are_the_transpose(T, X)
    T2 = _device.TransposedPanels(got, 64)
    for (_, _, Pa), (_, _, Pb) in zip(T.panels, T2.panels):
        assert torch.equal(Pa.pairs, Pb.pairs)


def test_tiled_fill_falls_back_when_the_pattern_changed(cuda, monkeypatch):
    C = _edge_matrix(5000, 30000, 0.02, seed=11)
    got = _device.tfidf_csr(mu.DeviceCSR.from_scipy(C))
    monkeypatch.setattr(_device.TransposedPanels, "L2_BUDGET", 1 << 18)
    assert _device.TransposedPanels(got, 64).tiled_fill
    # (1) per-block counts moved between two blocks of one panel: the column totals still agree with t_indptr,
    # only the fill itself can see that block 0 holds a different number of entries
    rb = got._aux["rb_counts"]
    col = int(torch.nonzero(rb[0] > 0)[0])
    saved = rb.clone()
    rb[0, col] -= 1
    rb[1, col] += 1
    T = _device.TransposedPanels(got, 64)
    assert T.counts_reused and not T.tiled_fill
    rb.copy_(saved)
    # (2) one entry moved to the next (empty) column after the counts were taken; the row stays sorted
    idx = C.indices[C.indptr[20]:C.indptr[21]]
    p = int(np.nonzero(idx[:-1] + 1 < idx[1:])[0][0])
    got.indices[int(C.indptr[20]) + p] += 1
    T = _device.TransposedPanels(got, 64)
    assert T.counts_reused and not T.tiled_fill
    got.indices[int(C.indptr[20]) + p] -= 1
    T = _device.TransposedPanels(got, 64)
    assert T.tiled_fill
    X = sp.csr_matrix((got.data.cpu().numpy(), C.indices, C.indptr), shape=C.shape)
    _assert_panels_are_the_transpose(T, X)
