"""H100: ``mu.tl.snf`` -- the unmodified reference's outputs (tests/golden/snf_small.npz), the float64 restatement
(oracle/snf_ref.py) on sparse kNN distances, bit-identical repeats and bit-symmetric states, the slots and keys,
every refusal, and one 30 000-cell run within the stated memory budget."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

import muon_b200 as mu
from muon_b200 import SimpleAnnData, SimpleMuData
from muon_b200 import _device, _snf
from oracle import snf_ref as R
from test_oracle_snf import assert_same_rows, golden_cases

pytestmark = pytest.mark.gpu


def _mdata(dists, key="neighbors", use_rep=None):
    mods = {}
    for m, d in enumerate(dists):
        a = SimpleAnnData(np.zeros((d.shape[0], 1)))
        a.obsp["distances"] = d
        params = {"n_neighbors": 15} if use_rep is None else {"n_neighbors": 15, "use_rep": use_rep, "n_pcs": 10}
        a.uns[key] = {"params": params, "distances_key": "distances", "connectivities_key": "connectivities"}
        mods[f"m{m}"] = a
    return SimpleMuData(mods)


def _max_rel(a, b):
    a, b = np.asarray(a), np.asarray(b)
    assert np.array_equal(a == 0, b == 0)
    nz = b != 0
    return float(np.max(np.abs(a[nz] - b[nz]) / np.abs(b[nz]))) if nz.any() else 0.0


@pytest.fixture(scope="module")
def sparse4k():
    dists, labels = R.planted_distances(4000, 3, k_graph=15, seed=11)
    return dists, labels


@pytest.mark.parametrize("case", range(5))
def test_reference_golden(cuda, case):
    params, dists, ref = golden_cases()[case]
    md = _mdata(dists)
    mu.tl.snf(md, **params)
    k = params["n_neighbors"]
    for key in ("distances", "connectivities"):
        got = md.obsp[key]
        assert isinstance(got, sp.csr_array) and got.dtype == np.float64
        assert np.array_equal(np.diff(got.indptr), np.full(got.shape[0], k))
        assert np.all(np.diff(got.data.reshape(-1, k), axis=1) >= 0)
        assert_same_rows(got, ref[key], rtol=1e-10)
    assert md.uns["neighbors"]["params"]["method"] == "snf"


@pytest.mark.parametrize("iters", [1, 20])
def test_restatement_sparse(cuda, sparse4k, iters):
    dists, _ = sparse4k
    got = _snf.fuse(dists, n_neighbors=20, n_iterations=iters, return_dense=True)
    ref = R.snf_ref(dists, n_neighbors=20, n_iterations=iters)
    assert _max_rel(got["w"].cpu().numpy(), ref["w"]) <= 1e-10
    for key in ("distances", "connectivities"):
        assert_same_rows(got[key], ref[key], rtol=1e-10)


def test_deterministic_and_bit_symmetric(cuda, sparse4k):
    dists, labels = sparse4k
    a = _snf.fuse(dists, n_neighbors=20, n_iterations=4, return_dense=True, return_modalities=True)
    a = {"w": a["w"].cpu().numpy(), "modalities": [x.cpu().numpy() for x in a["modalities"]],
         "distances": a["distances"], "connectivities": a["connectivities"]}
    b = _snf.fuse(dists, n_neighbors=20, n_iterations=4, return_dense=True, return_modalities=True)
    assert np.array_equal(a["w"], b["w"].cpu().numpy())
    for x, y in zip(a["modalities"], b["modalities"]):
        y = y.cpu().numpy()
        assert np.array_equal(x, y)
        assert np.array_equal(x, x.T)
        assert np.all(np.diag(x) == 0.5)
    assert np.array_equal(a["w"], a["w"].T)
    for key in ("distances", "connectivities"):
        assert np.array_equal(a[key].indices, b[key].indices) and np.array_equal(a[key].data, b[key].data)
    D = a["distances"]
    rows = np.repeat(np.arange(D.shape[0]), np.diff(D.indptr))
    assert np.mean(labels[rows] == labels[D.indices]) >= 0.95


def test_slots_and_keys(cuda):
    dists, _ = R.planted_distances(230, 3, k_graph=12, seed=2)
    md = _mdata(dists, use_rep="X_pca")
    assert mu.tl.snf(md, n_neighbors=10, key_added="fused") is None
    assert set(md.obsp) == {"fused_connectivities", "fused_distances"}
    u = md.uns["fused"]
    assert u["connectivities_key"] == "fused_connectivities" and u["distances_key"] == "fused_distances"
    assert u["params"] == {"n_neighbors": 10, "eps": np.finfo(np.float64).eps, "use_rep": dict.fromkeys(md.mod, "X_pca"),
                           "n_pcs": dict.fromkeys(md.mod, 10), "method": "snf"}
    ref = _snf.fuse(dists, n_neighbors=10)

    md2 = _mdata(dists, key="nn")
    out = mu.tl.snf(md2, n_neighbors=10, neighbor_keys="nn", copy=True)
    assert out is not md2 and "connectivities" not in md2.obsp
    assert np.array_equal(out.obsp["connectivities"].data, ref["connectivities"].data)
    assert np.array_equal(out.obsp["distances"].indices, ref["distances"].indices)
    assert out.uns["neighbors"]["params"]["use_rep"] == dict.fromkeys(md.mod, -1)

    # a dict selects its modalities: the third one is not fused
    md3 = _mdata(dists)
    mu.tl.snf(md3, n_neighbors=10, neighbor_keys={"m0": "neighbors", "m2": "neighbors"})
    sub = _snf.fuse([dists[0], dists[2]], n_neighbors=10)
    assert np.array_equal(md3.obsp["distances"].data, sub["distances"].data)
    assert set(md3.uns["neighbors"]["params"]["use_rep"]) == {"m0", "m2"}


def test_refusals(cuda, monkeypatch):
    dists, _ = R.planted_distances(300, 2, k_graph=10, seed=4)
    before = torch.cuda.memory_allocated()
    with pytest.raises(ValueError, match="seems to be too high"):
        mu.tl.snf(_mdata(dists), n_neighbors=300)
    with pytest.raises(NotImplementedError, match="255"):
        mu.tl.snf(_mdata(dists), n_neighbors=256)
    with pytest.raises(ValueError, match="at least two"):
        mu.tl.snf(_mdata(dists), neighbor_keys={"m1": "neighbors"})
    with pytest.raises(ValueError, match="Did not find"):
        mu.tl.snf(_mdata(dists), neighbor_keys="other")
    with pytest.raises(ValueError, match="same observations"):
        mu.tl.snf(_mdata([dists[0], dists[1][:200, :200]]), n_neighbors=5)
    with pytest.raises(NotImplementedError, match="16"):
        mu.tl.snf(_mdata(dists * 9), n_neighbors=5)
    monkeypatch.setattr(_snf, "free_device_bytes", lambda: _snf.state_bytes(300, 2, 20) - 1)
    with pytest.raises(NotImplementedError, match="device memory"):
        mu.tl.snf(_mdata(dists), n_neighbors=20)
    assert torch.cuda.memory_allocated() == before


def test_30k_cells_within_budget(cuda):
    n, k, m = 30000, 20, 2
    rng = np.random.default_rng(0)
    c = rng.integers(0, 20, n)
    dists = []
    for d in (30, 20):
        X = rng.normal(size=(n, d)).astype(np.float32) + 3.0 * rng.normal(size=(20, d)).astype(np.float32)[c]
        idx, dist = _device.knn_l2(torch.from_numpy(X).cuda(), 16)
        dists.append(sp.csr_matrix((dist[:, 1:].cpu().numpy().ravel().astype(np.float64),
                                    idx[:, 1:].cpu().numpy().ravel().astype(np.int64),
                                    np.arange(0, n * 15 + 1, 15)), shape=(n, n)))
        del idx, dist
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = _snf.fuse(dists, n_neighbors=k, return_dense=True, return_modalities=True)
    peak = torch.cuda.max_memory_allocated() - base
    assert peak <= (2 * m + 2) * n * n * 8 + 64 * n * (k + 1) * (m + 2)
    w = out["w"]
    assert bool(torch.isfinite(w).all())
    assert bool((w == w.T).all())
    assert bool((torch.diagonal(w) == 0.5).all())
    for x in out["modalities"]:
        assert bool((x == x.T).all()) and bool((torch.diagonal(x) == 0.5).all())
    for key in ("distances", "connectivities"):
        A = out[key]
        assert A.shape == (n, n) and np.array_equal(np.diff(A.indptr), np.full(n, k))
        assert np.all(np.isfinite(A.data)) and np.all(np.diff(A.data.reshape(-1, k), axis=1) >= 0)
    D = out["distances"]
    rows = np.repeat(np.arange(n), k)
    assert not np.any(rows == D.indices)
    assert np.mean(c[rows] == c[D.indices]) >= 0.95
