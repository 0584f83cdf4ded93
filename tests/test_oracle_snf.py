"""CPU: the SNF restatement (oracle/snf_ref.py) against the unmodified reference's outputs
(tests/golden/snf_small.npz), the sparse-distance rule, and the host side of ``mu.tl.snf``: its signature and the
errors it raises before any device work."""
import inspect
import json
import os

import numpy as np
import pytest
import scipy.sparse as sp
from scipy.spatial.distance import cdist

import muon_b200 as mu
from conftest import GOLDEN, load_golden
from muon_b200 import SimpleAnnData, SimpleMuData
from muon_b200 import _snf
from oracle import snf_ref as R


def golden_cases():
    z = load_golden("snf_small.npz")
    out = []
    for c in range(int(z["n_cases"])):
        coords = []
        while f"c{c}_X{len(coords)}" in z:
            coords.append(z[f"c{c}_X{len(coords)}"])
        k, iters, sigma = z[f"c{c}_params"]
        ref = {}
        for key in ("distances", "connectivities"):
            ref[key] = sp.csr_array((z[f"c{c}_{key}_data"], z[f"c{c}_{key}_indices"], z[f"c{c}_{key}_indptr"]),
                                    shape=tuple(z[f"c{c}_{key}_shape"]))
        out.append(({"n_neighbors": int(k), "n_iterations": int(iters), "sigma": float(sigma)},
                    [cdist(X, X) for X in coords], ref))
    return out


def assert_same_rows(got, ref, rtol):
    """Same neighbour set per row, and the values (taken in each row's ascending column order) within rtol."""
    got, ref = sp.csr_array(got), sp.csr_array(ref)
    assert got.shape == ref.shape
    assert np.array_equal(np.diff(got.indptr), np.diff(ref.indptr))
    for i in range(got.shape[0]):
        a, b = slice(got.indptr[i], got.indptr[i + 1]), slice(ref.indptr[i], ref.indptr[i + 1])
        ga, ra = np.argsort(got.indices[a]), np.argsort(ref.indices[b])
        assert np.array_equal(got.indices[a][ga], ref.indices[b][ra]), i
        np.testing.assert_allclose(got.data[a][ga], ref.data[b][ra], rtol=rtol, atol=0)


def test_signature_matches_reference():
    ref = json.load(open(os.path.join(GOLDEN, "snf_signature.json")))["snf"]
    sig = inspect.signature(_snf.snf)
    pos = [p for p in sig.parameters.values() if p.kind == p.POSITIONAL_OR_KEYWORD]
    assert [p.name for p in pos] == ref["params"]
    for i, (p, d) in enumerate(zip(pos, ref["defaults"])):
        if i < ref["required"]:
            assert p.default is inspect.Parameter.empty
        else:
            assert repr(p.default) == d, (p.name, p.default, d)
    assert all(p.kind == p.KEYWORD_ONLY for p in sig.parameters.values() if p.kind != p.POSITIONAL_OR_KEYWORD)
    assert mu.tl.snf.__doc__ and callable(mu.tl.snf)


@pytest.mark.parametrize("case", range(5))
def test_restatement_reproduces_reference(case):
    params, dists, ref = golden_cases()[case]
    got = R.snf_ref(dists, **params)
    for key in ("distances", "connectivities"):
        assert isinstance(got[key], sp.csr_array) and got[key].dtype == np.float64
        assert_same_rows(got[key], ref[key], rtol=1e-12)
        # ascending value order within each row, as the reference writes it
        d = got[key].data.reshape(-1, params["n_neighbors"])
        assert np.all(np.diff(d, axis=1) >= 0)


def test_complete_sparse_equals_dense():
    dists, _ = R.planted_distances(157, 2, seed=3)
    dense = R.snf_ref(dists, n_neighbors=7, n_iterations=5)
    complete = R.snf_ref([sp.csr_matrix(d) for d in dists], n_neighbors=7, n_iterations=5)
    for d in dists:
        assert sp.csr_matrix(d).nnz == d.size - d.shape[0]      # every off-diagonal pair is stored
    np.testing.assert_array_equal(dense["w"], complete["w"])
    for key in ("distances", "connectivities"):
        assert_same_rows(dense[key], complete[key], rtol=0)


def test_sparse_rule():
    # one-way edge -> d / 2, unstored -> +inf, stored zero -> dropped like scipy's eliminate_zeros, diagonal 0
    D = sp.csr_matrix(np.array([[0.0, 2.0, 0.0], [0.0, 5.0, 0.0], [1.0, 0.0, 0.0]]))
    F = R.symmetrised(D)
    expect = np.array([[0.0, 1.0, 0.5], [1.0, 0.0, np.inf], [0.5, np.inf, 0.0]])
    np.testing.assert_array_equal(F, expect)
    W = R.affinity(F, 1, 0.5)
    assert W[1, 2] == 0.0 and W[2, 1] == 0.0 and np.all(W[np.isfinite(F)] > 0)


def test_knn_sparse_planted_clusters():
    dists, labels = R.planted_distances(600, 2, k_graph=15, seed=5)
    out = R.snf_ref(dists, n_neighbors=20)
    D = out["distances"]
    rows = np.repeat(np.arange(D.shape[0]), np.diff(D.indptr))
    assert np.mean(labels[rows] == labels[D.indices]) >= 0.95
    assert not np.any(rows == D.indices)


def _mdata(n=40, n_mod=2, key="neighbors", sparse=True):
    dists, _ = R.planted_distances(n, n_mod, k_graph=8 if sparse else None, seed=1)
    mods = {}
    for m, d in enumerate(dists):
        a = SimpleAnnData(np.zeros((n, 1)))
        a.obsp["distances"] = d
        a.uns[key] = {"params": {"n_neighbors": 8}, "distances_key": "distances"}
        mods[f"m{m}"] = a
    return SimpleMuData(mods)


def test_refusals_before_device_work(monkeypatch):
    def no_device(*a, **k):
        raise AssertionError("device work before validation")
    monkeypatch.setattr(_snf, "free_device_bytes", lambda: 1 << 50)
    monkeypatch.setattr(_snf, "_upload_distances", no_device)
    with pytest.raises(ValueError, match="seems to be too high"):
        mu.tl.snf(_mdata(), n_neighbors=40)
    with pytest.raises(NotImplementedError, match="255"):
        mu.tl.snf(_mdata(n=300), n_neighbors=256)
    with pytest.raises(ValueError, match="at least two"):
        mu.tl.snf(_mdata(), neighbor_keys={"m0": "neighbors"})
    with pytest.raises(ValueError, match=r'Did not find \.uns\["nn"\] for modality "m0"'):
        mu.tl.snf(_mdata(), neighbor_keys="nn")
    md = _mdata(n_mod=17)
    with pytest.raises(NotImplementedError, match="16"):
        mu.tl.snf(md, n_neighbors=5)
    md = _mdata()
    b = SimpleAnnData(np.zeros((39, 1)))
    b.obsp["distances"] = sp.csr_matrix((39, 39))
    b.uns["neighbors"] = {"params": {}, "distances_key": "distances"}
    md.mod["m1"] = b
    with pytest.raises(ValueError, match="same observations"):
        mu.tl.snf(md, n_neighbors=5)
    monkeypatch.setattr(_snf, "free_device_bytes", lambda: 5 * 40 * 40 * 8)
    with pytest.raises(NotImplementedError, match="device memory"):
        mu.tl.snf(_mdata(), n_neighbors=5)


def test_state_bytes_within_budget():
    for n, m, k in [(30000, 2, 20), (4000, 3, 255), (1000, 16, 5)]:
        assert _snf.state_bytes(n, m, k) <= (2 * m + 2) * n * n * 8 + 64 * n * (k + 1) * (m + 2)
