"""CPU: the UMAP oracle (oracle/umap_ref.py) -- Philox, the closed-form schedule, the Jacobi epoch against a vertex
loop, the sequential layout on planted clusters -- and the host side of ``mu.tl.umap``: its signature, the
preparation it shares with umap-learn, and the errors it raises before any device work."""
import inspect
import json
import os
from fractions import Fraction

import numpy as np
import pytest
import scipy.sparse as sp

import muon_b200 as mu
from conftest import GOLDEN
from muon_b200 import SimpleAnnData, SimpleMuData
from muon_b200 import _umap
from oracle import umap_ref as R


def test_signature_matches_reference():
    ref = json.load(open(os.path.join(GOLDEN, "umap_signature.json")))["umap"]
    sig = inspect.signature(_umap.umap)
    pos = [p for p in sig.parameters.values() if p.kind == p.POSITIONAL_OR_KEYWORD]
    assert [p.name for p in pos] == ref["params"]
    for i, (p, d) in enumerate(zip(pos, ref["defaults"])):
        if i < ref["required"]:
            assert p.default is inspect.Parameter.empty
        else:
            assert repr(p.default) == d, (p.name, p.default, d)
    assert all(p.kind == p.KEYWORD_ONLY for p in sig.parameters.values() if p.kind != p.POSITIONAL_OR_KEYWORD)


@pytest.mark.parametrize("spread,min_dist", [(1.0, 0.5), (1.0, 0.1), (2.0, 0.3)])
def test_find_ab_is_a_direct_curve_fit(spread, min_dist):
    from scipy.optimize import curve_fit
    x = np.linspace(0, 3 * spread, 300)
    y = np.where(x < min_dist, 1.0, np.exp(-(x - min_dist) / spread))
    (a, b), _ = curve_fit(lambda x, a, b: 1.0 / (1.0 + a * x ** (2 * b)), x, y)
    assert R.find_ab(spread, min_dist) == (a, b)
    assert _umap.find_ab_params(spread, min_dist) == (a, b)


def test_philox_known_answers():
    # Random123 kat_vectors for philox4x32_10
    M = 0xFFFFFFFF
    cases = [((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
             ((M, M, M, M), (M, M), (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
             ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
              (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1))]
    for ctr, key, want in cases:
        got = R.philox4x32_10(*[[c] for c in ctr], *key)
        assert tuple(int(g[0]) for g in got) == want


def test_closed_form_schedule_is_umaps_counters_in_exact_arithmetic():
    rng = np.random.default_rng(0)
    eps = np.concatenate([[1.0, 1.5, 2.0, 3.0, 7.25], rng.uniform(1, 40, 200)]).astype(np.float32)
    rate, n_epochs = 5, 200
    for e, ef in enumerate(eps):
        E = Fraction(float(ef))
        nxt, eneg = E, E / rate
        nxt_neg = eneg
        for ep in range(n_epochs):
            hit, n_neg = R.schedule(ep, eps[e:e + 1], rate)
            if nxt <= ep:
                k = int((ep - nxt_neg) / eneg)          # umap: int() of the counter quotient (>= 0 here)
                assert hit[0] and n_neg[0] == k, (e, ep)
                nxt += E
                nxt_neg += k * eneg
            else:
                assert not hit[0], (e, ep)


def _graph(n, seed, k=6):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, 3))
    D = ((X[:, None] - X[None]) ** 2).sum(-1)
    np.fill_diagonal(D, np.inf)
    nn = np.argsort(D, axis=1)[:, :k]
    W = sp.csr_matrix((rng.uniform(0.05, 1.0, n * k).astype(np.float32), nn.ravel(), np.arange(0, n * k + 1, k)),
                      shape=(n, n))
    W = W.maximum(W.T).tocsr()                                    # symmetric pattern, asymmetric weights ok too
    W.data *= rng.uniform(0.5, 1.0, W.nnz).astype(np.float32)
    W.sort_indices()
    return W


@pytest.mark.parametrize("dim", [2, 3])
def test_epoch_ref_equals_vertex_loop(dim):
    W = _graph(50, dim)
    G = R.prune(W, 20)
    eps = R.epochs_per_sample(G.data)
    rs = np.random.RandomState(1)
    Y = R.init_ref(G, dim, "random", rs)
    Y[7] = Y[8]                                     # coincident vertices: the d^2 = 0 repulsion rule
    key = R.sampler_key(rs)
    a, b = R.find_ab(1.0, 0.5)
    for ep in range(1, 8):
        got = R.epoch_ref(G, eps, Y, ep, 20, a, b, 1.0, 1.0, 5, key)
        want = R.epoch_loop(G, eps, Y, ep, 20, a, b, 1.0, 1.0, 5, key)
        np.testing.assert_allclose(got, want, rtol=0, atol=2e-5)
        Y = got


def test_layout_ref_separates_planted_clusters():
    X, labels, W = R.planted_graph(n=400, n_clusters=4, spread=3.0, seed=3)
    Y = R.layout_ref(W, maxiter=200)
    assert Y.shape == (400, 2) and np.isfinite(Y).all()
    assert R.knn_label_agreement(Y, labels) > 0.95
    assert R.trustworthiness(X, Y) > 0.9


def test_fixture_scores_are_the_fixture_layouts():
    z = np.load(os.path.join(GOLDEN, "umap_small.npz"))
    assert float(z["trust_ref"]) == pytest.approx(R.trustworthiness(z["rep"], z["layout_ref"]), abs=1e-12)
    assert float(z["label_ref"]) == pytest.approx(R.knn_label_agreement(z["layout_ref"], z["labels"]), abs=1e-12)
    assert float(z["label_ref"]) > 0.95


def test_trustworthiness_matches_sklearn():
    manifold = pytest.importorskip("sklearn.manifold")
    rng = np.random.default_rng(0)
    X = rng.normal(size=(300, 8))
    Y = X[:, :2] + 0.3 * rng.normal(size=(300, 2))
    assert R.trustworthiness(X, Y, 15) == pytest.approx(manifold.trustworthiness(X, Y, n_neighbors=15), abs=1e-12)


@pytest.mark.parametrize("maxiter", [None, 0, 5, 50])
def test_host_preparation_matches_oracle(maxiter):
    W = _graph(80, 0)
    G, n_epochs = _umap.prune(W, 0 if maxiter is None else maxiter)
    assert n_epochs == R.n_epochs_for(80, maxiter)
    G2 = R.prune(W, n_epochs)
    for f in ("indptr", "indices", "data"):
        np.testing.assert_array_equal(getattr(G, f), getattr(G2, f))
    np.testing.assert_array_equal(_umap.epochs_per_sample(G.data), R.epochs_per_sample(G2.data))
    assert (_umap.epochs_per_sample(G.data) >= 1).all()
    rs1, rs2 = np.random.RandomState(5), np.random.RandomState(5)
    np.testing.assert_array_equal(_umap.initial_positions(G, 2, "random", rs1, None), R.init_ref(G2, 2, "random", rs2))
    assert _umap.sampler_key(rs1) == R.sampler_key(rs2)


def test_small_components_and_meta_positions_follow_umap():
    """Two components, one of 3 vertices (too small for an eigenproblem at dim 2): the small one is drawn uniform
    around its meta position, the other uses the eigenvectors it is given."""
    big = _graph(30, 1)
    small = sp.csr_matrix(np.array([[0, 1, 1], [1, 0, 1], [1, 1, 0]], dtype=np.float32))
    G = sp.block_diag([big, small]).tocsr()
    fake = lambda W, dim: np.linspace(-1, 1, W.shape[0] * dim).reshape(W.shape[0], dim)  # noqa: E731
    Y = _umap.spectral_layout(G, 2, np.random.RandomState(0), fake)
    np.testing.assert_allclose(Y[:30], fake(big, 2) * 1.0 + [1.0, 0.0])
    u = np.random.RandomState(0).uniform(low=-1.0, high=1.0, size=(3, 2)) + [-1.0, 0.0]
    np.testing.assert_allclose(Y[30:], u)


def _adata_with_graph(W, key="neighbors"):
    ad = SimpleAnnData(np.zeros((W.shape[0], 1), np.float32))
    ck = "connectivities" if key == "neighbors" else f"{key}_connectivities"
    ad.obsp[ck] = W
    ad.uns[key] = {"connectivities_key": ck, "params": {}}
    return ad


def test_errors_before_device_work(monkeypatch):
    def no_device(*a, **k):
        raise AssertionError("reached the device")

    monkeypatch.setattr(_umap, "Layout", no_device)
    monkeypatch.setattr(_umap, "spectral_vectors", no_device)
    W = _graph(40, 2)
    with pytest.raises(TypeError):
        mu.tl.umap(np.zeros((3, 3)))
    with pytest.raises(ValueError, match="Did not find"):
        mu.tl.umap(SimpleAnnData(np.zeros((4, 2))))
    with pytest.raises(ValueError, match="Did not find"):
        mu.tl.umap(SimpleMuData({"a": _adata_with_graph(W)}))
    with pytest.raises(ValueError, match="Did not find"):
        mu.tl.umap(_adata_with_graph(W), neighbors_key="wnn")
    with pytest.raises(NotImplementedError):
        mu.tl.umap(_adata_with_graph(W), n_components=17)
    with pytest.raises(ValueError):
        mu.tl.umap(_adata_with_graph(W), method="cuml")
    with pytest.raises(ValueError):
        mu.tl.umap(_adata_with_graph(W), init_pos=np.zeros((40, 3)))
    five = sp.block_diag([_graph(20, s) for s in range(5)]).tocsr()
    with pytest.raises(NotImplementedError, match="init_pos='random'"):
        mu.tl.umap(_adata_with_graph(five))
