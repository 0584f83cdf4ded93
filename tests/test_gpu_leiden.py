"""H100: ``mu.tl.leiden`` / ``mu.tl.louvain`` -- the sweep and refinement kernels against their numpy restatement
(tests/leiden_ref.py), exact aggregation, the reference driver's fixture (tests/golden/leiden_small.npz), the
Leiden guarantees, quality against networkx and the sequential oracle, determinism and the container surface."""
import json
import os

import numpy as np
import pytest
import scipy.sparse as sp

import leiden_ref as R
import muon_b200 as mu
from conftest import GOLDEN, golden_csr
from muon_b200 import SimpleAnnData, SimpleMuData, _leiden

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def knn():
    z = np.load(os.path.join(GOLDEN, "umap_small.npz"))
    return golden_csr(z, "W").astype(np.float64)


@pytest.fixture(scope="module")
def small():
    z = np.load(os.path.join(GOLDEN, "leiden_small.npz"))
    return z, golden_csr(z, "A"), golden_csr(z, "B")


def _adata(W, key=None):
    ad = SimpleAnnData(np.zeros((W.shape[0], 1), np.float32))
    nk = key or "neighbors"
    ck = "connectivities" if key is None else f"{key}_connectivities"
    ad.obsp[ck] = W
    ad.uns[nk] = {"connectivities_key": ck, "params": {}}
    return ad


def _mudata(graphs, key=None):
    return SimpleMuData({name: _adata(G, key) for name, G in graphs.items()})


def _hub_graph():
    """A kNN-like graph plus one vertex linked to 600 vertices that sit in 600 different communities, so its row
    overflows the shared-memory table and goes through the hub launch."""
    rng = np.random.default_rng(4)
    n = 1200
    labels = np.repeat(np.arange(40), 30)
    A = R.random_graph(labels, 0.25, 0.002, 9).tolil()
    for u in rng.choice(np.arange(1, n), 600, replace=False):
        A[0, u] = A[u, 0] = 0.7
    return A.tocsr().astype(np.float64)


def _compare_sweep(P, comm, key):
    import torch
    lev = _leiden.Level.from_problem(P)
    got, moved, target, gain = lev.sweep(torch.from_numpy(comm.astype(np.int32)).cuda(), key)
    want, wmoved, wtarget, wgain = R.sweep_ref(P, comm, key)
    np.testing.assert_array_equal(target.cpu().numpy(), wtarget)
    np.testing.assert_allclose(gain.cpu().numpy(), wgain, rtol=1e-9, atol=0)
    np.testing.assert_array_equal(got.cpu().numpy(), want)
    assert moved == wmoved
    return want


def _compare_refine(P, refined, comm, key):
    import torch
    lev = _leiden.Level.from_problem(P)
    got, moved, pending, target, gain = lev.refine_round(torch.from_numpy(refined.astype(np.int32)).cuda(),
                                                         torch.from_numpy(comm.astype(np.int32)).cuda(), key)
    want, wmoved, wpending, wtarget, wgain = R.refine_round_ref(P, refined, comm, key)
    np.testing.assert_array_equal(target.cpu().numpy(), wtarget)
    np.testing.assert_allclose(gain.cpu().numpy(), wgain, rtol=1e-9, atol=0)
    np.testing.assert_array_equal(got.cpu().numpy(), want)
    assert (moved, pending) == (wmoved, wpending)
    return want


@pytest.mark.parametrize("graph", ["knn", "hub", "multiplex"])
def test_sweep_and_refinement_match_numpy(cuda, knn, graph):
    if graph == "knn":
        P = _leiden.Problem([knn], [1.0], [1.0])
    elif graph == "hub":
        P = _leiden.Problem([_hub_graph()], [1.0], [1.0])
        assert np.diff(P.indptr).max() > _leiden_max_shared_degree()
    else:
        _, A, B = R.multiplex_case()
        P = _leiden.Problem([_leiden.layer_matrix(A, False), _leiden.layer_matrix(B, True)], [1.0, 0.6], [2.5, 2.0])
    rng = np.random.default_rng(0)
    comm = np.arange(P.n)
    for step in range(6):                                   # singletons, then the states the sweeps reach
        comm = _compare_sweep(P, comm, _leiden.stream_key(11, 0, 0, 0, step))
    coarse = R.compact(rng.integers(0, 25, P.n))             # many distinct neighbour communities per row
    _compare_sweep(P, coarse, _leiden.stream_key(11, 0, 0, 1, 0))
    refined = np.arange(P.n)
    for r in range(4):
        refined = _compare_refine(P, refined, comm, _leiden.stream_key(11, 1, 0, 0, r))


def _leiden_max_shared_degree():
    from muon_b200 import _lib
    return _lib.load().mub_leiden_max_shared_degree()


def test_aggregation_is_exact(cuda, knn):
    import torch
    _, A, B = R.multiplex_case()
    layers = [_leiden.layer_matrix(A, True), _leiden.layer_matrix(B, True)]
    P = _leiden.Problem(layers, [1.0, 0.5], [1.0, 1.5])
    lev = _leiden.Level.from_problem(P)
    rng = np.random.default_rng(2)
    rid = R.compact(rng.integers(0, 97, P.n))
    agg = lev.aggregate(torch.from_numpy(rid.astype(np.int32)).cuda(), int(rid.max()) + 1)
    for _ in range(3):
        part = rng.integers(0, 7, agg.n)
        lifted = part[rid]
        q_agg = agg.quality(torch.from_numpy(part.astype(np.int32)).cuda())
        q_lift = lev.quality(torch.from_numpy(lifted.astype(np.int32)).cuda())
        assert q_agg == pytest.approx(q_lift, rel=1e-12)
        assert q_lift == pytest.approx(R.quality(lifted, layers, [1.0, 0.5], [1.0, 1.5]), rel=1e-9)


def test_reference_driver_fixture(cuda, small):
    z, A, B = small
    for alg, fn in (("leiden", mu.tl.leiden), ("louvain", mu.tl.louvain)):
        for name, kw in R.REFERENCE_CALLS.items():
            md = _mudata({"rna": A, "atac": B})
            assert fn(md, **kw) is None
            assert np.array_equal(np.asarray(md.obs[alg].astype(int)), z[f"{alg}_{name}_labels"]), (alg, name)
            assert list(md.obs[alg].cat.categories) == list(z[f"{alg}_{name}_categories"])
            want = json.loads(str(z[f"{alg}_{name}_params"]))
            got = md.uns[alg]["params"]
            assert set(got) == set(want)
            assert json.loads(json.dumps(got["resolution"])) == want["resolution"]
            assert got["random_state"] == want["random_state"]
            assert got["partition_improvement"] == pytest.approx(want["partition_improvement"], rel=1e-6)


def test_multiplex_matters(cuda):
    from sklearn.metrics import adjusted_rand_score
    labels, A, B = R.multiplex_case()
    md = _mudata({"a": A, "b": B})
    mu.tl.leiden(md, resolution=2.5, n_iterations=-1)
    lab = np.asarray(md.obs["leiden"].astype(int))
    assert adjusted_rand_score(lab, labels) >= 0.95
    for G in (A, B):
        single = _mudata({"a": G})
        mu.tl.leiden(single, resolution=2.5, n_iterations=-1)
        assert adjusted_rand_score(np.asarray(single.obs["leiden"].astype(int)), labels) <= 0.8
    C = R.Collapsed([_leiden.layer_matrix(G, False) for G in (A, B)], [1.0, 1.0], [2.5, 2.5])
    assert R.disconnected_communities(C.A, lab) == 0
    assert R.node_optimality_violations(C, lab, 1e-9 * C.A.sum()) == 0


@pytest.mark.parametrize("weighted", [True, False])
def test_guarantees_and_quality_on_knn(cuda, knn, weighted):
    A = knn.copy()
    if not weighted:
        A.data[:] = 1.0
    C = R.Collapsed([A], [1.0], [1.0])
    ad = _adata(knn)
    mu.tl.leiden(ad, use_weights=weighted)
    lab = np.asarray(ad.obs["leiden"].astype(int))
    assert R.disconnected_communities(A, lab) == 0
    assert R.node_optimality_violations(C, lab, 1e-9 * A.sum()) == 0
    q = R.quality(lab, [A], [1.0], [1.0])
    import networkx as nx
    G = nx.from_scipy_sparse_array(A)
    q_nx = []
    for s in range(5):
        part = np.empty(A.shape[0], dtype=np.int64)
        for i, p in enumerate(nx.community.louvain_communities(G, weight="weight", seed=s)):
            part[list(p)] = i
        q_nx.append(R.quality(part, [A], [1.0], [1.0]))
    q_seq = R.quality(R.sequential(C, refine=True, n_iterations=-1, seed=0), [A], [1.0], [1.0])
    print(f"GPU {q / A.sum():.4f}, sequential {q_seq / A.sum():.4f}, networkx min {min(q_nx) / A.sum():.4f}")
    assert q >= min(q_nx) - 0.005 * abs(min(q_nx))
    assert q >= q_seq - 0.005 * abs(q_seq)
    # Louvain: node optimality only
    ad = _adata(knn)
    mu.tl.louvain(ad, use_weights=weighted)
    assert R.node_optimality_violations(C, np.asarray(ad.obs["louvain"].astype(int)), 1e-9 * A.sum()) == 0


def test_partition_improvement_and_directed(cuda):
    _, A, B = R.multiplex_case()
    weights, gammas = [1.0, 0.7], [2.0, 2.5]
    for directed in (True, False):
        md = _mudata({"a": A, "b": B})
        mu.tl.leiden(md, resolution=gammas, mod_weights=weights, directed=directed,
                     partition_kwargs={"weights": "weight"})
        lab = np.asarray(md.obs["leiden"].astype(int))
        layers = [sp.csr_matrix(G, dtype=np.float64) for G in (A, B)]
        want = (R.quality(lab, layers, weights, gammas, directed)
                - R.quality(np.arange(A.shape[0]), layers, weights, gammas, directed))
        assert md.uns["leiden"]["params"]["partition_improvement"] == pytest.approx(want, rel=1e-6)


def test_deterministic(cuda, knn):
    runs = []
    for rs in (5, 5, 6):
        ad = _adata(knn)
        mu.tl.leiden(ad, random_state=rs)
        runs.append(np.asarray(ad.obs["leiden"].astype(int)))
    assert np.array_equal(runs[0], runs[1])
    # another seed: another order of moves, still a connected, node-optimal partition
    C = R.Collapsed([knn], [1.0], [1.0])
    assert R.disconnected_communities(knn, runs[2]) == 0
    assert R.node_optimality_violations(C, runs[2], 1e-9 * knn.sum()) == 0


def test_200k_cells_deterministic(cuda):
    import torch

    from muon_b200 import _device
    from muon_b200.pp import _umap_connectivities
    N, k = 200_000, 15
    rng = np.random.default_rng(0)
    c = rng.integers(0, 30, N)
    X = rng.normal(size=(N, 20)).astype(np.float32) + 4.0 * rng.normal(size=(30, 20)).astype(np.float32)[c]
    idx, dist = _device.knn_l2(torch.from_numpy(X).cuda(), k)
    W = _umap_connectivities(idx.to(torch.int64), dist, N)
    outs = []
    for alg in ("leiden", "leiden", "louvain", "louvain"):
        ad = _adata(W)
        getattr(mu.tl, alg)(ad, random_state=1)
        outs.append(np.asarray(ad.obs[alg].astype(int)))
    assert np.array_equal(outs[0], outs[1]) and np.array_equal(outs[2], outs[3])
    assert outs[0].max() >= 1


def test_surface(cuda, small):
    z, A, B = small
    n = A.shape[0]
    planted = R.renumber_by_size(z["planted"])
    # AnnData: scanpy's slots and defaults
    ad = _adata(A)
    assert mu.tl.leiden(ad) is None
    assert np.array_equal(np.asarray(ad.obs["leiden"].astype(int)), planted)
    assert ad.uns["leiden"] == {"params": {"resolution": None, "random_state": 0, "n_iterations": -1}}
    ad = _adata(A, key="wnn")
    mu.tl.leiden(ad, neighbors_key="wnn", key_added="cl", resolution=0.9, n_iterations=2, use_weights=False)
    assert ad.uns["cl"]["params"] == {"resolution": 0.9, "random_state": 0, "n_iterations": 2}
    assert list(ad.obs["cl"].cat.categories) == [str(i) for i in range(4)]
    ad = _adata(A)
    out = mu.tl.louvain(ad, copy=True, random_state=3)
    assert "louvain" not in ad.uns and out.uns["louvain"] == {"params": {"resolution": None, "random_state": 3}}
    # MuData: scalar, list and dict resolution / mod_weights, neighbors_key, key_added, n_iterations
    for kw in ({"resolution": 1.0}, {"resolution": [1.0, 0.9]}, {"resolution": {"rna": 1.1, "atac": 0.9}},
               {"mod_weights": 2.0}, {"mod_weights": [1.0, 0.3]}, {"mod_weights": {"rna": 0.5}},
               {"partition_kwargs": {"weights": "weight", "resolution_parameter": 0.9}},
               {"n_iterations": 1}, {"n_iterations": 0}, {"directed": False}):
        md = _mudata({"rna": A, "atac": B}, key="wnn")
        mu.tl.leiden(md, neighbors_key="wnn", key_added="clusters", **kw)
        got = np.asarray(md.obs["clusters"].astype(int))
        if kw.get("n_iterations") == 0:
            assert np.unique(got).size == n and md.uns["leiden"]["params"]["partition_improvement"] == 0.0
        else:
            assert np.array_equal(got, planted), kw
        assert set(md.uns["leiden"]["params"]) == {"resolution", "random_state", "partition_improvement"}
    with pytest.raises(KeyError):
        mu.tl.leiden(_mudata({"rna": A, "atac": B}), neighbors_key="wnn")
    with pytest.raises(ValueError):
        mu.tl.leiden(_mudata({"rna": A, "atac": sp.csr_matrix((n, n), dtype=np.float32)}))
    with pytest.raises(NotImplementedError):
        mu.tl.louvain(_mudata({"rna": A, "atac": sp.csr_matrix(np.triu(B.toarray()))}))
    with pytest.raises(TypeError):
        mu.tl.louvain(_mudata({"rna": A, "atac": B}), n_iterations=3)
