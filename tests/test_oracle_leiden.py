"""CPU: the clustering oracle (tests/leiden_ref.py) -- quality against networkx, brute-force gains, the sequential
optimiser on planted and kNN graphs, the numpy restatement of the device sweep -- the reference driver with its
stand-ins against tests/golden/leiden_small.npz, and the host side of ``mu.tl.leiden`` / ``mu.tl.louvain``."""
import inspect
import json
import os

import numpy as np
import pytest
import scipy.sparse as sp

import leiden_ref as R
import muon_b200 as mu
from conftest import GOLDEN, golden_csr
from muon_b200 import SimpleAnnData, SimpleMuData, _leiden

nx = pytest.importorskip("networkx")


@pytest.fixture(scope="module")
def knn():
    z = np.load(os.path.join(GOLDEN, "umap_small.npz"))
    return golden_csr(z, "W").astype(np.float64)


def _nx_louvain_quality(W, weighted, seeds=range(5)):
    A = W.copy()
    if not weighted:
        A.data[:] = 1.0
    G = nx.from_scipy_sparse_array(A)
    qs = []
    for s in seeds:
        parts = nx.community.louvain_communities(G, weight="weight", seed=s)
        lab = np.empty(A.shape[0], dtype=np.int64)
        for i, p in enumerate(parts):
            lab[list(p)] = i
        qs.append(R.quality(lab, [A], [1.0], [1.0]))
    return A, min(qs)


@pytest.mark.parametrize("gamma", [0.5, 1.0, 2.0])
def test_quality_is_scaled_networkx_modularity(gamma):
    labels, A, _ = R.small_case()
    A = A.astype(np.float64)
    rng = np.random.default_rng(0)
    lab = np.where(rng.random(labels.size) < 0.2, rng.integers(0, 6, labels.size), labels)
    G = nx.from_scipy_sparse_array(A)
    comms = [set(np.nonzero(lab == c)[0]) for c in np.unique(lab)]
    want = A.sum() * nx.community.modularity(G, comms, resolution=gamma)
    assert R.quality(lab, [A], [1.0], [gamma]) == pytest.approx(want, rel=1e-9)
    perm = rng.permutation(10)
    assert R.quality(perm[lab], [A], [1.0], [gamma]) == pytest.approx(want, rel=1e-12)
    assert R.quality(lab, [A], [1.0], [gamma], directed=False) == pytest.approx(2 * want, rel=1e-12)


def test_brute_force_gains_equal_quality_differences():
    labels, A, B = R.small_case()
    C = R.Collapsed([A, B], [1.0, 0.7], [1.0, 1.3])
    rng = np.random.default_rng(1)
    lab = rng.integers(0, 6, labels.size)
    for v in rng.choice(labels.size, 40, replace=False):
        for b in (0, 3, 5, 99):
            after = lab.copy()
            after[v] = b
            want = R.quality(after, [A, B], [1.0, 0.7], [1.0, 1.3]) - R.quality(lab, [A, B], [1.0, 0.7], [1.0, 1.3])
            assert R.move_gain(C, lab, v, b) == pytest.approx(want, rel=1e-9, abs=1e-9)
            assert C.quality(after) - C.quality(lab) == pytest.approx(want, rel=1e-9, abs=1e-9)


def test_sequential_separates_planted_clusters():
    from sklearn.metrics import adjusted_rand_score
    labels, A, B = R.small_case()
    C = R.Collapsed([A, B], [1.0, 1.0], [1.0, 1.0])
    for refine in (True, False):
        lab = R.sequential(C, refine=refine, n_iterations=-1, seed=0)
        assert adjusted_rand_score(lab, labels) == 1.0
        assert R.disconnected_communities(C.A, lab) == 0


@pytest.mark.parametrize("weighted", [True, False])
def test_sequential_quality_on_knn_graph(knn, weighted):
    A, q_nx = _nx_louvain_quality(knn, weighted)
    C = R.Collapsed([A], [1.0], [1.0])
    lab = R.sequential(C, refine=True, n_iterations=-1, seed=0)
    q = R.quality(lab, [A], [1.0], [1.0])
    print(f"sequential {q / A.sum():.4f}, networkx louvain min over 5 seeds {q_nx / A.sum():.4f} (modularity)")
    assert q >= q_nx - 0.005 * abs(q_nx)
    assert R.disconnected_communities(A, lab) == 0
    assert R.node_optimality_violations(C, lab, 1e-9 * A.sum()) == 0


def test_device_sweep_restatement_raises_quality_and_ends_node_optimal(knn):
    P = _leiden.Problem([knn], [1.0], [1.0])
    C = R.Collapsed([knn], [1.0], [1.0])
    comm = np.arange(P.n)
    q = C.quality(comm)
    for step in range(10_000):
        comm, moved, target, gain = R.sweep_ref(P, comm, _leiden.stream_key(3, 0, 0, 0, step))
        if not moved:
            break
        q1 = C.quality(comm)
        assert q1 > q
        q = q1
    assert moved == 0
    assert R.node_optimality_violations(C, comm, 1e-9 * knn.sum()) == 0


def test_refinement_restatement_stays_inside_connected_parents(knn):
    P = _leiden.Problem([knn], [1.0], [1.0])
    comm = R.sequential(R.Collapsed([knn], [1.0], [1.0]), refine=False, n_iterations=1, seed=0)
    refined = np.arange(P.n)
    for r in range(1000):
        refined, moved, pending, _, _ = R.refine_round_ref(P, refined, comm, _leiden.stream_key(3, 1, 0, 0, r))
        if not moved and not pending:
            break
    assert not pending
    for s in np.unique(refined):
        assert np.unique(comm[refined == s]).size == 1
    assert R.disconnected_communities(knn, refined) == 0
    assert np.unique(refined).size < P.n


def _mudata(A, B):
    mods = {}
    for name, G in (("rna", A), ("atac", B)):
        ad = SimpleAnnData(np.zeros((G.shape[0], 1), np.float32))
        ad.obsp["connectivities"] = G
        ad.uns["neighbors"] = {"connectivities_key": "connectivities", "params": {}}
        mods[name] = ad
    return SimpleMuData(mods)


def test_reference_driver_reproduces_fixture():
    from oracle._refload import reference_available
    if not reference_available():
        pytest.skip("reference checkout not present")
    leiden, louvain = R.load_reference_cluster()
    z = np.load(os.path.join(GOLDEN, "leiden_small.npz"))
    A, B = golden_csr(z, "A"), golden_csr(z, "B")
    for alg, fn in (("leiden", leiden), ("louvain", louvain)):
        for name, kw in R.REFERENCE_CALLS.items():
            md = _mudata(A, B)
            fn(md, **kw)
            assert np.array_equal(np.asarray(md.obs[alg].astype(int)), z[f"{alg}_{name}_labels"])
            assert list(md.obs[alg].cat.categories) == list(z[f"{alg}_{name}_categories"])
            assert json.loads(json.dumps(md.uns[alg]["params"])) == json.loads(str(z[f"{alg}_{name}_params"]))
        with pytest.raises(AssertionError):
            fn(_mudata(A, B), mod_weights=[1.0, 2.0, 3.0])
        with pytest.raises(AssertionError):
            fn(_mudata(A, B), resolution=[1.0])
        with pytest.raises(TypeError):
            fn(A)


@pytest.mark.parametrize("name", ["leiden", "louvain"])
def test_signature_matches_reference(name):
    ref = json.load(open(os.path.join(GOLDEN, "cluster_signature.json")))[name]
    sig = inspect.signature(getattr(_leiden, name))
    pos = [p for p in sig.parameters.values() if p.kind == p.POSITIONAL_OR_KEYWORD]
    assert [p.name for p in pos] == ref["params"]
    for i, (p, d) in enumerate(zip(pos, ref["defaults"])):
        if i < ref["required"]:
            assert p.default is inspect.Parameter.empty
        elif d == "MappingProxyType({})":
            assert type(p.default).__name__ == "mappingproxy" and len(p.default) == 0
        else:
            assert repr(p.default) == d, (p.name, p.default, d)
    extra = [p for p in sig.parameters.values() if p.kind != p.POSITIONAL_OR_KEYWORD]
    assert [p.name for p in extra if p.kind == p.VAR_KEYWORD] == [ref["var_keyword"]]
    assert all(p.kind in (p.KEYWORD_ONLY, p.VAR_KEYWORD) for p in extra)


def test_errors_before_device_work():
    labels, A, B = R.small_case()
    with pytest.raises(TypeError):
        mu.tl.leiden(A)
    with pytest.raises(AssertionError):
        mu.tl.leiden(_mudata(A, B), mod_weights=[1.0])
    with pytest.raises(AssertionError):
        mu.tl.louvain(_mudata(A, B), resolution=[1.0, 2.0, 3.0])
    with pytest.raises(KeyError):
        mu.tl.leiden(_mudata(A, B), neighbors_key="wnn")
    with pytest.raises(NotImplementedError):
        mu.tl.leiden(_mudata(A, B), partition_type=type("ModularityVertexPartition", (), {}))
    with pytest.raises(NotImplementedError):
        mu.tl.leiden(_mudata(A, B), partition_kwargs={"node_sizes": [1]})
    with pytest.raises(NotImplementedError):
        mu.tl.leiden(_mudata(A, B), partition_kwargs={"weights": [1.0]})
    with pytest.raises(TypeError):
        mu.tl.leiden(_mudata(A, B), resolution=1.5, partition_kwargs={"resolution_parameter": 2.0})
    with pytest.raises(NotImplementedError):
        mu.tl.leiden(_mudata(A, B), is_membership_fixed=[False] * A.shape[0])
    with pytest.raises(TypeError):
        mu.tl.leiden(_mudata(A, B), max_comm_size=10)
    asym = sp.csr_matrix(np.triu(A.toarray()))
    with pytest.raises(NotImplementedError):
        mu.tl.leiden(_mudata(asym, B))
    with pytest.raises(ValueError):
        mu.tl.leiden(_mudata(sp.csr_matrix(A.shape, dtype=np.float32), B))
    five = SimpleMuData({f"m{i}": _mudata(A, B).mod["rna"] for i in range(5)})
    with pytest.raises(NotImplementedError):
        mu.tl.leiden(five)
    ad = _mudata(A, B).mod["rna"]
    for bad in ("restrict_to", "adjacency", "obsp", "flavor"):
        with pytest.raises(NotImplementedError):
            mu.tl.leiden(ad, **{bad: None})
    with pytest.raises(KeyError):
        mu.tl.louvain(ad, neighbors_key="wnn")


def test_renumber_by_size_breaks_ties_by_smallest_vertex():
    lab = np.array([5, 5, 2, 2, 9, 9, 9, 7])
    assert _leiden.renumber_by_size(lab).tolist() == [1, 1, 2, 2, 0, 0, 0, 3]
    assert R.renumber_by_size(lab).tolist() == [1, 1, 2, 2, 0, 0, 0, 3]
