"""H100: ``mu.tl.umap`` -- the spectral init against ARPACK, the epoch kernel against the numpy Jacobi epoch
(oracle/umap_ref.py), run-to-run determinism, layout quality against umap-learn's sequential layout
(tests/golden/umap_small.npz) and the AnnData / MuData surface."""
import os

import numpy as np
import pytest
import scipy.sparse as sp

import muon_b200 as mu
from conftest import GOLDEN, golden_csr
from muon_b200 import SimpleAnnData, SimpleMuData
from muon_b200 import _umap
from oracle import umap_ref as R

pytestmark = pytest.mark.gpu
K = 15


@pytest.fixture(scope="module")
def small():
    z = dict(np.load(os.path.join(GOLDEN, "umap_small.npz")))
    z["W"] = golden_csr(z, "W")
    return z


def _adata(W, key=None):
    ad = SimpleAnnData(np.zeros((W.shape[0], 1), np.float32))
    nk = key or "neighbors"
    ck = "connectivities" if key is None else f"{key}_connectivities"
    ad.obsp[ck] = W
    ad.uns[nk] = {"connectivities_key": ck, "distances_key": "distances", "params": {"method": "umap"}}
    return ad


def _principal_angles(A, B):
    Qa, _ = np.linalg.qr(A)
    Qb, _ = np.linalg.qr(B)
    s = np.clip(np.linalg.svd(Qa.T @ Qb, compute_uv=False), -1, 1)
    return np.arccos(s)


def _check_spectrum(W, k):
    """Eigenvalues within 1e-4 of ARPACK's; principal angles <= 1e-3 per group of eigenvalues whose gap to the rest
    (including the first eigenvalue not computed) is resolved (> 1e-2)."""
    lam, V = _umap.spectral_eigs(W, k)
    ref, Vr = R.laplacian_eigs(W, k + 1)
    np.testing.assert_allclose(lam, ref[:k], rtol=0, atol=1e-4)
    bounds = [0] + [i for i in range(1, k + 1) if ref[i] - ref[i - 1] > 1e-2]
    checked = 0
    for g0, g1 in zip(bounds[:-1], bounds[1:]):
        assert _principal_angles(V[:, g0:g1], Vr[:, g0:g1]).max() <= 1e-3, (g0, g1, lam, ref)
        checked += 1
    assert checked >= 1


def test_spectral_eigs_connected_graph(cuda):
    X, labels, W = R.planted_graph(n=1200, n_clusters=3, spread=1.0, seed=5)
    from scipy.sparse.csgraph import connected_components
    assert connected_components(W)[0] == 1
    _check_spectrum(W, 3)
    _check_spectrum(W, 5)


def test_spectral_eigs_two_components(cuda):
    _, _, W1 = R.planted_graph(n=600, n_clusters=2, spread=1.0, seed=6)
    _, _, W2 = R.planted_graph(n=500, n_clusters=2, spread=1.0, seed=7)
    W = sp.block_diag([W1, W2]).tocsr().astype(np.float32)
    _check_spectrum(W, 4)
    # the layout path: every component gets its own eigenvectors around +-e_1
    ad = _adata(W)
    mu.tl.umap(ad, maxiter=50)
    Y = ad.obsm["X_umap"]
    assert Y.shape == (1100, 2) and Y.dtype == np.float32 and np.isfinite(Y).all()


def test_philox_stream_matches_numpy(cuda):
    rng = np.random.default_rng(0)
    ctr = rng.integers(0, 2**32, size=(4096, 4), dtype=np.uint64).astype(np.uint32)
    k0, k1 = 0x12345678, 0x9ABCDEF0
    got = _umap.philox4x32_10(ctr, k0, k1)
    want = np.stack(R.philox4x32_10(ctr[:, 0], ctr[:, 1], ctr[:, 2], ctr[:, 3], k0, k1), 1)
    np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize("dim", [2, 3, 10])
def test_epochs_match_the_numpy_jacobi_epoch(cuda, small, dim):
    """From one start and one key, every epoch of the kernel agrees with ``epoch_ref`` applied to the same positions,
    over epochs 1..10, and chaining the kernel's epochs gives the same positions as one 1-, 2- or 10-epoch run.

    The two are not run freely side by side for 10 epochs: near coincident points the repulsion term changes at
    2 gamma b / 0.001 per unit of distance, so rounding differences of 1e-7 grow by about 100x per epoch
    (``epoch_ref`` against itself from a start perturbed by 1e-6 differs by O(10) after 10 epochs)."""
    n_epochs = 200
    G, _ = _umap.prune(small["W"], n_epochs)
    eps = _umap.epochs_per_sample(G.data)
    rs = np.random.RandomState(3)
    Y0 = _umap.initial_positions(G, dim, "random", rs, None)
    key = _umap.sampler_key(rs)
    a, b = _umap.find_ab_params(1.0, 0.5)
    lay = _umap.Layout(G, eps)
    kw = dict(a=a, b=b, gamma=1.0, alpha=1.0, negative_sample_rate=5, key=key)
    Y = Y0
    for ep in range(1, 11):
        got = lay.run(Y, range(ep, ep + 1), n_epochs, **kw).cpu().numpy()
        want = R.epoch_ref(G, eps, Y, ep, n_epochs, a, b, 1.0, 1.0, 5, key)
        np.testing.assert_allclose(got, want, rtol=0, atol=1e-4, err_msg=f"epoch {ep}")
        Y = got
        if ep in (1, 2, 10):
            assert np.array_equal(lay.run(Y0, range(1, ep + 1), n_epochs, **kw).cpu().numpy(), Y)


def test_deterministic_per_random_state(cuda, small):
    runs = []
    for rs in (42, 42, 7):
        ad = _adata(small["W"])
        mu.tl.umap(ad, random_state=rs)
        runs.append(ad.obsm["X_umap"])
    assert np.array_equal(runs[0], runs[1])
    assert not np.array_equal(runs[0], runs[2])


def test_quality_matches_sequential_umap(cuda, small):
    ad = _adata(small["W"])
    mu.tl.umap(ad)
    Y = ad.obsm["X_umap"]
    trust = R.trustworthiness(small["rep"], Y, K)
    agree = R.knn_label_agreement(Y, small["labels"], K)
    print(f"trustworthiness {trust:.4f} (sequential {float(small['trust_ref']):.4f}), "
          f"label agreement {agree:.4f} (sequential {float(small['label_ref']):.4f})")
    assert abs(trust - float(small["trust_ref"])) <= 0.02
    assert abs(agree - float(small["label_ref"])) <= 0.02


def test_mudata_anndata_keys_copy_and_init(cuda, small):
    W = small["W"]
    n = W.shape[0]
    a, b = _umap.find_ab_params(1.0, 0.5)

    ad = _adata(W)
    assert mu.tl.umap(ad, maxiter=30) is None
    Y_ad = ad.obsm["X_umap"]
    assert Y_ad.shape == (n, 2) and Y_ad.dtype == np.float32
    assert ad.uns["umap"] == {"params": {"a": a, "b": b, "random_state": 42}}

    md = SimpleMuData({"rna": SimpleAnnData(np.zeros((n, 3), np.float32)),
                       "atac": SimpleAnnData(np.zeros((n, 2), np.float32))})
    md.obsp["connectivities"] = W
    md.uns["neighbors"] = {"connectivities_key": "connectivities", "distances_key": "distances", "params": {}}
    assert mu.tl.umap(md, maxiter=30) is None
    np.testing.assert_array_equal(md.obsm["X_umap"], Y_ad)           # same graph, same seed: same layout
    assert set(md.uns["umap"]["params"]) == {"a", "b", "random_state"}

    wnn = _adata(W, key="wnn")
    out = mu.tl.umap(wnn, maxiter=30, neighbors_key="wnn", copy=True, random_state=0, method="rapids")
    assert "X_umap" not in wnn.obsm and "umap" not in wnn.uns
    assert out.obsm["X_umap"].shape == (n, 2)
    assert out.uns["umap"] == {"params": {"a": a, "b": b}}            # random_state 0 is not recorded

    ad3 = _adata(W)
    mu.tl.umap(ad3, maxiter=30, n_components=3, init_pos="random", a=1.5, b=0.8)
    assert ad3.obsm["X_umap"].shape == (n, 3) and np.isfinite(ad3.obsm["X_umap"]).all()
    assert ad3.uns["umap"]["params"]["a"] == 1.5 and ad3.uns["umap"]["params"]["b"] == 0.8

    init = np.random.default_rng(0).normal(size=(n, 2)).astype(np.float32)
    ad4, ad5 = _adata(W), _adata(W)
    mu.tl.umap(ad4, maxiter=30, init_pos=init)
    ad5.obsm["X_start"] = init
    mu.tl.umap(ad5, maxiter=30, init_pos="X_start")
    assert np.array_equal(ad4.obsm["X_umap"], ad5.obsm["X_umap"])
    assert R.knn_label_agreement(ad4.obsm["X_umap"], small["labels"]) > 0.5


def test_errors(cuda, small):
    W = small["W"]
    with pytest.raises(TypeError):
        mu.tl.umap(W)
    with pytest.raises(ValueError):
        mu.tl.umap(SimpleAnnData(np.zeros((5, 2), np.float32)))
    with pytest.raises(ValueError):
        mu.tl.umap(_adata(W), neighbors_key="wnn")
    with pytest.raises(NotImplementedError):
        mu.tl.umap(_adata(W), n_components=17)
    five = sp.block_diag([R.planted_graph(n=60, n_clusters=1, seed=s)[2] for s in range(5)]).tocsr()
    with pytest.raises(NotImplementedError):
        mu.tl.umap(_adata(five))
    ad = _adata(five)
    mu.tl.umap(ad, init_pos="random", maxiter=20)                      # the advertised way out
    assert np.isfinite(ad.obsm["X_umap"]).all()


def test_200k_cells_finite_and_deterministic(cuda):
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
    for _ in range(2):
        ad = _adata(W)
        mu.tl.umap(ad, init_pos="random")
        outs.append(ad.obsm["X_umap"])
    assert outs[0].shape == (N, 2) and np.isfinite(outs[0]).all()
    assert np.array_equal(outs[0], outs[1])
