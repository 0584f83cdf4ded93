"""GPU parity of the building-block kernels (SpMM, transpose, Gram, generator) through the C ABI."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

import muon_b200 as mu
from muon_b200 import _device
from muon_b200._synth import generate_device, generate_host, make_tables

pytestmark = pytest.mark.gpu


def _rand_csr(n, d, density, seed, skew=False):
    rng = np.random.default_rng(seed)
    X = sp.random(n, d, density, format="csr", random_state=seed, dtype=np.float32)
    if skew:  # a few very long rows and many empty ones
        rows = [sp.random(1, d, 0.9, format="csr", random_state=seed + i, dtype=np.float32) for i in range(3)]
        X = sp.vstack([X[: n - 3]] + rows).tocsr()
        X = sp.vstack([sp.csr_matrix((5, d), dtype=np.float32), X]).tocsr()
    X.sort_indices()
    return X


@pytest.mark.parametrize("P", [32, 64, 128])
@pytest.mark.parametrize("dynamic", [False, True])
@pytest.mark.parametrize("n,d,seed", [(3000, 2000, 1), (1500, 5000, 4)])
def test_spmm_vs_scipy(cuda, P, dynamic, n, d, seed):
    X = _rand_csr(n, d, 0.02, seed, skew=True)
    B = np.random.default_rng(2).standard_normal((d, P)).astype(np.float32)
    A = mu.DeviceCSR.from_scipy(X)
    Bd = torch.from_numpy(B).to(cuda)
    C = _device.spmm(A, Bd, dynamic=dynamic)
    ref = X.astype(np.float64) @ B.astype(np.float64)
    scale = np.abs(X).astype(np.float64) @ np.abs(B).astype(np.float64) + 1e-30
    err = np.abs(C.cpu().numpy() - ref) / scale
    assert err.max() < 5e-6, err.max()            # fp32 accumulation, relative to |A||B|
    # accumulate flag
    C2 = _device.spmm(A, Bd, out=C.clone(), accumulate=True, dynamic=dynamic)
    np.testing.assert_allclose(C2.cpu().numpy(), 2 * C.cpu().numpy(), rtol=1e-6, atol=1e-6)
    # a rerun gives the same bits, with either operand type
    np.testing.assert_array_equal(_device.spmm(A, Bd, dynamic=dynamic).cpu().numpy(), C.cpu().numpy())
    Bh = _device.to_half_scaled(Bd)
    Ch = _device.spmm(A, Bh, dynamic=dynamic)
    np.testing.assert_array_equal(_device.spmm(A, Bh, dynamic=dynamic).cpu().numpy(), Ch.cpu().numpy())


def test_spmm_edge_rows(cuda):
    # rows of length 0, 1, 31, 32, 33, 64, 65 exercise the full/tail segment paths
    d = 200
    lens = [0, 1, 31, 32, 33, 64, 65, 0, 127]
    rng = np.random.default_rng(0)
    rows = []
    for L in lens:
        cols = np.sort(rng.choice(d, L, replace=False))
        rows.append(sp.csr_matrix((rng.standard_normal(L).astype(np.float32), (np.zeros(L, int), cols)), shape=(1, d)))
    X = sp.vstack(rows).tocsr()
    B = rng.standard_normal((d, 64)).astype(np.float32)
    C = _device.spmm(mu.DeviceCSR.from_scipy(X), torch.from_numpy(B).to(cuda))
    np.testing.assert_allclose(C.cpu().numpy(), X @ B, rtol=1e-4, atol=1e-5)


def test_transpose_and_spmm_t(cuda):
    X = _rand_csr(2500, 1800, 0.03, 5, skew=True)
    A = mu.DeviceCSR.from_scipy(X)
    At = A.transpose()
    T = At.get()
    T.sort_indices()
    R = X.T.tocsr()
    R.sort_indices()
    np.testing.assert_array_equal(T.indptr, R.indptr)
    np.testing.assert_array_equal(T.indices, R.indices)     # bit-exact after canonical sort
    np.testing.assert_array_equal(T.data, R.data)
    Y = np.random.default_rng(3).standard_normal((X.shape[0], 64)).astype(np.float32)
    Z = _device.spmm(At, torch.from_numpy(Y).to(cuda))
    ref = X.T.astype(np.float64) @ Y.astype(np.float64)
    scale = np.abs(X.T).astype(np.float64) @ np.abs(Y).astype(np.float64) + 1e-30
    assert (np.abs(Z.cpu().numpy() - ref) / scale).max() < 5e-6
    # linearity property (size independent): A^T(aY1 + Y2) = a A^T Y1 + A^T Y2
    Y2 = torch.randn((X.shape[0], 64), device=cuda)
    Yt = torch.from_numpy(Y).to(cuda)
    lhs = _device.spmm(At, (2.5 * Yt + Y2).contiguous())
    rhs = 2.5 * Z + _device.spmm(At, Y2)
    assert float((lhs - rhs).abs().max() / rhs.abs().max()) < 1e-5


@pytest.mark.parametrize("P,l", [(32, 20), (64, 64), (128, 100)])
def test_gram(cuda, P, l):
    rng = np.random.default_rng(0)
    Y = rng.standard_normal((70001, P)).astype(np.float32)
    Y[:, l:] = 0
    w = rng.random(70001).astype(np.float32)
    Yd = torch.from_numpy(Y).to(cuda)
    G = _device.gram(Yd, l).cpu().numpy()
    ref = Y[:, :l].astype(np.float64).T @ Y[:, :l].astype(np.float64)
    np.testing.assert_allclose(G, ref, rtol=0, atol=2e-6 * np.abs(ref).max())
    Gw = _device.gram(Yd, l, weights=torch.from_numpy(w).to(cuda)).cpu().numpy()
    refw = (Y[:, :l].astype(np.float64) * w[:, None]).T @ Y[:, :l].astype(np.float64)
    np.testing.assert_allclose(Gw, refw, rtol=0, atol=2e-6 * np.abs(refw).max())
    G2 = _device.gram(Yd, l).cpu().numpy()
    np.testing.assert_array_equal(G, G2)                  # deterministic


def test_generator_device_equals_host(cuda):
    tb = make_tables(1537, 0.04, n_topics=7, seed=21)
    H = generate_host(333, 1537, 0.04, tables=tb, row0=100)
    D = generate_device(333, 1537, 0.04, tables=tb, row0=100).get()
    np.testing.assert_array_equal(D.indptr, H.indptr)
    np.testing.assert_array_equal(D.indices, H.indices)
    np.testing.assert_array_equal(D.data, H.data)


def test_transposed_panels_equal_full_transpose(cuda, monkeypatch):
    X = _rand_csr(3000, 900, 0.03, 9, skew=True)
    A = mu.DeviceCSR.from_scipy(X)
    monkeypatch.setattr(_device.TransposedPanels, "L2_BUDGET", 700 * 64 * 4)     # force 5 panels
    Tp = _device.TransposedPanels(A, 64)
    assert len(Tp.panels) >= 4 and Tp.panels[0][0] == 0 and Tp.panels[-1][1] == X.shape[0]
    assert all(isinstance(T, _device.DevicePairs) for _, _, T in Tp.panels)       # 8-byte (index, value) pairs
    r0, r1, T0 = Tp.panels[1]
    ref0 = X[r0:r1].T.tocsr()
    got0 = sp.csr_matrix((T0.data.cpu().numpy(), T0.indices.cpu().numpy(), T0.indptr.cpu().numpy()), shape=T0.shape)
    got0.sort_indices()
    ref0.sort_indices()
    np.testing.assert_array_equal(got0.indices, ref0.indices)
    np.testing.assert_array_equal(got0.data, ref0.data)
    Y = torch.randn((X.shape[0], 64), device=cuda)
    Z = Tp.spmm(Y)
    ref = X.T.astype(np.float64) @ Y.cpu().numpy().astype(np.float64)
    scale = np.abs(X.T).astype(np.float64) @ np.abs(Y.cpu().numpy()).astype(np.float64) + 1e-30
    assert (np.abs(Z.cpu().numpy() - ref) / scale).max() < 5e-6
