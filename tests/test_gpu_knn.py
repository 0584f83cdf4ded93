"""GPU: exact brute-force kNN kernel (groundwork for the WNN row) vs float64 numpy."""
import numpy as np
import pytest
import torch

from muon_b200 import _device

pytestmark = pytest.mark.gpu


def _ref(X, Y, k):
    D = np.sqrt(((X[:, None, :].astype(np.float64) - Y[None, :, :].astype(np.float64)) ** 2).sum(-1))
    idx = np.argsort(D, axis=1, kind="stable")[:, :k]
    return idx, np.take_along_axis(D, idx, axis=1), D


@pytest.mark.parametrize("n,d,k", [(1000, 50, 201), (777, 30, 16), (130, 7, 5), (300, 80, 64)])
def test_knn_self(cuda, n, d, k):
    rng = np.random.default_rng(n)
    X = rng.normal(size=(n, d)).astype(np.float32)
    X /= np.linalg.norm(X, axis=1, keepdims=True)            # WNN works on L2-normalised embeddings
    idx, dist = _device.knn_l2(torch.from_numpy(X).to(cuda), k)
    idx, dist = idx.cpu().numpy(), dist.cpu().numpy()
    ridx, rdist, D = _ref(X, X, k)
    np.testing.assert_array_equal(idx[:, 0], np.arange(n))   # self first ...
    assert np.all(dist[:, 0] == 0)                           # ... at distance exactly 0
    np.testing.assert_allclose(dist, rdist, rtol=2e-6, atol=2e-7)
    assert np.all(np.diff(dist, axis=1) >= 0)
    # same neighbour sets wherever the k-th and (k+1)-th distances are not a numerical tie
    kth, nxt = np.sort(D, axis=1)[:, k - 1], np.sort(D, axis=1)[:, min(k, n - 1)]
    clear = (nxt - kth) > 1e-5
    same = np.array([set(a) == set(b) for a, b in zip(idx, ridx)])
    assert same[clear].all() and clear.mean() > 0.9
    # returned distances are the true distances of the returned indices
    np.testing.assert_allclose(dist, np.take_along_axis(D, idx.astype(np.int64), axis=1), rtol=2e-6, atol=2e-7)


def test_knn_cross_and_short(cuda):
    rng = np.random.default_rng(5)
    X = rng.normal(size=(150, 12)).astype(np.float32)
    Y = rng.normal(size=(40, 12)).astype(np.float32)
    idx, dist = _device.knn_l2(torch.from_numpy(X).to(cuda), 50, torch.from_numpy(Y).to(cuda))
    idx, dist = idx.cpu().numpy(), dist.cpu().numpy()
    ridx, rdist, _ = _ref(X, Y, 40)
    np.testing.assert_array_equal(idx[:, :40], ridx)          # well-separated random data: identical order
    np.testing.assert_allclose(dist[:, :40], rdist, rtol=2e-6)
    assert np.all(idx[:, 40:] == -1) and np.all(np.isinf(dist[:, 40:]))   # fewer candidates than k
    # duplicates: ties resolved by the lower index
    Z = np.repeat(rng.normal(size=(20, 6)).astype(np.float32), 3, axis=0)
    idx, dist = _device.knn_l2(torch.from_numpy(Z).to(cuda), 3)
    idx = idx.cpu().numpy()
    np.testing.assert_array_equal(idx, (np.arange(60) // 3 * 3)[:, None] + np.arange(3)[None, :])


@pytest.mark.parametrize("nq,nc,d,k,normalise", [(3000, 3000, 50, 201, True), (777, 5000, 30, 64, True),
                                                  (300, 300, 7, 10, False), (1000, 2500, 128, 33, False),
                                                  (130, 100, 16, 120, True)])
def test_tensor_core_knn_is_bit_identical_to_the_simt_kernel(cuda, nq, nc, d, k, normalise):
    """wgmma TF32 candidate pass + fp32 re-rank must return exactly what the fp32 SIMT kernel returns (which is
    itself checked against the brute-force oracle above): same indices, same distance bits, same -1 padding."""
    import torch
    from muon_b200 import _device
    from muon_b200._lib import call, load, ptr, stream_ptr
    g = torch.Generator(device="cuda").manual_seed(nq + d)
    centres = torch.randn(9, d, generator=g, device="cuda") * 2.0
    Y = torch.randn(nc, d, generator=g, device="cuda") + centres[torch.randint(0, 9, (nc,), generator=g, device="cuda")]
    X = Y[:nq].clone() if nq <= nc else torch.cat([Y, torch.randn(nq - nc, d, generator=g, device="cuda")])
    if normalise:
        X = torch.nn.functional.normalize(X)
        Y = torch.nn.functional.normalize(Y)
    X, Y = X.contiguous(), Y.contiguous()
    i0, d0 = _device.knn_l2(X, k, Y, algo="simt")
    # call the C ABI directly so that a fallback inside knn_l2 cannot mask a failure
    idx = torch.empty((nq, k), dtype=torch.int32, device="cuda")
    dist = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    nbytes = int(load().mub_knn_l2_tc_workspace_bytes(nq, nc, d))
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    call("mub_knn_l2_tc_f32", ptr(X), nq, ptr(Y), nc, d, d, k, ptr(idx), ptr(dist), ptr(ws), nbytes, ptr(status), stream_ptr())
    assert int(status[0]) == 0
    assert torch.equal(idx, i0)
    assert torch.equal(dist.view(torch.int32), d0.view(torch.int32))
