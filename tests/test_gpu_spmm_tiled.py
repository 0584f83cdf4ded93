"""Products of matrices flagged sorted against the same arrays flagged unsorted and float64 scipy, on CSR arrays and on
the pairs layout, fp32 and half operand, P = 32, 64, 128.  A fp32 product on sorted CSR arrays runs the tiled kernel
(B staged in shared memory tile by tile), everything else the row-warp kernel; the two kernels assign every entry to
the same lane and sum in the same order, so all results agree bit for bit."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

import muon_b200 as mu
from muon_b200 import _device

pytestmark = pytest.mark.gpu

D = 2500    # not a multiple of any tile height (128 .. 1024 rows of B)
N = 301     # not a multiple of the band height (96 or 128 rows)


def _matrix(n, d, seed):
    """Sorted CSR with empty rows, a row inside one tile, a row with every column (so it spans every tile and runs
    through more than 32 entries of one tile), and random rows of 0 .. 8 % density."""
    rng = np.random.default_rng(seed)
    rows = []
    for i in range(n):
        if i % 17 == 3:
            cols = np.arange(0)
        elif i % 17 == 5:
            cols = np.arange(600, 611)
        elif i == n - 2 or (i == 0 and n == 1):
            cols = np.arange(d)
        else:
            cols = np.sort(rng.choice(d, int(rng.integers(0, d // 12)), replace=False))
        rows.append(sp.csr_matrix((rng.standard_normal(cols.size).astype(np.float32), (np.zeros(cols.size, int), cols)),
                                  shape=(1, d)))
    X = sp.vstack(rows).tocsr()
    X.sort_indices()
    return X


def _operands(X, layout, cuda):
    """(sorted, unsorted) views of X on the device: the same arrays, flagged for the tiled and the row-warp kernel"""
    if layout == "csr":
        A = mu.DeviceCSR.from_scipy(X)
        assert A.sorted_indices
        return A, mu.DeviceCSR(A.indptr, A.indices, A.data, A.shape, sorted_indices=False)
    pairs = np.stack([X.indices.astype(np.int32), X.data.astype(np.float32).view(np.int32)], axis=1)
    indptr = torch.from_numpy(X.indptr.astype(np.int64)).to(cuda)
    pairs = torch.from_numpy(np.ascontiguousarray(pairs)).to(cuda)
    return (_device.DevicePairs(indptr, pairs, X.shape, sorted_indices=True),
            _device.DevicePairs(indptr, pairs, X.shape, sorted_indices=False))


def _bits(t):
    return t.cpu().numpy().view(np.uint32)


@pytest.mark.parametrize("P", [32, 64, 128])
@pytest.mark.parametrize("half", [False, True])
@pytest.mark.parametrize("layout", ["csr", "pairs"])
@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("n", [N, 1])
def test_tiled_matches_rowwarp_and_scipy(cuda, P, half, layout, accumulate, n):
    X = _matrix(n, D, seed=P + n)
    A, Au = _operands(X, layout, cuda)
    B = (np.random.default_rng(1).standard_normal((D, P)) / 8).astype(np.float32)   # |B| < 1: finite once scaled to half
    Bd = torch.from_numpy(B).to(cuda)
    Bop = _device.to_half_scaled(Bd) if half else Bd
    C0 = torch.from_numpy(np.random.default_rng(2).standard_normal((n, P)).astype(np.float32)).to(cuda)

    def run(M, dynamic=False):
        return _device.spmm(M, Bop, out=C0.clone() if accumulate else None, accumulate=accumulate, dynamic=dynamic)

    C = run(A)
    assert np.array_equal(_bits(C), _bits(run(A)))               # run to run
    assert np.array_equal(_bits(C), _bits(run(Au)))              # tiled == row-warp
    assert np.array_equal(_bits(C), _bits(run(Au, dynamic=True)))
    Bref = (Bop.float() / _device.HALF_SCALE).cpu().numpy().astype(np.float64) if half else B.astype(np.float64)
    ref = X.astype(np.float64) @ Bref + (C0.cpu().numpy() if accumulate else 0.0)
    scale = np.abs(X).astype(np.float64) @ np.abs(Bref) + (np.abs(C0.cpu().numpy()) if accumulate else 0.0) + 1e-30
    err = np.abs(C.cpu().numpy() - ref) / scale
    assert err.max() < 5e-6, err.max()


@pytest.mark.parametrize("P", [32, 64, 128])
@pytest.mark.parametrize("half", [False, True])
@pytest.mark.parametrize("layout", ["csr", "pairs"])
def test_tiled_row_range(cuda, P, half, layout):
    """rows=(j0, j1, o0): a sub-range of the rows, written to a compact buffer, as the sampled residual check does"""
    X = _matrix(N, D, seed=7)
    A, Au = _operands(X, layout, cuda)
    Bd = torch.from_numpy((np.random.default_rng(3).standard_normal((D, P)) / 8).astype(np.float32)).to(cuda)
    Bop = _device.to_half_scaled(Bd) if half else Bd
    full = _device.spmm(A, Bop)
    for j0, j1, o0 in [(0, 1, 0), (130, 299, 5), (N - 1, N, 0)]:
        out = torch.full((o0 + j1 - j0 + 3, P), 7.0, device=cuda)
        got = _device.spmm(A, Bop, out=out.clone(), rows=(j0, j1, o0))
        assert np.array_equal(_bits(got), _bits(_device.spmm(Au, Bop, out=out.clone(), rows=(j0, j1, o0))))
        assert np.array_equal(_bits(got[o0:o0 + j1 - j0]), _bits(full[j0:j1]))
        assert (got[:o0] == 7.0).all() and (got[o0 + j1 - j0:] == 7.0).all()


def test_panels_from_tiled_fill_are_flagged_sorted(cuda):
    """Aᵀ panels from the deterministic fill are flagged sorted; their product is the same flagged or not"""
    from muon_b200._synth import generate_device, make_tables
    A = _device.tfidf_csr(generate_device(3000, 4000, 0.03, tables=make_tables(4000, 0.03, 64, 1)))
    Tp = A.transpose_panels(64)
    assert Tp.tiled_fill and all(T.sorted_indices for _, _, T in Tp.panels)
    Y = torch.randn((3000, 64), device=cuda, generator=torch.Generator(device=cuda).manual_seed(0)) / 8
    for half in (False, True):
        Z = Tp.spmm(Y, half=half)
        Yop = _device.to_half_scaled(Y) if half else Y
        ref = torch.empty_like(Z)
        for i, (r0, r1, T) in enumerate(Tp.panels):
            Tu = _device.DevicePairs(T.indptr, T.pairs, T.shape, sorted_indices=False)
            _device.spmm(Tu, Yop[r0:r1], out=ref, accumulate=i > 0)
        assert np.array_equal(_bits(Z), _bits(ref))
