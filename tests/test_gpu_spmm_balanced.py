"""The tiled SpMM kernel on bands of extreme skew.  Each 128-row band's rows are ranked by length and dealt to the warps
snake-wise; a row's sum does not depend on which warp owns it, so the tiled kernel (rows flagged sorted, fp32 operand,
at least one band per SM) must still match the row-warp kernel (the same arrays flagged unsorted) bit for bit, on CSR
arrays and on the pairs layout.  The matrix has more bands than twice the SM count, so every CTA's pipeline crosses
from one band into the next."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

from muon_b200 import _device

pytestmark = pytest.mark.gpu

D = 2500    # not a multiple of any tile height (192 .. 768 rows of B)
BAND = 128


def _n_rows():
    """more than 2 x SMs bands, the last one 45 rows short of full"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return (2 * sms + 7) * BAND + 45


def _band_kinds(n):
    """row density per band: all empty, one row with every column among empty rows, alternating empty and full rows,
    one full row among random rows, and heavy-tailed random rows elsewhere (the last, partial band included)"""
    rng = np.random.default_rng(11)
    dens = np.minimum(rng.pareto(1.5, n) * 0.01, 1.0)
    nb = -(-n // BAND)
    for b, kind in ((0, "empty"), (1, "one_full"), (2, "alternate"), (3, "full_first"), (4, "full_last"),
                    (nb // 2, "alternate"), (nb // 2 + 1, "empty"), (nb - 2, "one_full")):
        r0 = b * BAND
        band = dens[r0:r0 + BAND]
        if kind == "empty":
            band[:] = 0.0
        elif kind == "one_full":
            band[:] = 0.0
            band[37] = 1.0
        elif kind == "alternate":
            band[0::2] = 0.0
            band[1::2] = 1.0
        elif kind == "full_first":
            band[0] = 1.0
        else:
            band[:] = 0.0
            band[-1] = 1.0
    return dens


@pytest.fixture(scope="module")
def skewed(cuda):
    """sorted CSR, n x D: rows of density 1 hold every column, rows of density 0 none"""
    n = _n_rows()
    dens = _band_kinds(n)
    rng = np.random.default_rng(12)
    blocks = []
    for r0 in range(0, n, 4096):
        m = rng.random((min(n, r0 + 4096) - r0, D), dtype=np.float32) < dens[r0:r0 + 4096, None]
        blocks.append(sp.csr_matrix(m))
    X = sp.vstack(blocks).tocsr().astype(np.float32)
    X.data[:] = rng.standard_normal(X.nnz).astype(np.float32)
    X.sort_indices()
    lens = np.diff(X.indptr)
    assert lens[:BAND].max() == 0 and lens[BAND + 37] == D and (lens[2 * BAND + 1:3 * BAND:2] == D).all()
    return X


def _operands(X, layout, cuda):
    """(sorted, unsorted) views of X on the device: the same arrays, flagged for the tiled and the row-warp kernel"""
    indptr = torch.from_numpy(X.indptr.astype(np.int64)).to(cuda)
    if layout == "csr":
        indices = torch.from_numpy(X.indices.astype(np.int32)).to(cuda)
        data = torch.from_numpy(X.data).to(cuda)
        return (_device.DeviceCSR(indptr, indices, data, X.shape, sorted_indices=True),
                _device.DeviceCSR(indptr, indices, data, X.shape, sorted_indices=False))
    pairs = np.stack([X.indices.astype(np.int32), X.data.view(np.int32)], axis=1)
    pairs = torch.from_numpy(np.ascontiguousarray(pairs)).to(cuda)
    return (_device.DevicePairs(indptr, pairs, X.shape, sorted_indices=True),
            _device.DevicePairs(indptr, pairs, X.shape, sorted_indices=False))


def _bits(t):
    return t.cpu().numpy().view(np.uint32)


@pytest.mark.parametrize("P", [32, 64, 128])
@pytest.mark.parametrize("layout", ["csr", "pairs"])
@pytest.mark.parametrize("accumulate", [False, True])
def test_balanced_bands_match_rowwarp_and_scipy(cuda, skewed, P, layout, accumulate):
    X = skewed
    n = X.shape[0]
    A, Au = _operands(X, layout, cuda)
    B = (np.random.default_rng(P).standard_normal((D, P)) / 8).astype(np.float32)
    Bd = torch.from_numpy(B).to(cuda)
    C0 = torch.from_numpy(np.random.default_rng(P + 1).standard_normal((n, P)).astype(np.float32)).to(cuda)

    def run(M, dynamic=False):
        # without accumulate every row must be written: the output starts as NaN
        out = C0.clone() if accumulate else torch.full((n, P), float("nan"), device=cuda)
        return _device.spmm(M, Bd, out=out, accumulate=accumulate, dynamic=dynamic)

    C = run(A)
    assert np.array_equal(_bits(C), _bits(run(A)))               # run to run
    assert np.array_equal(_bits(C), _bits(run(Au)))              # tiled == row-warp
    assert np.array_equal(_bits(C), _bits(run(Au, dynamic=True)))
    c0 = C0.cpu().numpy().astype(np.float64) if accumulate else 0.0
    X64 = X.astype(np.float64)
    ref = X64 @ B.astype(np.float64) + c0
    scale = abs(X64) @ np.abs(B.astype(np.float64)) + np.abs(c0) + 1e-30
    err = np.abs(C.cpu().numpy() - ref) / scale
    assert err.max() < 5e-6, err.max()


@pytest.mark.parametrize("layout", ["csr", "pairs"])
def test_balanced_row_ranges(cuda, skewed, layout):
    """rows=(j0, j1, o0): a range of at least one band per SM takes the tiled kernel from a shifted indptr, a few
    rows the row-warp kernel; both write the same bits as the full product"""
    X = skewed
    n, P = X.shape[0], 64
    A, Au = _operands(X, layout, cuda)
    Bd = torch.from_numpy((np.random.default_rng(5).standard_normal((D, P)) / 8).astype(np.float32)).to(cuda)
    full = _device.spmm(A, Bd)
    for j0, j1, o0 in [(BAND + 37, n - 3, 5), (0, n, 0), (2 * BAND + 1, 3 * BAND + 7, 0), (n - 1, n, 2)]:
        out = torch.full((o0 + j1 - j0 + 3, P), 7.0, device=cuda)
        got = _device.spmm(A, Bd, out=out.clone(), rows=(j0, j1, o0))
        assert np.array_equal(_bits(got), _bits(_device.spmm(Au, Bd, out=out.clone(), rows=(j0, j1, o0))))
        assert np.array_equal(_bits(got[o0:o0 + j1 - j0]), _bits(full[j0:j1]))
        assert (got[:o0] == 7.0).all() and (got[o0 + j1 - j0:] == 7.0).all()


def test_all_rows_empty(cuda):
    """a matrix without entries: every band's rows tie at length zero; the product is zero, or C itself"""
    n, P = _n_rows(), 32
    X = sp.csr_matrix((n, D), dtype=np.float32)
    Bd = torch.ones((D, P), device=cuda)
    for layout in ("csr", "pairs"):
        A, _ = _operands(X, layout, cuda)
        got = _device.spmm(A, Bd, out=torch.full((n, P), float("nan"), device=cuda))
        assert (got == 0).all()
        C0 = torch.randn((n, P), device=cuda)
        got = _device.spmm(A, Bd, out=C0.clone(), accumulate=True)
        assert np.array_equal(_bits(got), _bits(C0))
