"""GPU, BASELINE-scale shapes: size-independent properties instead of an oracle (the scipy path cannot
hold these matrices).  400k cells x 200k peaks at 3 % = 2.4e9 non-zeros, i.e. beyond 2^31 so that every
64-bit offset path is exercised.  Peak HBM: counts 19 GB + TF-IDF values 10 GB + transposed panels 19 GB."""
import pytest
import torch

import muon_b200 as mu
from muon_b200 import _device
from muon_b200._lsi import CsrOperator, truncated_svd
from muon_b200._synth import generate_device, make_tables

pytestmark = pytest.mark.gpu

N, D, DENS = 400_000, 200_000, 0.03


@pytest.fixture(scope="module")
def big(cuda):
    torch.cuda.empty_cache()               # blocks cached by earlier tests count as used in mem_get_info
    free, _ = torch.cuda.mem_get_info()
    if free < 60 << 30:
        pytest.skip("needs ~60 GB of free HBM")
    A = generate_device(N, D, DENS, tables=make_tables(D, DENS, 64, 1))
    assert A.nnz > 2**31
    return A


def _slice_rows(A, r0, r1):
    """Rows [r0, r1) re-based as their own small CSR (independent of 64-bit offsets)."""
    k0, k1 = int(A.indptr[r0]), int(A.indptr[r1])
    return mu.DeviceCSR((A.indptr[r0:r1 + 1] - k0).contiguous(), A.indices[k0:k1].clone(), A.data[k0:k1].clone(),
                        (r1 - r0, A.shape[1]))


def test_tfidf_properties_beyond_2_31(big):
    X = _device.tfidf_csr(big)
    aux = X._aux
    # pattern untouched, counts untouched, sums exact (integer-valued fp32 counts)
    assert X.indices.data_ptr() == big.indices.data_ptr() and X.data.data_ptr() != big.data.data_ptr()
    f64 = torch.float64      # each individual sum is an integer < 2^24, exact in fp32; totals need fp64
    assert float(aux["col_sum"].sum(dtype=f64)) == float(aux["row_sum"].sum(dtype=f64)) == float(big.data.sum(dtype=f64))
    # rows past the 2^31-th non-zero: values equal the closed form evaluated with torch on a re-based slice
    r0 = N - 2000
    S = _slice_rows(big, r0, N)
    rows = torch.repeat_interleave(torch.arange(2000, device=S.data.device), S.indptr[1:] - S.indptr[:-1])
    inv_r = 1.0 / aux["row_sum"][r0:][rows]
    ref = torch.log1p((inv_r * S.data) * 1e4) * aux["idf"][S.indices.long()]
    k0 = int(big.indptr[r0])
    assert k0 > 2**31
    got = X.data[k0:]
    assert float(((got - ref).abs() / ref.abs()).max()) < 2e-6
    assert bool(torch.isfinite(X.data[::1009]).all()) and float(X.data[::1009].min()) > 0


def test_spmm_and_transpose_beyond_2_31(big):
    B = torch.randn((D, 64), device=big.data.device)
    C = _device.spmm(big, B, dynamic=False)
    r0 = N - 1500
    Cs = _device.spmm(_slice_rows(big, r0, N), B, dynamic=False)
    assert torch.equal(C[r0:], Cs)                       # same kernel, same order: bit-identical
    # linearity
    B2 = torch.randn((D, 64), device=big.data.device)
    lhs = _device.spmm(big, (B + 0.5 * B2).contiguous(), dynamic=False)
    rhs = C + 0.5 * _device.spmm(big, B2, dynamic=False)
    assert float((lhs - rhs).abs().max() / rhs.abs().max()) < 2e-5
    # adjoint identity  <A B, Y> == <B, A^T Y>  through the transposed row panels
    Y = torch.randn((N, 64), device=big.data.device)
    At = big.transpose_panels(64)
    assert sum(T.nnz for _, _, T in At.panels) == big.nnz
    Z = At.spmm(Y)
    a = float((C.double() * Y.double()).sum())
    b = float((B.double() * Z.double()).sum())
    assert abs(a - b) / abs(a) < 1e-5
    big._tp = None


def test_lsi_properties_at_scale(big):
    X = _device.tfidf_csr(big)
    k = 50
    U, s, V, info = truncated_svd(CsrOperator(X, 64), k, 64, tol=1e-5)
    assert info.converged and info.passes <= 25
    eye = torch.eye(k, dtype=torch.float64, device=U.device)
    assert float((U.double().T @ U.double() - eye).abs().max()) < 1e-4
    assert float((V.double().T @ V.double() - eye).abs().max()) < 1e-4
    assert bool((s[:-1] >= s[1:]).all())
    # singular-triplet residuals  ||A v - sigma u|| / sigma  on the resident matrix
    AV = _device.spmm(X, torch.nn.functional.pad(V, (0, 64 - k)).contiguous(), dynamic=False)[:, :k]
    res = (AV.double() - U.double() * s).norm(dim=0) / s
    assert float(res.max()) < 5e-5
