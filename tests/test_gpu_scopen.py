"""H100: ``mu.atac.pp.scopen`` -- the pattern, SpMM and Gram kernels against exact / float64 references, the device fit
from the stored init against the fixtures (tests/golden/scopen_small.npz) for both bounds, the public call against
the unmodified reference, repeatability, the limits, and a 20,000 x 200,000 fit at 3 % density checked against
scipy-sparse products on sampled rows."""
import time
import warnings

import numpy as np
import pytest
import scipy.sparse as sp

import muon_b200 as mu
import muon_b200._snf as snf
from muon_b200 import SimpleAnnData, SimpleMuData
from muon_b200 import _scopen
from conftest import load_golden
from oracle import scopen_ref as R
from scopen_cases import CASES, arguments, matrix, planted_counts, sample_rows

pytestmark = pytest.mark.gpu

DEFAULTS = {"n_components": 30, "max_iter": 500, "min_rho": 0.0, "max_rho": 0.5, "alpha": 1}


@pytest.fixture(scope="module")
def golden():
    return load_golden("scopen_small.npz")


def _t(a, dt=None):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a if dt is None else a.astype(dt))).cuda()


def _call(name, *args):
    from muon_b200._lib import call, stream_ptr
    call(name, *args, stream_ptr())


def _awkward_csr(n, m, dtype, seed):
    """Rows of every length class: empty, short, and a few long rows, with zeros and negatives stored."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(0, 40, n)
    lens[::7] = 0
    lens[3], lens[10] = m, m // 2
    rows = [np.sort(rng.choice(m, size=L, replace=False)) for L in lens]
    indptr = np.concatenate([[0], np.cumsum(lens)])
    indices = np.concatenate(rows).astype(np.int32)
    data = rng.choice([-2.0, -0.5, 0.0, 0.25, 1.0, 3.0], size=indices.size).astype(dtype)
    return sp.csr_matrix((data, indices, indptr), shape=(n, m))


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_pattern_kernels_are_exact(cuda, dtype):
    import torch

    from muon_b200._lib import ptr
    X = _awkward_csr(500, 3000, dtype, 1)
    sfx = "f32" if dtype == np.float32 else "f64"
    indptr, indices, data = _t(X.indptr, np.int64), _t(X.indices, np.int32), _t(X.data)
    count = torch.empty(X.shape[0], dtype=torch.int64, device=cuda)
    _call(f"mub_scopen_pattern_count_{sfx}", ptr(indptr), ptr(data), X.shape[0], ptr(count))
    pos = X.data > 0
    want = np.diff(np.concatenate([[0], np.cumsum(pos)])[X.indptr])
    np.testing.assert_array_equal(count.cpu().numpy(), want)
    out_indptr = torch.zeros(X.shape[0] + 1, dtype=torch.int64, device=cuda)
    torch.cumsum(count, 0, out=out_indptr[1:])
    scale = _t(np.linspace(0.5, 2.0, X.shape[0]), np.float32)
    nnz = int(want.sum())
    oi = torch.empty(nnz, dtype=torch.int32, device=cuda)
    od = torch.empty(nnz, dtype=torch.float32, device=cuda)
    _call(f"mub_scopen_pattern_fill_{sfx}", ptr(indptr), ptr(indices), ptr(data), X.shape[0], ptr(out_indptr),
          ptr(scale), ptr(oi), ptr(od))
    np.testing.assert_array_equal(oi.cpu().numpy(), X.indices[pos])
    rows = np.repeat(np.arange(X.shape[0]), want)
    np.testing.assert_array_equal(od.cpu().numpy(), scale.cpu().numpy()[rows])


@pytest.mark.parametrize("k", [1, 7, 30, 32, 33, 64])
def test_pattern_spmm_and_gram_match_float64(cuda, k):
    import torch

    from muon_b200._lib import load, ptr
    X = _awkward_csr(700, 2500, np.float64, k)
    P = sp.csr_matrix((np.ones(X.nnz), X.indices, X.indptr), shape=X.shape)
    rng = np.random.default_rng(k)
    B = rng.standard_normal((X.shape[1], k))
    rs, cs = rng.uniform(0.5, 2, X.shape[0]), rng.uniform(0.5, 2, X.shape[1])
    # every device operand is held in a name until the kernel has run: a temporary freed inside the argument list
    # could hand its memory to the next operand
    indptr, indices, Bd = _t(X.indptr, np.int64), _t(X.indices, np.int32), _t(B)
    rs_d, cs_d = _t(rs), _t(cs)
    for row_scale, col_scale in ((None, None), (rs, None), (None, cs), (rs, cs)):
        C = torch.empty((X.shape[0], k), dtype=torch.float64, device=cuda)
        _call("mub_scopen_spmm_f64", ptr(indptr), ptr(indices), X.shape[0], ptr(None if row_scale is None else rs_d),
              ptr(None if col_scale is None else cs_d), ptr(Bd), k, ptr(C))
        want = P @ (B if col_scale is None else col_scale[:, None] * B)
        want = want if row_scale is None else row_scale[:, None] * want
        got = C.cpu().numpy()
        scale = np.maximum(np.abs(P) @ np.abs(B if col_scale is None else col_scale[:, None] * B), 1e-300)
        scale = scale if row_scale is None else row_scale[:, None] * scale
        assert np.all(np.abs(got - want) <= 1e-13 * scale.max(axis=1, keepdims=True))
        assert np.all(got[np.diff(X.indptr) == 0] == 0)
    for rows in (1, 31, 33, 100_003):
        Y = rng.standard_normal((rows, k))
        ws = torch.empty(max(int(load().mub_scopen_workspace_bytes(rows, k)), 8), dtype=torch.uint8, device=cuda)
        G = torch.empty((k, k), dtype=torch.float64, device=cuda)
        Yd = _t(Y)
        _call("mub_scopen_gram_f64", ptr(Yd), rows, k, ptr(ws), ptr(G))
        want = Y.T @ Y
        norms = np.sqrt(np.diag(np.abs(Y).T @ np.abs(Y)))
        assert np.all(np.abs(G.cpu().numpy() - want) <= 1e-13 * np.outer(norms, norms))


def _device_fit(case, init, upper):
    kw = {**DEFAULTS, **CASES[case][5]}
    X, _ = matrix(case)
    src, counts = _scopen.host_pattern_source(X)
    fit = _scopen.Fit(src, kw["n_components"])
    fit.positives()
    fit.build(_scopen.scale_of(counts, kw["min_rho"], kw["max_rho"]))
    fit.set_factors(*init)
    n_iter = _scopen.solve(fit, kw["max_iter"], float(kw["alpha"]), upper=upper)
    return fit, n_iter


def _assert_columns_close(got, want, rtol):
    scale = np.maximum(np.abs(want).max(axis=0), 1e-300)
    gap = (np.abs(got - want) / scale).max()
    assert gap <= rtol, gap
    return gap


@pytest.mark.parametrize("case", list(CASES))
def test_device_fit_from_stored_init(cuda, golden, case):
    z = golden
    init = (z[f"{case}_W0"], z[f"{case}_H0"])
    for upper, sfx in ((1.0, ""), (np.inf, "_inf")):
        fit, n_iter = _device_fit(case, init, upper)
        W, H = fit.factors()
        assert n_iter == int(z[f"{case}_n_iter{sfx}"])
        gw = _assert_columns_close(W, z[f"{case}_W{sfx}"], 1e-10)
        gh = _assert_columns_close(H.T, z[f"{case}_H{sfx}"].T, 1e-10)
        print(f"{case} bound {upper}: W gap {gw:.2e}, H gap {gh:.2e}")


@pytest.mark.parametrize("case", list(CASES))
def test_public_call_matches_the_reference(cuda, golden, capsys, case):
    z = golden
    data, ad, kw = arguments(case, (SimpleAnnData, SimpleMuData))
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        assert mu.atac.pp.scopen(data, **kw) is None
    lines = capsys.readouterr().out.splitlines()
    assert lines[:3] == list(z[f"{case}_lines"])
    assert [str(w.message) for w in rec] == list(z[f"{case}_warnings"])
    W, Ht, M = ad.varm["scopen"], ad.obsm["X_scopen"], ad.X.T
    assert M.flags.c_contiguous and M.dtype == np.float64
    floor = 1e-12      # float64 rounding of sums taken in another order
    tol_M = 2 * float(z[f"{case}_sens_M"]) + floor
    tol_W = 2 * float(z[f"{case}_sens_W"]) + floor
    gap_M = np.abs(M[sample_rows(M.shape[0])] - z[f"{case}_M_rows"]).max()
    gap_W = _assert_columns_close(W, z[f"{case}_W"], tol_W)
    gap_H = _assert_columns_close(Ht, z[f"{case}_H"].T, tol_W)
    kw_all = {**DEFAULTS, **kw}
    P, c = R.pattern_of(matrix(case)[0])
    Xd = R.dense_of(P, R.scale_of(c, kw_all["min_rho"], kw_all["max_rho"]))
    obj = R.objective(Xd, W, Ht.T, float(kw_all["alpha"]))
    gap_obj = abs(obj - float(z[f"{case}_objective"])) / float(z[f"{case}_objective"])
    print(f"{case}: M gap {gap_M:.2e} (allowed {tol_M:.2e}), W gap {gap_W:.2e}, H gap {gap_H:.2e} "
          f"(allowed {tol_W:.2e}), objective gap {gap_obj:.2e}")
    assert gap_M <= tol_M
    assert gap_obj <= 1e-8


def test_repeatable_device_input_and_limits(cuda, monkeypatch):
    X, _ = matrix("csr_f32")
    outs = []
    for _ in range(2):
        ad = SimpleAnnData(X.copy())
        mu.atac.pp.scopen(ad, n_components=10, max_iter=50)
        outs.append(ad)
    for key in ("X_scopen",):
        assert np.array_equal(outs[0].obsm[key], outs[1].obsm[key])
    assert np.array_equal(outs[0].varm["scopen"], outs[1].varm["scopen"])
    assert np.array_equal(outs[0].X, outs[1].X)

    src, _ = _scopen.host_pattern_source(X)
    ad = SimpleAnnData(mu.DeviceCSR.from_scipy(src))
    mu.atac.pp.scopen(ad, n_components=10, max_iter=50)
    assert np.array_equal(ad.varm["scopen"], outs[0].varm["scopen"])
    assert np.array_equal(ad.X, outs[0].X)

    big = sp.csr_matrix(planted_counts(0, 80, 150, 4))
    ad = SimpleAnnData(big.copy())
    mu.atac.pp.scopen(ad, n_components=64, max_iter=3)
    assert ad.obsm["X_scopen"].shape == (80, 64)
    with pytest.raises(NotImplementedError, match="at most 64"):
        mu.atac.pp.scopen(SimpleAnnData(big.copy()), n_components=65)
    monkeypatch.setattr(snf, "free_device_bytes", lambda: 1 << 20)
    with pytest.raises(NotImplementedError, match="GiB of device memory"):
        mu.atac.pp.scopen(SimpleAnnData(big.copy()), n_components=4)


def test_scale_20k_cells_200k_peaks(cuda):
    """20,000 cells x 200,000 peaks at 3 % density, k = 30, through the internal fit (no dense output): after four
    iterations from the NNDSVD init, the fifth is recomputed on sampled rows with scipy-sparse products in float64."""
    import torch

    from muon_b200._synth import generate_device
    n, m, k, alpha = 20_000, 200_000, 30, 1.0
    A = generate_device(n, m, 0.03, seed=3)
    fit = _scopen.Fit(A, k)
    counts = fit.positives()
    s = _scopen.scale_of(counts, 0.0, 0.5)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fit.build(s)
    W0, H0 = _scopen.nndsvd(*fit.svd())
    fit.set_factors(W0, H0)
    assert _scopen.solve(fit, 4, alpha) == 4
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    W4, H4 = fit.factors()
    fit.iterate(alpha, _scopen.UPPER)
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    W5, H5 = fit.factors()
    print(f"scale: nnz {fit.nnz}, build + init + 4 iterations {t1 - t0:.2f} s, one iteration {t2 - t1:.3f} s")
    assert fit.nnz == int(counts.sum()) and fit.nnz > 0.02 * n * m

    P = fit.P.get()
    P = sp.csr_matrix((np.ones(P.nnz), P.indices, P.indptr), shape=P.shape)
    rng = np.random.default_rng(0)
    peaks, cells = np.sort(rng.choice(m, 64, replace=False)), np.sort(rng.choice(n, 64, replace=False))
    PT_rows = P[:, peaks].T.tocsr()
    Ht4 = H4.T
    XHt = PT_rows @ (s[:, None] * Ht4)
    W_rows = W4[peaks].copy()
    R.cd_sweep(W_rows, Ht4.T @ Ht4 + alpha * np.eye(k), XHt, 1.0)
    gw = _assert_columns_close(W5[peaks], W_rows, 1e-10)
    XtW = s[cells, None] * (P[cells] @ W5)
    H_rows = Ht4[cells].copy()
    R.cd_sweep(H_rows, W5.T @ W5 + alpha * np.eye(k), XtW, 1.0)
    gh = _assert_columns_close(H5.T[cells], H_rows, 1e-10)
    print(f"scale: sampled-row gaps W {gw:.2e}, H {gh:.2e}")
