"""GPU: grouped / union / feature-subset MOFA on device-resident views.  The CSR selection kernel (csrc/select.cu)
against scipy, the zero-copy slices and the deterministic transposition it enables, and the fits against the float64
oracle and the host-matrix path."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

import muon_b200 as mu
from muon_b200 import _device
from muon_b200._containers import SimpleAnnData, SimpleMuData
from muon_b200._lib import MuonB200Error
from oracle.mofa_ref import mofa_ref_general

pytestmark = pytest.mark.gpu


# ---- 1. the kernel against scipy ----------------------------------------------------------------------------------
def _source(seed=0):
    """1500 x 3000 sorted CSR (not a multiple of 512 rows) with empty rows, rows of 33..40 entries and rows of more
    than 1024 entries, explicit zeros included"""
    rng = np.random.default_rng(seed)
    n, d = 1500, 3000
    lens = rng.integers(0, 30, n)
    lens[::7] = 0
    lens[3::11] = rng.integers(33, 41, len(lens[3::11]))
    lens[5::97] = rng.integers(1025, 2500, len(lens[5::97]))
    indptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    indices = np.concatenate([np.sort(rng.choice(d, k, replace=False)) for k in lens]).astype(np.int32)
    data = rng.normal(size=indptr[-1]).astype(np.float32)
    data[::13] = 0.0
    return sp.csr_matrix((data, indices, indptr), shape=(n, d))


def _cases(n, d):
    rng = np.random.default_rng(1)
    some = rng.random(d) < 0.4
    return [
        ("all", None, None),
        ("mask only", None, some),
        ("range", np.arange(100, 1400), None),
        ("range + mask", np.arange(100, 1400), some),
        ("unsorted repeated rows", rng.integers(0, n, 2000), None),
        ("unsorted repeated rows + mask", rng.integers(0, n, 2000), some),
        ("permutation + mask", rng.permutation(n), some),
        ("long rows", np.arange(5, n, 97), some),
        ("empty row list", np.array([], dtype=np.int64), some),
        ("empty row list, no mask", np.array([], dtype=np.int64), None),
        ("every column dropped", np.arange(0, n, 3), np.zeros(d, dtype=bool)),
        ("every column kept", rng.permutation(n)[:700], np.ones(d, dtype=bool)),
    ]


def _expect(X, rows, mask):
    Y = X if rows is None else X[rows]
    return Y if mask is None else Y[:, np.nonzero(mask)[0]]


def _assert_same(got, ref, what):
    assert got.shape == ref.shape, what
    np.testing.assert_array_equal(got.indptr.cpu().numpy(), ref.indptr.astype(np.int64), err_msg=what)
    np.testing.assert_array_equal(got.indices.cpu().numpy(), ref.indices.astype(np.int32), err_msg=what)
    # byte for byte: explicit zeros and signed zeros included
    assert got.data.cpu().numpy().tobytes() == ref.data.astype(np.float32).tobytes(), what


def test_select_matches_scipy(cuda):
    X = _source()
    A = mu.DeviceCSR.from_scipy(X)
    for what, rows, mask in _cases(*X.shape):
        _assert_same(_device.csr_select(A, rows, mask), _expect(X, rows, mask), what)
    # bad arguments: a status with a message, never a launch
    with pytest.raises(IndexError):
        _device.csr_select(A, np.array([0, X.shape[0]]))
    with pytest.raises(IndexError):
        _device.csr_select(A, np.array([-1]))
    with pytest.raises(ValueError):
        _device.csr_select(A, None, np.ones(7, dtype=bool))
    with pytest.raises(MuonB200Error, match="n_rows_out must equal"):
        mu._lib.call("mub_csr_select_count", mu._lib.ptr(A.indptr), mu._lib.ptr(A.indices), X.shape[0], X.shape[1], None,
                     5, None, mu._lib.ptr(A.indptr), mu._lib.stream_ptr())


def test_select_with_offsets_beyond_2_31(cuda):
    """the same inputs stored at the end of index / value arrays longer than 2^31 entries, poisoned below the base"""
    X = _source(seed=2)
    C = mu.DeviceCSR.from_scipy(X)
    base = (1 << 31) + 12_345_678
    big_idx = torch.empty(base + C.nnz, dtype=torch.int32, device=cuda)
    big_val = torch.empty(base + C.nnz, dtype=torch.float32, device=cuda)
    big_idx[:base].fill_(-1)
    big_val[:base].fill_(float("nan"))
    big_idx[base:] = C.indices
    big_val[base:] = C.data
    A = mu.DeviceCSR(C.indptr + base, big_idx, big_val, X.shape)
    for what, rows, mask in _cases(*X.shape):
        got = _device.csr_select(A, rows, mask)
        _assert_same(got, _expect(X, rows, mask), what + " (offsets beyond 2^31)")
        assert got.shape[0] == 0 or got.shape[1] == 0 or "rb_counts" in got._aux
    del A, big_idx, big_val
    torch.cuda.empty_cache()


# ---- 2. zero copy and the counts of the deterministic fill ---------------------------------------------------------
def test_slices_share_storage_and_every_block_fills_tiled(cuda):
    X = _source(seed=3)
    A = mu.DeviceCSR.from_scipy(X)
    rng = np.random.default_rng(0)
    sl = _device.csr_select(A, np.arange(512, 1400))
    assert sl.data.untyped_storage().data_ptr() == A.data.untyped_storage().data_ptr()
    assert sl.indices.untyped_storage().data_ptr() == A.indices.untyped_storage().data_ptr()
    assert int(sl.indptr[0]) == 0 and sl.nnz == X[512:1400].nnz
    whole = _device.csr_select(A)
    assert whole.data.untyped_storage().data_ptr() == A.data.untyped_storage().data_ptr()
    gathered = _device.csr_select(A, rng.permutation(X.shape[0])[:1000])
    masked = _device.csr_select(A, np.arange(0, 1000), rng.random(X.shape[1]) < 0.5)
    assert gathered.data.untyped_storage().data_ptr() != A.data.untyped_storage().data_ptr()
    for B in (sl, whole, gathered, masked):
        P = B.transpose_panels(64)
        assert P.tiled_fill is True
        # the panels equal scipy's transpose
        T = B.get().T.tocsr()
        T.sort_indices()
        got = sp.csr_matrix((P.panels[0][2].data.cpu().numpy(), P.panels[0][2].indices.cpu().numpy(),
                             P.panels[0][2].indptr.cpu().numpy()), shape=T.shape)
        np.testing.assert_array_equal(got.indptr, T.indptr)
        np.testing.assert_array_equal(got.indices, T.indices)
        np.testing.assert_array_equal(got.data, T.data)
    # an unsorted row: no counts, the atomic-cursor fill as before
    Xu = X.copy()
    r = int(np.nonzero(np.diff(Xu.indptr) > 3)[0][0])
    k0 = Xu.indptr[r]
    Xu.indices[k0], Xu.indices[k0 + 1] = Xu.indices[k0 + 1], Xu.indices[k0]
    U = _device.csr_select(mu.DeviceCSR.from_scipy(Xu), np.arange(0, 1200))
    assert "rb_counts" not in (getattr(U, "_aux", None) or {}) and U.transpose_panels(64).tiled_fill is False


# ---- 3. parity with the float64 oracle ------------------------------------------------------------------------------
def _planted(N, dims, K, seed, noise=0.5):
    rng = np.random.default_rng(seed)
    Z = rng.normal(size=(N, K))
    views = []
    for D in dims:
        W = rng.normal(size=(D, K)) * (rng.random((D, K)) < 0.5)
        Y = Z @ W.T + noise * rng.normal(size=(N, D)) - 1.0
        views.append(sp.csr_matrix(np.maximum(Y, 0).astype(np.float32)))
    return views


def _z0_for_oracle(groups, K, seed):
    """mofa() draws Z0 in its cell order (cells ordered by group); the oracle keeps the input order"""
    names = list(dict.fromkeys(groups.tolist()))
    perm = np.argsort(np.array([names.index(g) for g in groups]), kind="stable")
    Z0 = np.empty((len(groups), K))
    Z0[perm] = np.random.RandomState(seed).normal(size=(len(groups), K))
    return Z0


def _union_case(groups, hv=None):
    N, dims = 300, [140, 90]
    views = _planted(N, dims, 3, seed=11)
    names = [f"c{i}" for i in range(N)]
    a = SimpleAnnData(mu.DeviceCSR.from_scipy(views[0][:270]), obs=names[:270])
    b = SimpleAnnData(mu.DeviceCSR.from_scipy(views[1][30:]), obs=names[30:])
    if hv is not None:
        a.var["highly_variable"], b.var["highly_variable"] = hv
    md = SimpleMuData({"rna": a, "atac": b})
    md.obs["grp"] = groups
    Y1 = np.full((N, dims[0]), np.nan)
    Y1[:270] = views[0][:270].toarray()
    Y2 = np.full((N, dims[1]), np.nan)
    Y2[30:] = views[1][30:].toarray()
    if hv is not None:
        Y1, Y2 = Y1[:, hv[0]], Y2[:, hv[1]]
    return md, [Y1, Y2]


CONTIGUOUS = np.array(["g1"] * 120 + ["g2"] * 180)
INTERLEAVED = np.array(["g1", "g2", "g2"] * 100)
HV = (np.arange(140) % 4 != 1, np.arange(90) % 3 != 0)


@pytest.mark.parametrize("layout", ["contiguous", "interleaved", "use_var"])
def test_device_views_match_general_oracle(cuda, layout):
    """test_gpu_mofa.py::test_groups_and_union_match_general_oracle with DeviceCSR views"""
    groups = INTERLEAVED if layout == "interleaved" else CONTIGUOUS
    hv = HV if layout == "use_var" else None
    K = 5
    for kw in ({}, {"scale_groups": True}):
        md, Ys = _union_case(groups, hv)
        mu.tl.mofa(md, use_var="highly_variable" if hv else None, n_factors=K, n_iterations=20,
                   convergence_mode="slow", use_obs="union", groups_label="grp", seed=3, **kw)
        want = {"contiguous": "slice", "interleaved": "gather", "use_var": "gather"}[layout]
        assert md.uns["mofa"]["_b200"]["blocks"] == {"rna": [want] * 2, "atac": [want] * 2}
        ref = mofa_ref_general(Ys, groups=groups, n_factors=K, n_iterations=20, convergence_mode="slow", seed=3,
                               Z0=_z0_for_oracle(groups, K, 3), **kw)
        np.testing.assert_allclose(md.uns["mofa"]["_b200"]["elbo"], ref["elbo"], rtol=1e-5)
        Zg, Zr = md.obsm["X_mofa"], ref["Z"]
        act = np.sum([v.sum(0) for v in ref["variance"]], axis=0) > 2.0
        assert act.sum() >= 2
        assert (np.abs(Zg - Zr).max(0) / np.abs(Zr).max(0))[act].max() < 2e-4
        Wr = np.concatenate(ref["W"], axis=0)
        lfs = md.varm["LFs"]
        if hv is not None:
            keep = np.concatenate(hv)
            assert np.all(lfs[~keep] == 0)
            lfs = lfs[keep]
        assert (np.abs(lfs - Wr).max(0) / np.abs(Wr).max(0))[act].max() < 2e-4
        assert set(md.uns["mofa"]["variance"]["rna"]) == {"g1", "g2"}
        np.testing.assert_allclose(md.uns["mofa"]["variance"]["atac"]["g2"][act], ref["variance"][1][1][act], rtol=2e-3)


def _count_views(N, seed):
    rng = np.random.default_rng(seed)
    Z = rng.normal(size=(N, 3))
    W1 = rng.normal(size=(70, 3)) * (rng.random((70, 3)) < 0.5)
    W2 = rng.normal(size=(45, 3)) * (rng.random((45, 3)) < 0.5)
    W3 = rng.normal(size=(30, 3))
    Yp = rng.poisson(np.log1p(np.exp(Z @ W1.T + 0.5))).astype(np.float64)
    Yb = (rng.random((N, 45)) < 1 / (1 + np.exp(-(Z @ W2.T)))).astype(np.float64)
    Yg = Z @ W3.T + rng.normal(size=(N, 30))
    return Yp, Yb, Yg


def test_sparse_pseudo_device_views_match_oracle(cuda, monkeypatch):
    """poisson + bernoulli + gaussian device views, interleaved groups, non-gaussian views kept sparse"""
    monkeypatch.setenv("MUON_B200_MOFA_PSEUDO", "sparse")
    N, K = 400, 5
    Yp, Yb, Yg = _count_views(N, 0)
    dv = lambda Y: SimpleAnnData(mu.DeviceCSR.from_scipy(sp.csr_matrix(Y.astype(np.float32))))   # noqa: E731
    md = SimpleMuData({"counts": dv(Yp), "binary": dv(Yb), "cont": dv(Yg)})
    grp = np.array(["a", "b"] * 200)
    md.obs["grp"] = grp
    mu.tl.mofa(md, use_var=None, n_factors=K, n_iterations=15, convergence_mode="slow", groups_label="grp", seed=2)
    assert list(md.uns["mofa"]["params"]["data"]["likelihoods"]) == ["poisson", "bernoulli", "gaussian"]
    assert md.uns["mofa"]["_b200"]["pseudo"] == {"counts": "sparse", "binary": "sparse"}
    assert md.uns["mofa"]["_b200"]["blocks"]["counts"] == ["gather", "gather"]
    ref = mofa_ref_general([Yp, Yb, Yg], groups=grp, n_factors=K, n_iterations=15, convergence_mode="slow", seed=2,
                           likelihoods=["poisson", "bernoulli", "gaussian"], Z0=_z0_for_oracle(grp, K, 2))
    np.testing.assert_allclose(md.uns["mofa"]["_b200"]["elbo"], ref["elbo"], rtol=2e-5)
    act = np.sum([v.sum(0) for v in ref["variance"]], axis=0) > 2.0
    assert act.sum() >= 2
    Zg, Zr = md.obsm["X_mofa"], ref["Z"]
    assert (np.abs(Zg - Zr).max(0) / np.abs(Zr).max(0))[act].max() < 5e-4
    Wr = np.concatenate(ref["W"], axis=0)
    assert (np.abs(md.varm["LFs"] - Wr).max(0) / np.abs(Wr).max(0))[act].max() < 5e-4


def test_likelihood_guess_looks_at_kept_features_only(cuda):
    """a count view whose non-integer values all sit in features outside use_var is guessed poisson, as on the host"""
    Yp, _, _ = _count_views(200, 4)
    Y = Yp.astype(np.float32)
    Y[:, :5] += 0.5
    hv = np.arange(Y.shape[1]) >= 5
    outs = []
    for X in (sp.csr_matrix(Y), mu.DeviceCSR.from_scipy(sp.csr_matrix(Y))):
        ad = SimpleAnnData(X)
        ad.var["highly_variable"] = hv
        md = SimpleMuData({"counts": ad})
        mu.tl.mofa(md, n_factors=3, n_iterations=3)
        outs.append(list(md.uns["mofa"]["params"]["data"]["likelihoods"]))
        assert np.all(md.varm["LFs"][:5] == 0)
    assert outs == [["poisson"], ["poisson"]]


# ---- 4. reproducibility and 5. the plan and its memory ---------------------------------------------------------------
def test_grouped_device_fit_is_bit_reproducible_and_copies_once(cuda, monkeypatch):
    made = []
    orig = _device.csr_select

    def spy(A, rows=None, col_mask=None):
        out = orig(A, rows, col_mask)
        made.append((A, col_mask, out))
        return out

    monkeypatch.setattr(_device, "csr_select", spy)
    runs = []
    for _ in range(2):
        made.clear()
        md, _ = _union_case(INTERLEAVED, HV)
        mu.tl.mofa(md, n_factors=5, n_iterations=10, convergence_mode="slow", use_obs="union", groups_label="grp",
                   seed=3)
        runs.append(md)
        assert md.uns["mofa"]["_b200"]["blocks"] == {"rna": ["gather"] * 2, "atac": ["gather"] * 2}
        # the gathers of a view together hold its kept entries exactly once
        for m, hv in zip(("rna", "atac"), HV):
            src = md.mod[m].X
            blocks = [out for A, _, out in made if A is src]
            assert len(blocks) == 2
            kept = int(torch.from_numpy(hv).to(cuda)[src.indices.long()].sum())
            assert sum(b.nnz for b in blocks) == kept
            assert all(b.transpose_panels(64).tiled_fill for b in blocks)
    a, b = runs
    assert np.array_equal(a.obsm["X_mofa"], b.obsm["X_mofa"], equal_nan=True)
    assert np.array_equal(a.varm["LFs"], b.varm["LFs"])
    assert a.uns["mofa"]["_b200"]["elbo"] == b.uns["mofa"]["_b200"]["elbo"]


# ---- 6. scale -------------------------------------------------------------------------------------------------------
def test_interleaved_masked_view_at_scale_matches_host_path(cuda):
    """150k x 120k at 1 %, 3 interleaved groups and a use_var mask: the device blocks fit as the host blocks do"""
    from muon_b200._synth import generate_device
    N, D, K = 150_000, 120_000, 10
    A = _device.tfidf_csr(generate_device(N, D, 0.01, seed=3), inplace_values=True)
    host = A.get()
    hv = np.random.default_rng(0).random(D) < 0.6
    grp = np.array(["a", "b", "c"])[np.arange(N) % 3]
    elbos = []
    for X in (A, host):
        ad = SimpleAnnData(X)
        ad.var["highly_variable"] = hv
        md = SimpleMuData({"atac": ad})
        md.obs["grp"] = grp
        mu.tl.mofa(md, n_factors=K, n_iterations=5, convergence_mode="slow", groups_label="grp", seed=1,
                   likelihoods="gaussian")
        elbos.append(md.uns["mofa"]["_b200"]["elbo"])
        kinds = md.uns["mofa"]["_b200"]["blocks"]["atac"]
        assert kinds == (["gather"] * 3 if X is A else ["host"] * 3)
        del md, ad
        torch.cuda.empty_cache()
    assert len(elbos[0]) == len(elbos[1]) == 5
    np.testing.assert_allclose(elbos[0], elbos[1], rtol=1e-5)


# ---- shard position, float64 views, unsorted sources ---------------------------------------------------------------
def test_selection_keeps_the_shard_position_and_unsorted_sources_get_no_counts(cuda):
    X = _source(seed=5)
    A = mu.DeviceCSR.from_scipy(X)
    A.row0, A._n_total = 4000, 9000                      # rows [4000, 5500) of a 9000-cell matrix sharded over ranks
    mask = np.arange(X.shape[1]) % 3 != 0
    for cm in (None, mask):
        out = _device.csr_select(A, None, cm)
        assert (out.row0, out.n_total) == (4000, 9000)
    part = _device.csr_select(A, np.arange(10, 20), mask)
    assert (part.row0, part.n_total) == (0, 10)
    # a shard not marked sorted gets no tiled reduce pass: no counts, the atomic-cursor fill
    U = mu.DeviceCSR(A.indptr, A.indices, A.data, A.shape, row0=A.row0, n_total=A._n_total, sorted_indices=False)
    plain = _device.csr_select(U, None, mask)
    assert "rb_counts" not in (getattr(plain, "_aux", None) or {}) and plain.transpose_panels(64).tiled_fill is False
    _assert_same(plain, _expect(X, None, mask), "unsorted source")


def test_use_var_on_a_cell_shard_fits_as_the_premasked_shard(cuda):
    """one-group mofa() on a device shard (row0 / n_total set) with use_var: the shard's place in the whole matrix
    decides its initial factors and the group's cell count, exactly as for the same shard masked beforehand"""
    X = _planted(300, [120], 3, seed=8)[0]
    hv = np.arange(120) % 4 != 2
    fits = []
    for src, use_var in ((X, "highly_variable"), (X[:, np.nonzero(hv)[0]].tocsr(), None)):
        A = mu.DeviceCSR.from_scipy(src)
        A.row0, A._n_total = 200, 1000
        ad = SimpleAnnData(A)
        if use_var:
            ad.var["highly_variable"] = hv
        md = SimpleMuData({"rna": ad})
        mu.tl.mofa(md, use_var=use_var, n_factors=4, n_iterations=12, convergence_mode="slow", seed=2,
                   likelihoods="gaussian")
        fits.append(md)
    masked, pre = fits
    assert masked.uns["mofa"]["_b200"]["blocks"] == {"rna": ["gather"]}
    np.testing.assert_allclose(masked.uns["mofa"]["_b200"]["elbo"], pre.uns["mofa"]["_b200"]["elbo"], rtol=1e-5)
    np.testing.assert_allclose(masked.obsm["X_mofa"], pre.obsm["X_mofa"], rtol=1e-4, atol=1e-5)
    np.testing.assert_allclose(masked.varm["LFs"][hv], pre.varm["LFs"], rtol=1e-4, atol=1e-5)


def test_float64_device_views_record_their_conversion(cuda):
    views = _planted(200, [60, 40], 3, seed=9)
    md = SimpleMuData({"rna": SimpleAnnData(mu.DeviceCSR.from_scipy(views[0], dtype=np.float64)),
                       "atac": SimpleAnnData(mu.DeviceCSR.from_scipy(views[1]))})
    mu.tl.mofa(md, use_var=None, n_factors=3, n_iterations=3, likelihoods="gaussian")
    assert md.uns["mofa"]["_b200"]["blocks"] == {"rna": ["convert+slice"], "atac": ["slice"]}
    md.obs["grp"] = np.array(["a", "b"] * 100)
    mu.tl.mofa(md, use_var=None, n_factors=3, n_iterations=3, likelihoods="gaussian", groups_label="grp")
    assert md.uns["mofa"]["_b200"]["blocks"] == {"rna": ["convert+gather"] * 2, "atac": ["gather"] * 2}
