"""GPU: poisson / bernoulli MOFA views kept sparse (csrc/mofa_lowrank.cu) -- the kernels against a float64 evaluation
of the same formulas, the fit against the float64 oracle, and a view too large for the dense pseudo-data."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

import muon_b200 as mu
from muon_b200 import _device
from muon_b200._containers import SimpleAnnData, SimpleMuData
from muon_b200._lib import call, ptr, stream_ptr
from muon_b200._mofa import _check_dense_fits, _SparsePseudoBlock
from oracle.mofa_ref import mofa_ref_general

pytestmark = pytest.mark.gpu
f64 = torch.float64
TOL = 3e-5


def _ref_terms(Zz, Wz, y_dense, kappa, kind):
    """float64: g over all elements, s at the stored entries (0 elsewhere), ln p dense part and stored part"""
    z = Zz.to(f64) @ Wz.to(f64).T
    k = kappa.to(f64)[None, :]
    sig = torch.sigmoid(z)
    spl = torch.where(z > 20, z, torch.log1p(torch.exp(z)))
    r = spl.clamp_min(1e-30)
    g = z - sig / k
    s = y_dense * sig / (k * r) if kind == 1 else y_dense / k
    ll_dense = -r if kind == 1 else -spl
    ll_nnz = y_dense * torch.log(r) if kind == 1 else y_dense * z
    return z, g, s, ll_dense, ll_nnz


def _close(got, ref, scale, what):
    err = (got.to(f64) - ref).abs()
    bad = err > TOL * scale + 1e-30
    assert not bool(bad.any()), f"{what}: max err / scale = {float((err / (scale + 1e-300)).max()):.3g}"


def _problem(n, D, K, kind, seed, dev):
    g = torch.Generator(device="cpu").manual_seed(seed)
    ld = _device.pad_width(K)
    Z = torch.zeros((n, ld))
    W = torch.zeros((D, ld))
    Z[:, :K] = torch.randn((n, K), generator=g)
    W[:, :K] = torch.randn((D, K), generator=g) / np.sqrt(K)
    Z[: n // 20] *= 30.0                                   # pushes |zeta| past 20 for some cells
    mask = torch.rand((n, D), generator=g) < 0.05
    y = torch.where(mask, torch.randint(1, 6, (n, D), generator=g).float(), torch.zeros(()))
    if kind == 2:
        y = (y > 0).float()
    mx = y.max(0).values
    kappa = 0.25 + 0.17 * mx if kind == 1 else torch.full((D,), 0.25)
    kappa = kappa * (1.0 + torch.rand(D, generator=g))      # per-column precisions, not all equal
    A = _device.DeviceCSR.from_scipy(sp.csr_matrix(y.numpy()), dtype=np.float32)
    return ld, Z.to(dev).contiguous(), W.to(dev).contiguous(), y.to(dev).to(f64), kappa.to(dev).contiguous(), A


@pytest.mark.parametrize("kind", [1, 2])
@pytest.mark.parametrize("K", [1, 5, 30, 64])
@pytest.mark.parametrize("shape", [(1000, 777), (3001, 2049)])
def test_lowrank_kernels_match_float64(cuda, shape, K, kind):
    n, D = shape
    ld, Z, W, y, kappa, A = _problem(n, D, K, kind, seed=n + K + kind, dev=cuda)
    zeta, g, s, lld, lln = _ref_terms(Z, W, y, kappa, kind)
    assert bool((zeta.abs() > 20).any())
    st = stream_ptr()
    B = torch.zeros((D, ld), device=cuda)
    B[:, :K] = torch.randn((D, K), device=cuda)
    Bd = B.to(f64)
    # row sweep: g B, accumulated onto what out held
    out = torch.ones((n, ld), device=cuda)
    call("mub_mofa_lowrank_rows_f32", ptr(Z), n, ptr(W), D, ptr(kappa), ptr(B), ld, kind, ptr(out), 1, None, st)
    _close(out - 1.0, g @ Bd, g.abs() @ Bd.abs(), "g B")
    # column sweep: g^T Z and sum g^2
    P = torch.empty((D, ld), device=cuda)
    ssq = torch.empty(D, dtype=f64, device=cuda)
    call("mub_mofa_lowrank_cols_f32", ptr(Z), n, ptr(W), D, ptr(kappa), ptr(Z), ld, kind, ptr(P), ptr(ssq), st)
    Zd = Z.to(f64)
    _close(P, g.T @ Zd, g.abs().T @ Zd.abs(), "g^T Z")
    _close(ssq, (g * g).sum(0), (g * g).sum(0), "sum g^2")
    # log-likelihood, dense part
    acc = torch.zeros(1, dtype=f64, device=cuda)
    call("mub_mofa_lowrank_rows_f32", ptr(Z), n, ptr(W), D, None, None, ld, kind, None, 0, ptr(acc), st)
    _close(acc, lld.sum()[None], lld.abs().sum()[None], "dense ln p")
    # corrections at the stored entries, CSR: S B and the stored part of ln p
    Q = torch.zeros((n, ld), device=cuda)
    call("mub_mofa_nnz_rows_f32", ptr(A.indptr), ptr(A.indices), ptr(A.data), n, ptr(Z), ptr(W), ptr(kappa), ptr(B),
         ld, kind, ptr(Q), None, st)
    _close(Q, s @ Bd, s.abs() @ Bd.abs(), "S B")
    acc.zero_()
    call("mub_mofa_nnz_rows_f32", ptr(A.indptr), ptr(A.indices), ptr(A.data), n, ptr(Z), ptr(W), None, None, ld, kind,
         None, ptr(acc), st)
    _close(acc, lln.sum()[None], lln.abs().sum()[None], "stored ln p")
    # corrections, transposed pairs panels: S^T Z and the cross terms of sum yhat^2
    Pc, sq = torch.zeros((D, ld), device=cuda), torch.zeros(D, dtype=f64, device=cuda)
    At = A.transpose_panels(ld)
    for r0, _, T in At.panels:
        call("mub_mofa_nnz_cols_f32", ptr(T.indptr), ptr(T.pairs), D, ptr(Z) + 4 * ld * r0, ptr(W), ptr(kappa),
             ptr(Z) + 4 * ld * r0, ld, kind, ptr(Pc), ptr(sq), st)
    _close(Pc, s.T @ Zd, s.abs().T @ Zd.abs(), "S^T Z")
    cross = 2 * g * s + s * s
    _close(sq, cross.sum(0), (2 * (g * s).abs() + s * s).sum(0), "cross terms")
    # the padded columns stay zero
    assert bool((out[:, K:] == 1.0).all()) and bool((P[:, K:] == 0).all()) and bool((Pc[:, K:] == 0).all())


def test_block_contractions_are_deterministic_and_exact(cuda):
    """_SparsePseudoBlock: P = Yhat^T Z, ssq and Q = Yhat B equal the float64 pseudo-data's, bit-identical on a rerun"""
    n, D, K = 3001, 2049, 30
    for kind in (1, 2):
        ld, Z, W, y, kappa, A = _problem(n, D, K, kind, seed=11 + kind, dev=cuda)
        _, g, s, _, _ = _ref_terms(Z, W, y, kappa, kind)
        yhat = g + s
        b = _SparsePseudoBlock(A, None, 0, n, ld, kind)
        tw = torch.zeros((D, ld), device=cuda)
        tw[:, :K] = torch.randn((D, K), device=cuda)
        runs = []
        for _ in range(2):
            P, ssq = b.pseudo(Z, W, kappa, K)
            Q = torch.zeros((n, ld), device=cuda)
            b.add_av(Q, tw)
            runs.append((P.clone(), ssq.clone(), Q))
        for x, x2 in zip(runs[0], runs[1]):
            assert torch.equal(x, x2)
        P, ssq, Q = runs[0]
        Zd, Td = Z.to(f64), tw.to(f64)
        _close(P, yhat.T @ Zd, (g.abs() + s.abs()).T @ Zd.abs(), "Yhat^T Z")
        _close(ssq, (yhat * yhat).sum(0), (g * g + 2 * (g * s).abs() + s * s).sum(0), "sum Yhat^2")
        _close(Q, yhat @ Td, (g.abs() + s.abs()) @ Td.abs(), "Yhat tw")
        # an empty block is a no-op for every kernel
        E = _device.DeviceCSR.from_scipy(sp.csr_matrix((0, D), dtype=np.float32))
        call("mub_mofa_lowrank_cols_f32", ptr(Z), 0, ptr(W), D, ptr(kappa), ptr(Z), ld, kind, ptr(P), ptr(ssq), stream_ptr())
        call("mub_mofa_nnz_rows_f32", ptr(E.indptr), ptr(E.indices), ptr(E.data), 0, ptr(Z), ptr(W), ptr(kappa), ptr(tw),
             ld, kind, ptr(Q), None, stream_ptr())
        assert torch.equal(P, runs[1][0]) and torch.equal(Q, runs[1][2])


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


def _assert_matches(md, ref, act_min=2):
    np.testing.assert_allclose(md.uns["mofa"]["_b200"]["elbo"], ref["elbo"], rtol=2e-5)
    act = np.sum([v.sum(0) for v in ref["variance"]], axis=0) > 2.0
    assert act.sum() >= act_min
    Zg, Zr = md.obsm["X_mofa"], ref["Z"]
    assert (np.abs(Zg - Zr).max(0) / np.abs(Zr).max(0))[act].max() < 5e-4
    Wr = np.concatenate(ref["W"], axis=0)
    assert (np.abs(md.varm["LFs"] - Wr).max(0) / np.abs(Wr).max(0))[act].max() < 5e-4


def test_sparse_views_match_oracle(cuda, monkeypatch):
    """the three cases of the dense-view oracle test, with the non-gaussian views kept sparse"""
    monkeypatch.setenv("MUON_B200_MOFA_PSEUDO", "sparse")
    N, K, T = 400, 5, 25
    Yp, Yb, Yg = _count_views(N, 0)
    # guessed likelihoods (the binary view is a dense host array: converted to CSR on the host)
    md = SimpleMuData({"counts": SimpleAnnData(sp.csr_matrix(Yp)), "binary": SimpleAnnData(Yb), "cont": SimpleAnnData(Yg)})
    mu.tl.mofa(md, use_var=None, n_factors=K, n_iterations=T, convergence_mode="slow", seed=5)
    assert list(md.uns["mofa"]["params"]["data"]["likelihoods"]) == ["poisson", "bernoulli", "gaussian"]
    assert md.uns["mofa"]["_b200"]["pseudo"] == {"counts": "sparse", "binary": "sparse"}
    ref = mofa_ref_general([Yp, Yb, Yg], n_factors=K, n_iterations=T, convergence_mode="slow", seed=5,
                           likelihoods=["poisson", "bernoulli", "gaussian"])
    assert len(md.uns["mofa"]["_b200"]["elbo"]) == len(ref["elbo"])
    _assert_matches(md, ref)
    # explicit likelihoods
    md1 = SimpleMuData({"counts": SimpleAnnData(sp.csr_matrix(Yp)), "binary": SimpleAnnData(sp.csr_matrix(Yb))})
    mu.tl.mofa(md1, use_var=None, n_factors=K, n_iterations=T, convergence_mode="slow", seed=3,
               likelihoods=["poisson", "bernoulli"])
    ref1 = mofa_ref_general([Yp, Yb], n_factors=K, n_iterations=T, convergence_mode="slow", seed=3,
                            likelihoods=["poisson", "bernoulli"])
    np.testing.assert_allclose(md1.uns["mofa"]["_b200"]["elbo"], ref1["elbo"], rtol=2e-5)
    # groups + poisson through the general path
    md3 = SimpleMuData({"counts": SimpleAnnData(sp.csr_matrix(Yp)), "cont": SimpleAnnData(Yg)})
    grp = np.array(["a"] * 150 + ["b"] * 250)
    md3.obs["grp"] = grp
    mu.tl.mofa(md3, use_var=None, n_factors=K, n_iterations=15, convergence_mode="slow", groups_label="grp", seed=2)
    assert md3.uns["mofa"]["_b200"]["pseudo"] == {"counts": "sparse"}
    ref3 = mofa_ref_general([Yp, Yg], groups=grp, n_factors=K, n_iterations=15, convergence_mode="slow", seed=2,
                            likelihoods=["poisson", "gaussian"])
    np.testing.assert_allclose(md3.uns["mofa"]["_b200"]["elbo"], ref3["elbo"], rtol=2e-5)


def _fit(monkeypatch, mode, make, **kw):
    monkeypatch.setenv("MUON_B200_MOFA_PSEUDO", mode)
    md = make()
    mu.tl.mofa(md, use_var=None, n_factors=5, n_iterations=20, convergence_mode="slow", seed=4, **kw)
    return md


def test_union_and_device_views_match_dense_path(cuda, monkeypatch):
    """use_obs='union' with a poisson view missing cells, and a device-resident bernoulli view: the sparse path gives
    the dense path's fit (which the oracle test pins), and the DeviceCSR view is not densified"""
    Yp, Yb, Yg = _count_views(300, 1)

    def union():
        return SimpleMuData({"counts": SimpleAnnData(sp.csr_matrix(Yp))[:-40], "cont": SimpleAnnData(Yg)[25:]})

    dense = _fit(monkeypatch, "dense", union, use_obs="union")
    sparse = _fit(monkeypatch, "sparse", union, use_obs="union")
    assert dense.uns["mofa"]["_b200"]["pseudo"] == {"counts": "dense"}
    assert sparse.uns["mofa"]["_b200"]["pseudo"] == {"counts": "sparse"}
    np.testing.assert_allclose(sparse.uns["mofa"]["_b200"]["elbo"], dense.uns["mofa"]["_b200"]["elbo"], rtol=2e-5)
    np.testing.assert_allclose(np.nan_to_num(sparse.obsm["X_mofa"]), np.nan_to_num(dense.obsm["X_mofa"]), atol=5e-4)
    # the variance explained reads Yhat^T Z, which the sparse path forms once after the last iteration
    np.testing.assert_allclose(sparse.uns["mofa"]["variance"]["counts"], dense.uns["mofa"]["variance"]["counts"],
                               rtol=1e-3, atol=1e-3)

    Xb = _device.DeviceCSR.from_scipy(sp.csr_matrix(Yb.astype(np.float32)))
    calls = []
    orig = _SparsePseudoBlock.__init__

    def spy(self, A, *a, **k):
        calls.append(A)
        orig(self, A, *a, **k)

    def device_view():
        return SimpleMuData({"binary": SimpleAnnData(Xb), "cont": SimpleAnnData(Yg)})

    dense = _fit(monkeypatch, "dense", device_view)
    monkeypatch.setattr(_SparsePseudoBlock, "__init__", spy)
    sparse = _fit(monkeypatch, "sparse", device_view)
    assert len(calls) == 1 and calls[0].data.data_ptr() == Xb.data.data_ptr()
    auto = _fit(monkeypatch, "auto", device_view)          # it fits: auto keeps the dense path
    assert auto.uns["mofa"]["_b200"]["pseudo"] == {"binary": "dense"}
    assert sparse.uns["mofa"]["_b200"]["pseudo"] == {"binary": "sparse"}
    np.testing.assert_allclose(sparse.uns["mofa"]["_b200"]["elbo"], dense.uns["mofa"]["_b200"]["elbo"], rtol=2e-5)
    np.testing.assert_allclose(auto.uns["mofa"]["_b200"]["elbo"], dense.uns["mofa"]["_b200"]["elbo"], rtol=1e-5)


def test_one_group_mofa_fits_the_model_run_mofa_device_fits(cuda, monkeypatch):
    """one-group mofa() on a gaussian and a bernoulli device view carrying entry counts, and run_mofa_device (what
    bench.py times) with the same likelihoods, the initial factors mofa() draws, its convergence check and its factor
    order: bit-identical fits"""
    from muon_b200._mofa import run_mofa_device
    from muon_b200._synth import generate_device
    monkeypatch.setenv("MUON_B200_MOFA_PSEUDO", "sparse")
    N, D, K, T, seed = 3000, 2000, 6, 15, 4
    Xg = _device.attach_block_counts(_device.tfidf_csr(generate_device(N, D, 0.02, seed=5)))
    Xb = _device.attach_block_counts(Xg.with_data(torch.ones_like(Xg.data)))
    assert all("rb_counts" in X._aux for X in (Xg, Xb))
    md = SimpleMuData({"cont": SimpleAnnData(Xg), "binary": SimpleAnnData(Xb)})
    mu.tl.mofa(md, use_var=None, likelihoods=["gaussian", "bernoulli"], n_factors=K, n_iterations=T, seed=seed)
    assert md.uns["mofa"]["_b200"]["pseudo"] == {"binary": "sparse"}
    assert md.uns["mofa"]["_b200"]["blocks"] == {"cont": ["slice"], "binary": ["slice"]}
    Z0 = np.random.RandomState(seed).normal(size=(Xg.n_total, K))[Xg.row0:Xg.row0 + N]
    res = run_mofa_device([Xg, Xb], K, T, Xg.n_total, torch.from_numpy(Z0), likelihoods=["gaussian", "bernoulli"],
                          check_convergence=True, sort_factors=True)
    assert md.uns["mofa"]["_b200"]["elbo"] == res["elbo"]
    assert np.array_equal(md.obsm["X_mofa"], res["Z"].cpu().numpy().astype(np.float64))
    assert np.array_equal(md.varm["LFs"], np.concatenate([W.cpu().numpy() for W in res["W"]]).astype(np.float64))


def test_views_too_large_for_dense_pseudo_data(cuda, monkeypatch):
    """150k x 120k poisson and bernoulli views at 1 %: dense pseudo-data would need 216 GB, the sparse path runs"""
    from muon_b200._synth import generate_device
    monkeypatch.setenv("MUON_B200_MOFA_PSEUDO", "auto")
    N, D, K = 150_000, 120_000, 10
    Xp = generate_device(N, D, 0.01, seed=3)
    Xb = Xp.with_data(torch.ones_like(Xp.data))
    with pytest.raises(NotImplementedError):
        _check_dense_fits("counts", (N, D), "poisson", cuda)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    md = SimpleMuData({"counts": SimpleAnnData(Xp), "binary": SimpleAnnData(Xb)})
    mu.tl.mofa(md, use_var=None, n_factors=K, n_iterations=5, convergence_mode="slow", seed=1,
               likelihoods=["poisson", "bernoulli"])
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated()
    nnz = Xp.nnz + Xb.nnz
    bound = 40 * nnz + 2048 * (N + 2 * D)
    print(f"peak {peak / 2**30:.2f} GiB for {nnz} stored entries (bound {bound / 2**30:.2f} GiB)")
    assert md.uns["mofa"]["_b200"]["pseudo"] == {"counts": "sparse", "binary": "sparse"}
    assert np.isfinite(md.uns["mofa"]["_b200"]["elbo"]).all()
    assert peak < bound
    # one _pseudo call's P rows for 256 features and one Q for 256 cells against float64
    ld = _device.pad_width(K)
    gen = torch.Generator(device="cpu").manual_seed(0)
    Z = torch.zeros((N, ld), device=cuda)
    W = torch.zeros((D, ld), device=cuda)
    Z[:, :K] = torch.randn((N, K), generator=gen).to(cuda)
    W[:, :K] = (torch.randn((D, K), generator=gen) / 3).to(cuda)
    feats = torch.randperm(D, generator=gen)[:256].to(cuda)
    cells = torch.randperm(N, generator=gen)[:256].to(cuda)
    rows = torch.repeat_interleave(torch.arange(N, device=cuda), Xp.indptr.diff())
    for kind, X in ((1, Xp), (2, Xb)):
        mx = torch.zeros(D, device=cuda).scatter_reduce_(0, X.indices.long(), X.data, "amax")
        kappa = (0.25 + 0.17 * mx if kind == 1 else torch.full((D,), 0.25, device=cuda)).contiguous()
        b = _SparsePseudoBlock(X, None, 0, N, ld, kind)
        P, _ = b.pseudo(Z, W, kappa, K)
        tw = torch.zeros((D, ld), device=cuda)
        tw[:, :K] = torch.randn((D, K), device=cuda)
        Q = torch.zeros((N, ld), device=cuda)
        b.add_av(Q, tw)
        # P rows: the feature columns of Y, dense over all cells
        sel = torch.isin(X.indices, feats.to(torch.int32))
        pos = torch.searchsorted(feats.sort().values, X.indices[sel].long())
        fs = feats.sort().values
        y = torch.zeros((N, 256), dtype=f64, device=cuda)
        y[rows[sel], pos] = X.data[sel].to(f64)
        _, g, s, _, _ = _ref_terms(Z, W[fs], y, kappa[fs], kind)
        Zd = Z.to(f64)
        _close(P[fs], (g + s).T @ Zd, (g.abs() + s.abs()).T @ Zd.abs(), f"P rows kind {kind}")
        # Q rows: the cells' rows of Y, dense over all features
        y = torch.zeros((256, D), dtype=f64, device=cuda)
        for i, c in enumerate(cells.tolist()):
            k0, k1 = int(X.indptr[c]), int(X.indptr[c + 1])
            y[i, X.indices[k0:k1].long()] = X.data[k0:k1].to(f64)
        _, g, s, _, _ = _ref_terms(Z[cells], W, y, kappa, kind)
        Td = tw.to(f64)
        _close(Q[cells], (g + s) @ Td, (g.abs() + s.abs()) @ Td.abs(), f"Q rows kind {kind}")
