"""H100: ``mu.tl.ica`` -- the unmodified reference's outputs (tests/golden/ica_small.npz), the warnings and slots of
the golden run, AnnData / MuData / ``copy``, bit-identical repeats, the generator left as sklearn leaves it, 128
features, and a 1M x 50 float32 fit against the float64 restatement (oracle/ica_ref.py)."""
import warnings

import numpy as np
import pytest

import muon_b200 as mu
from muon_b200 import SimpleAnnData, SimpleMuData
from muon_b200 import _ica
from muon_b200.prot.pp import ConvergenceWarning
from conftest import load_golden
from ica_cases import CASES, arguments, planted
from oracle.ica_ref import fastica_ref, match_sources
from test_oracle_ica import assert_columns_close, assert_matches_golden_rows, assert_matches_restatement, f32_rtol

pytestmark = pytest.mark.gpu


def _adata(X, key="X_pca"):
    a = SimpleAnnData(np.zeros((X.shape[0], 1)))
    a.obsm[key] = X
    return a


@pytest.fixture(scope="module")
def golden():
    return load_golden("ica_small.npz")


@pytest.mark.parametrize("case", list(CASES))
def test_golden_cases(cuda, golden, case):
    z = golden
    X, _, rs, scale, kw = arguments(case)
    ad = _adata(X)
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        res, info = mu.tl.ica(ad, random_state=rs, scale=scale, return_info=True, **kw)
    assert res is None
    got = ad.obsm["X_ica"]
    assert info["n_iter"] == int(z[f"{case}_n_iter"])
    assert [str(w.message) for w in rec] == list(z[f"{case}_warnings"])
    conv = [w for w in rec if "did not converge" in str(w.message)]
    assert all(issubclass(w.category, ConvergenceWarning) for w in conv)
    rtol = 1e-8 if got.dtype == np.float64 else f32_rtol(z, case)
    assert_matches_golden_rows(got, z, case, rtol)
    assert_matches_restatement(got, case)
    for key in ("components", "mixing", "unmixing", "mean", "whitening"):
        if f"{case}_{key}" in z:
            assert info[key].dtype == got.dtype
            assert_columns_close(info[key], z[f"{case}_{key}"], rtol, key)
        else:
            assert info[key] is None


def test_mudata_copy_and_integer_input(cuda, golden):
    X, _, rs, scale, kw = arguments("p7_par_exp")
    md = SimpleMuData({"a": _adata(X)})
    md.obsm["X_mofa"] = X
    out = mu.tl.ica(md, basis="X_mofa", random_state=rs, copy=True, **kw)
    assert "X_ica" not in md.obsm and "X_ica" in out.obsm
    assert_matches_golden_rows(out.obsm["X_ica"], golden, "p7_par_exp", 1e-8)
    Xi = np.round(X * 100).astype(np.int32)
    a, b = _adata(Xi), _adata(Xi.astype(np.float64))
    mu.tl.ica(a, random_state=3)
    mu.tl.ica(b, random_state=3)
    assert a.obsm["X_ica"].dtype == np.float64 and np.array_equal(a.obsm["X_ica"], b.obsm["X_ica"])


@pytest.mark.parametrize("case", ["p7_par_exp", "p7_def_logcosh_a15", "f32_p50_def_k5_scale"])
def test_two_calls_bit_identical(cuda, case):
    outs = []
    for _ in range(2):
        X, _, rs, scale, kw = arguments(case)
        ad = _adata(X)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            mu.tl.ica(ad, random_state=rs, scale=scale, **kw)
        outs.append(ad.obsm["X_ica"])
    assert outs[0].tobytes() == outs[1].tobytes()


def test_generator_left_in_sklearn_state(cuda):
    X, _, _, _, _ = arguments("p7_par_cube")
    rs = np.random.RandomState(5)
    mu.tl.ica(_adata(X), n_components=4, random_state=rs)
    ref = np.random.RandomState(5)
    ref.normal(size=(4, 4))
    assert rs.randint(1 << 30) == ref.randint(1 << 30)
    np.random.seed(11)
    mu.tl.ica(_adata(X), algorithm="deflation")
    np.random.seed(11)
    np.random.normal(size=(7, 7))
    expect = np.random.randint(1 << 30)
    np.random.seed(11)
    mu.tl.ica(_adata(X), algorithm="deflation")
    assert np.random.randint(1 << 30) == expect


def test_128_features(cuda):
    X, S = planted(6001, 128, 40, np.float64)
    ad = _adata(X)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        _, info = mu.tl.ica(ad, random_state=0, max_iter=4, tol=0.0, return_info=True)
    ref = fastica_ref(X, random_state=0, max_iter=4, tol=0.0)
    assert info["n_iter"] == ref["n_iter"] == 4
    assert_columns_close(ad.obsm["X_ica"], ref["sources"], 1e-8, "X_ica")
    assert_columns_close(info["unmixing"], ref["unmixing"], 1e-8, "unmixing")
    with pytest.raises(NotImplementedError):
        mu.tl.ica(_adata(np.hstack([X, X[:, :1]])))


def test_million_cells(cuda, monkeypatch):
    # 50 planted sources: every direction is fixed by the contrast, so rounding does not grow over the iterations
    X, _ = planted(1_000_001, 50, 41, np.float32)
    ad = _adata(X)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        _, info = mu.tl.ica(ad, random_state=1, max_iter=5, tol=0.0, return_info=True)
        # the "svd" whitening here is the Gram route, which the restatement's "eigh" solver takes in numpy (no
        # eigenvalue is near its clamp); against LAPACK's SVD the two agree to float64 rounding x cond(X)^2
        ref = fastica_ref(X, random_state=1, max_iter=5, tol=0.0, whiten_solver="eigh")
    assert info["n_iter"] == 5
    err = np.max(np.abs(info["unmixing"].astype(np.float64) - ref["unmixing"])) / np.max(np.abs(ref["unmixing"]))
    assert err <= 1e-6, err          # info is rounded to float32; the float64 W is checked below
    W64 = _unmixing_f64(monkeypatch, X, random_state=1, max_iter=5, tol=0.0)
    err = np.max(np.abs(W64 - ref["unmixing"])) / np.max(np.abs(ref["unmixing"]))
    # the sums over a million cells run in another order than numpy's; the first steps from a random start amplify
    # that difference to 1.6e-9 on an H100
    assert err <= 1e-8, err
    # 10 planted sources in the leading subspace, weak Gaussian noise in the other 40 features
    X, S = planted(1_000_001, 50, 41, np.float32, m=10)
    ad = _adata(X)
    with warnings.catch_warnings():
        warnings.simplefilter("error", ConvergenceWarning)
        _, info = mu.tl.ica(ad, n_components=10, random_state=2, return_info=True)
    assert info["n_iter"] < 200
    assert match_sources(ad.obsm["X_ica"].astype(np.float64), S) >= 0.99


def _unmixing_f64(monkeypatch, X, **kw):
    """W after the unit-variance rescale in float64 (``info`` holds it rounded to the input dtype), captured from
    the std pass of the same fit."""
    captured = {}
    orig = _ica._Device.sources

    def sources(self, M, d1=None, d2=None, stats=False):
        out = orig(self, M, d1, d2, stats)
        if stats and d1 is None:
            captured["W"] = M * np.sqrt(self.n) / out[1][:, None]
        return out
    with monkeypatch.context() as m:
        m.setattr(_ica._Device, "sources", sources)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            _ica.fit_transform(X, **kw)
    return captured["W"]
