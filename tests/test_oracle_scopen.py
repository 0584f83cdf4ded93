"""CPU: the float64 scOpen restatement (oracle/scopen_ref.py) against sklearn's coordinate-descent NMF and NNDSVD, the
reference run through its ``scopen.MF`` stand-in, and the fixtures (tests/golden/scopen_small.npz)."""
import contextlib
import io
import warnings

import numpy as np
import pytest

from muon_b200 import SimpleAnnData, SimpleMuData
from muon_b200 import _scopen
from conftest import load_golden
from oracle import scopen_ref as R
from oracle._refload import reference_available
from scopen_cases import CASES, arguments, matrix, sample_rows

DEFAULTS = {"n_components": 30, "max_iter": 500, "min_rho": 0.0, "max_rho": 0.5, "alpha": 1}


@pytest.fixture(scope="module")
def golden():
    return load_golden("scopen_small.npz")


def kwargs(case):
    return {**DEFAULTS, **CASES[case][5]}


def pattern_matrix(case):
    X, _ = matrix(case)
    kw = kwargs(case)
    P, c = R.pattern_of(X)
    s = R.scale_of(c, kw["min_rho"], kw["max_rho"])
    return P, s


def test_golden_records_every_case(golden):
    assert list(golden["cases"]) == list(CASES)
    for case in CASES:
        kw = kwargs(case)
        assert golden[f"{case}_W0"].shape[1] == kw["n_components"]


@pytest.mark.parametrize("case", list(CASES))
def test_unbounded_restatement_is_sklearn(golden, case):
    from sklearn.decomposition import _nmf
    P, s = pattern_matrix(case)
    kw = kwargs(case)
    W0, H0 = golden[f"{case}_W0"], golden[f"{case}_H0"]
    a = float(kw["alpha"])
    Ws, Hs, n_sk = _nmf._fit_coordinate_descent(R.dense_of(P, s), W0.copy(), H0.copy(), tol=R.TOL,
                                                max_iter=kw["max_iter"], l2_reg_W=a, l2_reg_H=a)
    W, H, n_iter, _ = R.fit(R.PatternMatrix(P, s), W0, H0, a, kw["max_iter"], R.TOL, np.inf)
    assert n_iter == n_sk == int(golden[f"{case}_n_iter_inf"])
    assert np.abs(W - Ws).max() <= 1e-12 * np.abs(Ws).max()
    assert np.abs(H - Hs).max() <= 1e-12 * np.abs(Hs).max()
    np.testing.assert_array_equal(W, golden[f"{case}_W_inf"])


@pytest.mark.parametrize("case", ["csr_f32", "k1", "k30"])
def test_nndsvd_is_sklearns_given_the_same_svd(monkeypatch, case):
    from sklearn.decomposition import _nmf
    P, s = pattern_matrix(case)
    X = R.dense_of(P, s)
    k = kwargs(case)["n_components"]
    U, S, V = R.exact_svd(X, k)
    monkeypatch.setattr(_nmf, "_randomized_svd", lambda *a, **kw: (U, S, V))
    Wsk, Hsk = _nmf._initialize_nmf(X, k, init="nndsvd", eps=1e-6)
    for W, H in (R.nndsvd(U, S, V), _scopen.nndsvd(U, S, V)):
        assert np.abs(W - Wsk).max() <= 1e-12 * np.abs(Wsk).max()
        assert np.abs(H - Hsk).max() <= 1e-12 * np.abs(Hsk).max()
    # a joint sign flip of a triplet leaves NNDSVD unchanged
    f = np.where(np.arange(k) % 2 == 1, -1.0, 1.0)
    W2, H2 = _scopen.nndsvd(U * f, S, V * f[:, None])
    np.testing.assert_array_equal(W2, Wsk)
    np.testing.assert_array_equal(H2, Hsk)


def test_product_scale_and_pattern_match_the_restatement():
    for case in CASES:
        X, _ = matrix(case)
        kw = kwargs(case)
        P, c = R.pattern_of(X)
        src, counts = _scopen.host_pattern_source(X)
        np.testing.assert_array_equal(counts, c)
        np.testing.assert_array_equal(_scopen.scale_of(counts, kw["min_rho"], kw["max_rho"]),
                                      R.scale_of(c, kw["min_rho"], kw["max_rho"]))


@pytest.mark.parametrize("case", list(CASES))
def test_restatement_reproduces_the_fixture(golden, case):
    X, _ = matrix(case)
    r = R.scopen_ref(X, upper=1.0, init=(golden[f"{case}_W0"], golden[f"{case}_H0"]), **kwargs(case))
    assert r["n_iter"] == int(golden[f"{case}_n_iter"])
    np.testing.assert_array_equal(r["W"], golden[f"{case}_W"])
    np.testing.assert_array_equal(r["H"], golden[f"{case}_H"])
    np.testing.assert_array_equal(r["M"][sample_rows(r["M"].shape[0])], golden[f"{case}_M_rows"])
    gap = min(abs(x - R.TOL) for x in r["ratios"]) / R.TOL
    assert gap >= 1e-6
    assert r["H"].max() <= 1.0 and r["W"].max() <= 1.0


@pytest.mark.skipif(not reference_available(), reason="reference sources not available")
@pytest.mark.parametrize("case", ["csc_maxiter", "converges", "mudata", "dense_f64"])
def test_reference_through_stand_in_is_the_restatement(golden, case):
    ref = R.load_reference_scopen()
    data, ad, kw = arguments(case, (SimpleAnnData, SimpleMuData))
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf), warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        ref(data, **kw)
    X, _ = matrix(case)
    r = R.scopen_ref(X, upper=1.0, **kwargs(case))
    np.testing.assert_array_equal(ad.varm["scopen"], r["W"])
    np.testing.assert_array_equal(ad.obsm["X_scopen"], r["H"].T)
    np.testing.assert_array_equal(ad.X, r["M"].T)
    assert ad.X.flags.f_contiguous
    assert buf.getvalue().splitlines()[:3] == list(golden[f"{case}_lines"])
    assert [str(w.message) for w in rec] == list(golden[f"{case}_warnings"])
