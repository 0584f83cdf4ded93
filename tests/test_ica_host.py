"""CPU: the host side of ``mu.tl.ica`` with no device work -- the signature, every refusal and error, the warnings,
the ``random_state`` consumption, and the host logic end to end with the four device passes replaced by numpy."""
import inspect
import json
import os
import warnings

import numpy as np
import pytest
import scipy.sparse as sp

import muon_b200 as mu
from muon_b200 import SimpleAnnData, SimpleMuData
from muon_b200 import _ica
from muon_b200.prot.pp import ConvergenceWarning
from conftest import GOLDEN, load_golden
from ica_cases import CASES, arguments
from oracle.ica_ref import contrast
from test_oracle_ica import assert_columns_close, assert_matches_golden_rows, assert_matches_restatement, f32_rtol


class NumpyDevice:
    """The passes of csrc/ica.cu in numpy float64: what ``_ica._Device`` computes, without a device."""

    def __init__(self, X, k):
        self.X = np.asarray(X, dtype=np.float64)
        self.dt = X.dtype
        self.n, self.p = X.shape
        self.k = k

    def _finite(self):
        if not np.all(np.isfinite(self.X)):
            raise ValueError("Input X contains NaN or infinity.")

    def moments(self):
        self._finite()
        self.mean = self.X.mean(axis=0)
        Xc = self.X - self.mean
        return self.mean, Xc.T @ Xc

    def project(self, K):
        self._finite()
        self.X1 = self.X.copy() if K is None else (self.X - self.mean) @ (K * np.sqrt(self.n)).T

    def step(self, W, fun, alpha):
        gx, _ = contrast(fun, alpha)(self.X1 @ W.T)
        _, gp = contrast(fun, alpha)((self.X1 @ W.T).T)
        return gx.T @ self.X1, gp * self.n

    def sources(self, M, d1=None, d2=None, stats=False):
        v = (self.X1 @ M.T).astype(self.dt).astype(np.float64)
        if d1 is not None:
            v = (v / d1).astype(self.dt).astype(np.float64)
        if d2 is not None:
            v = (v / d2).astype(self.dt).astype(np.float64)
        if stats:
            return v.mean(axis=0), v.std(axis=0)
        return v.astype(self.dt)


@pytest.fixture
def host(monkeypatch):
    monkeypatch.setattr(_ica, "_Device", NumpyDevice)
    import muon_b200._snf as snf
    monkeypatch.setattr(snf, "free_device_bytes", lambda: 1 << 40)
    return _ica


def _adata(X):
    a = SimpleAnnData(np.zeros((X.shape[0], 1)))
    a.obsm["X_pca"] = X
    return a


def small(n=301, p=5, seed=0, dtype=np.float64):
    rs = np.random.RandomState(seed)
    return (rs.laplace(size=(n, p)) @ rs.normal(size=(p, p))).astype(dtype)


def test_signature_matches_reference():
    sig = json.load(open(os.path.join(GOLDEN, "ica_signature.json")))["ica"]
    ps = inspect.signature(mu.tl.ica.__wrapped__ if hasattr(mu.tl.ica, "__wrapped__") else _ica.ica).parameters
    names = list(ps)
    assert names[: len(sig["params"])] == sig["params"]
    for name, d in zip(sig["params"][-len(sig["defaults"]):], sig["defaults"]):
        assert ps[name].default == eval(d)
    for name, d in zip(sig["kwonly"], sig["kw_defaults"]):
        assert ps[name].kind is inspect.Parameter.KEYWORD_ONLY and ps[name].default == eval(d)
    assert ps["return_info"].kind is inspect.Parameter.KEYWORD_ONLY and ps["return_info"].default is False
    assert ps[sig["varkw"]].kind is inspect.Parameter.VAR_KEYWORD
    assert hasattr(mu.tl, "ica")


@pytest.mark.parametrize("kw", [{"bogus": 1}, {"n_iter": 5}, {"whiten_solve": "svd"}])
def test_unknown_keyword_is_a_type_error(host, kw):
    with pytest.raises(TypeError, match="unexpected keyword"):
        mu.tl.ica(_adata(small()), **kw)


@pytest.mark.parametrize("kw", [
    {"algorithm": "serial"}, {"whiten": True}, {"whiten": "unit"}, {"fun": "tanh"}, {"fun_args": [1.5]},
    {"max_iter": 0}, {"max_iter": 2.5}, {"tol": -1e-3}, {"whiten_solver": "qr"}, {"n_components": 0},
    {"n_components": 2.0}, {"random_state": "seed"},
])
def test_invalid_parameter_values(host, kw):
    with pytest.raises(ValueError):
        mu.tl.ica(_adata(small()), **kw)


@pytest.mark.parametrize("alpha", [0.5, 2.5])
def test_alpha_outside_range(host, alpha):
    with pytest.raises(ValueError, match=r"alpha must be in \[1,2\]"):
        mu.tl.ica(_adata(small()), fun_args={"alpha": alpha})


def test_callable_fun_is_not_implemented(host):
    with pytest.raises(NotImplementedError):
        mu.tl.ica(_adata(small()), fun=lambda x: (x, x))


def test_input_refusals(host):
    with pytest.raises(TypeError, match="Sparse"):
        mu.tl.ica(_adata(sp.csr_matrix(small())))
    with pytest.raises(ValueError, match="minimum of 2"):
        mu.tl.ica(_adata(small(n=1)))
    for bad in (np.nan, np.inf):
        X = small()
        X[3, 2] = bad
        with pytest.raises(ValueError, match="NaN or infinity"):
            mu.tl.ica(_adata(X))
    X = small()
    X[0, 0] = np.nan
    with pytest.raises(ValueError, match="NaN or infinity"):
        mu.tl.ica(_adata(X), whiten=False)
    with pytest.raises(ValueError, match="w_init has invalid shape"):
        mu.tl.ica(_adata(small()), n_components=3, w_init=np.eye(5))


def test_limits_refused_before_device_work(monkeypatch):
    def no_device(*a, **k):
        raise AssertionError("device work started")
    monkeypatch.setattr(_ica, "_Device", no_device)
    import muon_b200._snf as snf
    monkeypatch.setattr(snf, "free_device_bytes", lambda: 1 << 40)
    with pytest.raises(NotImplementedError, match="at most 128"):
        mu.tl.ica(_adata(small(p=129)))
    mu_ok = _adata(small(p=128, n=400))
    monkeypatch.setattr(snf, "free_device_bytes", lambda: 1 << 20)
    with pytest.raises(NotImplementedError, match="device memory"):
        mu.tl.ica(mu_ok)
    assert _ica.device_bytes(10**6, 50, 50, 4) > 10**6 * 50 * (4 + 8 + 4)


def test_warnings(host):
    with pytest.warns(UserWarning, match="Ignoring n_components with whiten=False"):
        mu.tl.ica(_adata(small()), n_components=2, whiten=False, max_iter=3)
    with pytest.warns(UserWarning, match="n_components is too large: it will be set to 5"):
        mu.tl.ica(_adata(small()), n_components=9, random_state=0)
    with pytest.warns(ConvergenceWarning, match="FastICA did not converge"):
        mu.tl.ica(_adata(small()), max_iter=1, random_state=0)
    assert issubclass(ConvergenceWarning, UserWarning)
    X = small(p=4)
    X[:, 3] = 5.0                           # a constant column: a Gram eigenvalue of exactly 0
    with pytest.warns(UserWarning, match="small singular values"):
        mu.tl.ica(_adata(X), whiten_solver="eigh", random_state=0, max_iter=5)
    X[:, 3] = X[:, 0]                       # a duplicated column: rank-deficient to rounding
    with pytest.warns(UserWarning, match="rank-deficient"):
        mu.tl.ica(_adata(X), random_state=0, max_iter=5)
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        mu.tl.ica(_adata(small()), algorithm="deflation", max_iter=1, random_state=0)   # deflation never warns


def test_random_state_consumption(host):
    rs = np.random.RandomState(7)
    mu.tl.ica(_adata(small()), n_components=3, random_state=rs)
    ref = np.random.RandomState(7)
    ref.normal(size=(3, 3))
    assert rs.randint(1 << 30) == ref.randint(1 << 30)
    np.random.seed(3)
    mu.tl.ica(_adata(small()), n_components=4)
    np.random.seed(3)
    np.random.normal(size=(4, 4))
    after = np.random.randint(1 << 30)
    np.random.seed(3)
    mu.tl.ica(_adata(small()), n_components=4)
    assert np.random.randint(1 << 30) == after
    rs = np.random.RandomState(7)
    mu.tl.ica(_adata(small()), n_components=3, random_state=rs, w_init=np.eye(3))
    assert rs.randint(1 << 30) == np.random.RandomState(7).randint(1 << 30)     # nothing drawn
    rs = np.random.RandomState(7)
    with pytest.raises(ValueError):
        mu.tl.ica(_adata(small()), random_state=rs, fun_args={"alpha": 3})
    assert rs.randint(1 << 30) == np.random.RandomState(7).randint(1 << 30)


@pytest.mark.parametrize("case", list(CASES))
def test_host_logic_reproduces_goldens(host, case):
    """The host steps around the device passes, with the passes in numpy: every golden case, n_iter equal."""
    z = load_golden("ica_small.npz")
    X, _, rs, scale, kw = arguments(case)
    ad = _adata(X)
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        _, info = mu.tl.ica(ad, random_state=rs, scale=scale, return_info=True, **kw)
    got = ad.obsm["X_ica"]
    assert info["n_iter"] == int(z[f"{case}_n_iter"])
    assert [str(w.message) for w in rec] == list(z[f"{case}_warnings"])
    rtol = 1e-8 if got.dtype == np.float64 else f32_rtol(z, case)
    assert_matches_golden_rows(got, z, case, rtol)
    assert_matches_restatement(got, case)
    for key in ("components", "mixing", "unmixing", "mean", "whitening"):
        if f"{case}_{key}" in z:
            assert_columns_close(info[key], z[f"{case}_{key}"], rtol, key)
        else:
            assert info[key] is None


def test_slots_copy_and_dtypes(host):
    X = small()
    ad = _adata(X)
    out = mu.tl.ica(ad, random_state=0, copy=True)
    assert "X_ica" not in ad.obsm and out.obsm["X_ica"].shape == (301, 5)
    md = SimpleMuData({"a": _adata(X)})
    md.obsm["X_mofa"] = X
    assert mu.tl.ica(md, basis="X_mofa", n_components=2, random_state=0) is None
    assert md.obsm["X_ica"].shape == (301, 2) and md.obsm["X_ica"].dtype == np.float64
    ad = _adata(np.round(X * 10).astype(np.int64))
    mu.tl.ica(ad, random_state=0)
    assert ad.obsm["X_ica"].dtype == np.float64
    ad = _adata(X.astype(np.float32))
    res, info = mu.tl.ica(ad, random_state=0, return_info=True, scale=True)
    assert res is None and ad.obsm["X_ica"].dtype == np.float32
    np.testing.assert_allclose(ad.obsm["X_ica"].std(axis=0), 1.0, rtol=1e-5)
