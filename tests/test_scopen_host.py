"""CPU: the host side of ``mu.atac.pp.scopen`` with no device work -- the signature, every error and refusal (all
raised before any device work), the prints, the warning, and the slots' dtypes and layouts, with the device passes
of ``_scopen.Fit`` replaced by the float64 restatement (oracle/scopen_ref.py)."""
import inspect
import json
import os
import warnings

import numpy as np
import pytest
import scipy.sparse as sp

import muon_b200 as mu
import muon_b200._snf as snf
from muon_b200 import SimpleAnnData, SimpleMuData
from muon_b200 import _scopen
from muon_b200.prot.pp import ConvergenceWarning
from conftest import GOLDEN, load_golden
from oracle import scopen_ref as R
from scopen_cases import CASES, arguments, matrix, planted_counts, sample_rows


class NumpyFit:
    """What ``_scopen.Fit`` computes, in numpy float64 on the host (exact SVD for the init)."""

    created = 0

    def __init__(self, X, k):
        NumpyFit.created += 1
        self.X, self.k = sp.csr_matrix(X), k

    def positives(self):
        return np.diff(np.concatenate([[0], np.cumsum(self.X.data > 0)])[self.X.indptr])

    def build(self, s):
        P, _ = R.pattern_of(self.X)
        self.RX = R.PatternMatrix(P, s)
        self.dense = R.dense_of(P, s)

    def svd(self):
        return R.exact_svd(self.dense, self.k)

    def set_factors(self, W, H):
        self.W, self.Ht = np.array(W, order="C"), np.array(np.asarray(H).T, order="C")

    def iterate(self, alpha, upper):
        return R.w_step(self.RX, self.W, self.Ht, alpha, upper), R.h_step(self.RX, self.W, self.Ht, alpha, upper)

    def factors(self):
        return self.W.copy(), self.Ht.T.copy()

    def impute(self, out):
        out[:] = np.clip(self.W @ self.Ht.T, 0, 1)
        return out


def no_device(*a, **k):
    raise AssertionError("device work started")


@pytest.fixture
def host(monkeypatch):
    monkeypatch.setattr(_scopen, "Fit", NumpyFit)
    monkeypatch.setattr(snf, "free_device_bytes", lambda: 1 << 40)


@pytest.fixture
def refuse_device(monkeypatch):
    monkeypatch.setattr(_scopen, "Fit", no_device)
    monkeypatch.setattr(snf, "free_device_bytes", lambda: 1 << 40)


def _ad(n=40, m=90, seed=0):
    return SimpleAnnData(sp.csr_matrix(planted_counts(seed, n, m, 4)))


def test_signature_matches_reference():
    ref = json.load(open(os.path.join(GOLDEN, "scopen_signature.json")))["scopen"]
    sig = inspect.signature(mu.atac.pp.scopen)
    assert list(sig.parameters) == ref["params"]
    got = [repr(p.default) for p in sig.parameters.values() if p.default is not inspect.Parameter.empty]
    assert got == ref["defaults"]


def test_type_error_before_device_work(refuse_device):
    with pytest.raises(TypeError, match="Expected AnnData or MuData object with 'atac' modality"):
        mu.atac.pp.scopen(np.ones((3, 3)))
    with pytest.raises(TypeError, match="'atac' modality"):
        mu.atac.pp.scopen(SimpleMuData({"rna": _ad()}))


@pytest.mark.parametrize("kw,match", [
    ({"n_components": 0}, "Number of components must be a positive integer"),
    ({"n_components": 2.5}, "Number of components must be a positive integer"),
    ({"n_components": 41}, "can only be used when n_components <= min"),
    ({"max_iter": -1}, "Maximum number of iterations must be a positive integer"),
])
def test_parameter_errors_before_device_work(refuse_device, kw, match):
    with pytest.raises(ValueError, match=match):
        mu.atac.pp.scopen(_ad(), **kw)


def test_non_finite_scales_before_device_work(refuse_device):
    C = planted_counts(0, 40, 90, 4)
    empty = C.copy()
    empty[3] = 0                                                    # a cell without open regions
    equal = np.zeros((5, 8))
    equal[:, :2] = 1                                                # every cell has the same count
    for X, kw in ((empty, {}), (equal, {"n_components": 2}), (C, {"max_rho": 1.0})):
        with pytest.raises(ValueError, match="Input contains NaN, infinity"):
            mu.atac.pp.scopen(SimpleAnnData(sp.csr_matrix(X)), **kw)


def test_refusals_before_device_work(monkeypatch, refuse_device):
    big = SimpleAnnData(sp.csr_matrix(planted_counts(0, 70, 90, 4)))
    with pytest.raises(NotImplementedError, match="at most 64"):
        mu.atac.pp.scopen(big, n_components=65)
    monkeypatch.setattr(_scopen, "MAX_DIM", 80)
    with pytest.raises(NotImplementedError, match="cells x 90 peaks"):
        mu.atac.pp.scopen(_ad(), n_components=2)
    monkeypatch.setattr(_scopen, "MAX_DIM", 2**31 - 1)
    monkeypatch.setattr(snf, "free_device_bytes", lambda: 1 << 20)
    with pytest.raises(NotImplementedError, match="GiB of device memory"):
        mu.atac.pp.scopen(_ad(), n_components=2)


def test_sixty_four_components_run(host):
    ad = SimpleAnnData(sp.csr_matrix(planted_counts(0, 70, 90, 4)))
    mu.atac.pp.scopen(ad, n_components=64, max_iter=2)
    assert ad.obsm["X_scopen"].shape == (70, 64)


@pytest.mark.parametrize("case", list(CASES))
def test_host_logic_reproduces_goldens(host, capsys, case):
    z = load_golden("scopen_small.npz")
    data, ad, kw = arguments(case, (SimpleAnnData, SimpleMuData))
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        assert mu.atac.pp.scopen(data, **kw) is None
    lines = capsys.readouterr().out.splitlines()
    assert lines[:3] == list(z[f"{case}_lines"])
    assert len(lines) == 4 and lines[3].startswith("[total time:  ") and lines[3].endswith(" ]")
    assert [str(w.message) for w in rec] == list(z[f"{case}_warnings"])
    assert all(issubclass(w.category, ConvergenceWarning) for w in rec)
    np.testing.assert_array_equal(ad.varm["scopen"], z[f"{case}_W"])
    np.testing.assert_array_equal(ad.obsm["X_scopen"], z[f"{case}_H"].T)
    m = ad.varm["scopen"].shape[0]
    np.testing.assert_array_equal(ad.X.T[sample_rows(m)], z[f"{case}_M_rows"])
    n, k = ad.obsm["X_scopen"].shape
    assert ad.X.shape == (n, m) and ad.X.dtype == np.float64 and ad.X.flags.f_contiguous
    assert ad.X.T.flags.c_contiguous
    assert ad.obsm["X_scopen"].dtype == np.float64 and ad.varm["scopen"].dtype == np.float64
    assert ad.varm["scopen"].shape == (m, k)


def test_verbose_prints_sklearns_lines(host, capsys):
    data, ad, kw = arguments("converges", (SimpleAnnData, SimpleMuData))
    mu.atac.pp.scopen(data, verbose=True, **kw)
    lines = capsys.readouterr().out.splitlines()
    z = load_golden("scopen_small.npz")
    n_iter = int(z["converges_n_iter"])
    viol = [x for x in lines if x.startswith("violation: ")]
    assert len(viol) == n_iter
    assert f"Converged at iteration {n_iter + 1}" in lines
    assert float(viol[-1].split()[1]) <= R.TOL


def test_host_input_layouts_and_duplicates(host):
    X, _ = matrix("csr_f32")
    assert not X.has_canonical_format
    outs = []
    for Y in (X, X.tocoo(), sp.csr_matrix(X.toarray().astype(np.float64)), X.toarray()):
        ad = SimpleAnnData(Y)
        mu.atac.pp.scopen(ad, n_components=4, max_iter=3)
        outs.append(ad.varm["scopen"])
    for o in outs[1:]:
        np.testing.assert_array_equal(o, outs[0])
