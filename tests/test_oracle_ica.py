"""CPU: the float64 restatement of FastICA (oracle/ica_ref.py) against the unmodified reference's outputs
(tests/golden/ica_small.npz, made by tests/golden/make_golden_ica.py), against live sklearn when it is importable,
and on the planted sources."""
import warnings

import numpy as np
import pytest

from conftest import load_golden
from ica_cases import CASES, arguments, sample_rows
from oracle.ica_ref import fastica_ref, match_sources

F64 = [c for c in CASES if CASES[c][2] == np.float64]


def golden():
    return load_golden("ica_small.npz")


def assert_columns_close(got, want, rtol, what=""):
    """|got - want| <= rtol x the column's max |want|, column by column (rows of a 1-D array: one scale)."""
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    scale = np.max(np.abs(want), axis=0) if want.ndim > 1 else np.max(np.abs(want))
    err = np.max(np.abs(got - want) / scale)
    assert err <= rtol, f"{what}: max error {err:.3e} relative to the column scale > {rtol:g}"


def f32_rtol(z, case):
    """1e-4 relative, or twice the distance of sklearn's float32 run from its float64 run when that is larger:
    float32 input is fitted in float64 here."""
    return max(1e-4, 2 * float(z[f"{case}_f32_gap"]))


def assert_matches_golden_rows(got, z, case, rtol):
    """The output's shape and dtype, and its fixture rows (``ica_cases.sample_rows``) against the reference's."""
    want = z[f"{case}_X_ica"]
    assert tuple(got.shape) == tuple(int(v) for v in z[f"{case}_X_ica_shape"])
    assert got.dtype == want.dtype
    assert_columns_close(got[sample_rows(got.shape[0])], want, rtol, "X_ica rows")


def assert_matches_restatement(got, case):
    """Every row of an output against the float64 restatement of the same case: 1e-8 of each column's scale for
    float64 input, 1e-5 for float32 input (the output is rounded to float32)."""
    out, _ = run_ref(case)
    assert_columns_close(got, out["sources"], 1e-8 if got.dtype == np.float64 else 1e-5, "X_ica vs restatement")


def run_ref(case):
    X, S, rs, scale, kw = arguments(case)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        out = fastica_ref(X, random_state=rs, **kw)
    if scale:
        out["sources"] = out["sources"] / out["sources"].std(axis=0)
    return out, S


def test_golden_records_its_sklearn_version_and_every_case():
    z = golden()
    assert str(z["sklearn_version"]).startswith("1.")
    assert list(z["cases"]) == list(CASES)


@pytest.mark.parametrize("case", F64)
def test_restatement_reproduces_float64_goldens(case):
    z = golden()
    out, _ = run_ref(case)
    assert out["n_iter"] == int(z[f"{case}_n_iter"])
    assert_matches_golden_rows(out["sources"], z, case, 1e-10)
    for key in ("components", "mixing", "unmixing"):
        assert_columns_close(out[key], z[f"{case}_{key}"], 1e-10, key)
    if f"{case}_mean" in z:
        assert_columns_close(out["mean"], z[f"{case}_mean"], 1e-12, "mean")
        assert_columns_close(out["whitening"], z[f"{case}_whitening"], 1e-10, "whitening")


@pytest.mark.parametrize("case", ["p7_par_exp", "p7_def_exp_global", "p7_eigh_a15", "p7_nowhiten"])
def test_restatement_matches_live_sklearn(case):
    sk = pytest.importorskip("sklearn.decomposition")
    X, _, rs, scale, kw = arguments(case)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        est = sk.FastICA(random_state=rs, **kw)
        S = est.fit_transform(X)
    out, _ = run_ref(case)
    assert out["n_iter"] == est.n_iter_
    assert_columns_close(out["sources"], S, 1e-10, "sources")
    assert_columns_close(out["components"], est.components_, 1e-10, "components")


@pytest.mark.parametrize("case", ["p7_par_exp", "p7_def_logcosh_a15", "p7_def_cube_k4", "p50_par_k10", "f32_p7_par"])
def test_restatement_recovers_planted_sources(case):
    out, S = run_ref(case)
    assert match_sources(out["sources"], S) >= 0.99
