"""CPU: the DSB oracle against the reference's fixtures, the drop-in surface of ``mu.prot.pp.dsb`` and its
host-side bookkeeping (argument errors and warnings come before any device work)."""
import json
import os
import warnings

import numpy as np
import pytest
import scipy.sparse as sp

import muon_b200 as mu
from conftest import GOLDEN
from dsb_cases import CASES, build_call, kwargs, ref_arguments
from muon_b200 import SimpleAnnData, SimpleMuData
from muon_b200.prot import pp as prot_pp
from oracle.dsb_ref import dsb_ref


def load(name):
    return dict(np.load(os.path.join(GOLDEN, f"dsb_{name}.npz")))


def agreeing_cells(z, model, n_iter):
    """Cells whose chosen model and its iteration count match the fixture.  float32 input is fitted by the
    reference in float32: a fit whose lower-bound change lands next to the tolerance can stop one round
    earlier or later there, which moves that cell's bgmean by up to the tolerance."""
    m = z["model"]
    return (model == m) & (n_iter[np.arange(len(m)), m] == z["n_iter"][np.arange(len(m)), m])


@pytest.mark.parametrize("name", list(CASES))
def test_dsb_ref_reproduces_fixture(name):
    z = load(name)
    cells, empty, kw = ref_arguments(name, z)
    r = dsb_ref(cells, empty, **kw)
    assert r["out"].dtype == z["out"].dtype
    f64 = z["out"].dtype == np.float64
    if "bgmean" not in z:
        np.testing.assert_allclose(r["out"], z["out"], rtol=1e-12 if f64 else 1e-6, atol=1e-12 if f64 else 1e-6)
        return
    ok = agreeing_cells(z, r["model"], r["n_iter"])
    assert ok.mean() >= 0.995
    if f64:
        assert ok.all()
        np.testing.assert_allclose(r["bgmean"], z["bgmean"], rtol=0, atol=1e-12)
        np.testing.assert_allclose(r["out"], z["out"], rtol=0, atol=1e-12)
    else:
        np.testing.assert_allclose(r["bgmean"][ok], z["bgmean"][ok], rtol=0, atol=1e-5)
        np.testing.assert_allclose(r["out"][ok], z["out"][ok], rtol=0, atol=1e-4)


def _reference_or_skip():
    from oracle._refload import reference_available
    if not reference_available():
        pytest.skip("reference checkout not present")
    pytest.importorskip("sklearn")
    from oracle.dsb_ref import load_reference_dsb
    return load_reference_dsb()


@pytest.mark.parametrize("name", list(CASES))
def test_live_reference_matches_fixture(name):
    dsb = _reference_or_skip()
    from dsb_cases import result_of
    z = load(name)
    data, raw, kw = build_call(name, z, SimpleAnnData, SimpleMuData)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ret = dsb(data, raw, **kw)
    X, obs = result_of(name, data, raw, ret)
    np.testing.assert_array_equal(X, z["out"])
    np.testing.assert_array_equal(obs, z["obs_names_out"])


def test_signature_matches_reference():
    import inspect
    ref = json.load(open(os.path.join(GOLDEN, "dsb_signature.json")))["dsb"]
    sig = inspect.signature(mu.prot.pp.dsb)
    pos = [p for p in sig.parameters.values() if p.kind == p.POSITIONAL_OR_KEYWORD]
    assert [p.name for p in pos] == ref["params"]
    for i, (p, d) in enumerate(zip(pos, ref["defaults"])):
        if i < ref["required"]:
            assert p.default is inspect.Parameter.empty
        else:
            assert repr(p.default) == d, (p.name, p.default, d)
    extra = [p for p in sig.parameters.values() if p.kind != p.POSITIONAL_OR_KEYWORD]
    assert [p.name for p in extra] == ["return_info"] and all(p.kind == p.KEYWORD_ONLY for p in extra)


@pytest.fixture
def no_device(monkeypatch):
    """Replace the device part with a recorder: whatever reaches it is what the host bookkeeping passed on."""
    seen = []

    def fake(X, E, out_dt, *rest):
        seen.append((X, E, out_dt) + rest)
        return np.zeros(X.shape, out_dt), {}

    monkeypatch.setattr(prot_pp, "_dsb_device", fake)
    return seen


@pytest.mark.parametrize("name", list(CASES))
def test_branches_select_the_reference_droplets_and_warn_alike(name, no_device):
    z = load(name)
    data, raw, kw = build_call(name, z, SimpleAnnData, SimpleMuData)
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        ret = mu.prot.pp.dsb(data, raw, **kw)
    got = [f"{x.category.__name__}: {x.message}" for x in w]
    assert got == [str(s) for s in z["warnings"]]
    cells, empty, _ = ref_arguments(name, z)
    X, E = no_device[0][0], no_device[0][1]
    dense = lambda M: M.toarray() if sp.issparse(M) else np.asarray(M)  # noqa: E731
    np.testing.assert_array_equal(dense(X), dense(cells))
    np.testing.assert_array_equal(dense(E), dense(empty))
    assert no_device[0][2] == z["out"].dtype
    if CASES[name]["layout"] == "mudata_none":
        assert list(ret.mod["prot"].obs_names) == [str(s) for s in z["obs_names_out"]]
    else:
        assert ret is None


def _small(P=6, n=20, m=30, seed=0):
    rng = np.random.default_rng(seed)
    cells = SimpleAnnData(rng.poisson(5.0, (n, P)).astype(np.float32), var=[f"p{j}" for j in range(P)])
    raw = SimpleAnnData(rng.poisson(1.0, (m, P)).astype(np.float32), obs=[f"e{i}" for i in range(m)],
                        var=[f"p{j}" for j in range(P)])
    return cells, raw


@pytest.mark.parametrize("call,exc", [
    (lambda c, r: mu.prot.pp.dsb(c), ValueError),
    (lambda c, r: mu.prot.pp.dsb(c, empty_counts_range=(1, 3), cell_counts_range=(2, 4)), ValueError),
    (lambda c, r: mu.prot.pp.dsb(c, empty_counts_range=(1, 2), cell_counts_range=(2, 4)), TypeError),
    (lambda c, r: mu.prot.pp.dsb(c, np.zeros((3, 6))), TypeError),
    (lambda c, r: mu.prot.pp.dsb(SimpleMuData({"rna": c}), r), TypeError),
    (lambda c, r: mu.prot.pp.dsb(c, r, pseudocount=-1), ValueError),
    (lambda c, r: mu.prot.pp.dsb(c, r, quantile_clipping=True, quantile_clip=(0.1,)), ValueError),
    (lambda c, r: mu.prot.pp.dsb(c, r, quantile_clipping=True, quantile_clip=(0.1, 1.5)), ValueError),
    (lambda c, r: mu.prot.pp.dsb(c, SimpleAnnData(np.ones((4, 5)))), ValueError),
    (lambda c, r: mu.prot.pp.dsb(c, r, random_state=np.random.default_rng(0)), ValueError),
    (lambda c, r: mu.prot.pp.dsb(c[:, [0]], r[:, [0]]), ValueError),
    (lambda c, r: mu.prot.pp.dsb(*_small(P=16), isotype_controls=[f"p{j}" for j in range(15)]), NotImplementedError),
    (lambda c, r: mu.prot.pp.dsb(*_small(P=1025)), NotImplementedError),
])
def test_argument_errors_before_device_work(call, exc, no_device):
    cells, raw = _small()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        with pytest.raises(exc):
            call(cells, raw)
    assert not no_device


def test_p1025_without_denoising_is_refused_too(no_device):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        with pytest.raises(NotImplementedError):
            mu.prot.pp.dsb(*_small(P=1025), denoise_counts=False)
    assert not no_device


def test_simple_mudata_selects_observation_names():
    a = SimpleAnnData(np.arange(12.0).reshape(4, 3), obs=["a", "b", "c", "d"])
    b = SimpleAnnData(np.arange(8.0).reshape(4, 2), obs=["a", "b", "c", "d"])
    md = SimpleMuData({"x": a, "y": b})
    import pandas as pd
    sub = md[pd.Index(["d", "b"]), :].copy()
    assert list(sub.mod["x"].obs_names) == ["d", "b"]
    np.testing.assert_array_equal(sub.mod["x"].X, a.X[[3, 1]])
    np.testing.assert_array_equal(sub.mod["y"].X, b.X[[3, 1]])
    assert list(md[["c"]].mod["y"].obs_names) == ["c"]          # what worked before still does
    with pytest.raises(NotImplementedError):
        md[["c"], [0]]


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("n", [1, 2, 7, 1000, 4097])
def test_quantiles_match_numpy(dtype, n):
    rng = np.random.default_rng(n)
    a = (rng.normal(size=n) * 3).astype(dtype)
    qs = np.asarray([0.0, 0.001, 0.25, 0.5, 0.9995, 1.0])
    srt = np.sort(a)
    got = prot_pp._quantiles_linear(n, qs, lambda k: srt[k], dtype)
    np.testing.assert_array_equal(got, np.quantile(a, qs))


def test_kwargs_roundtrip():
    for name in CASES:
        assert set(kwargs(name)) == set(CASES[name]["kw"])
