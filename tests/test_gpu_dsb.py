"""GPU: ``mu.prot.pp.dsb`` against the reference's fixtures, run-to-run identity, the random-stream protocol,
its refusals, and a 1M-cell run checked on a sample against ``oracle.dsb_ref``."""
import os
import warnings

import numpy as np
import pytest

import muon_b200 as mu
from conftest import GOLDEN
from dsb_cases import CASES, build_call, result_of
from muon_b200 import SimpleAnnData, SimpleMuData
from oracle.dsb_ref import background_means, scale, synth_citeseq

pytestmark = pytest.mark.gpu


def load(name):
    return dict(np.load(os.path.join(GOLDEN, f"dsb_{name}.npz")))


def run(name, z):
    data, raw, kw = build_call(name, z, SimpleAnnData, SimpleMuData)
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        ret, info = mu.prot.pp.dsb(data, raw, **kw, return_info=True)
    X, obs = result_of(name, data, raw, ret)
    return X, obs, info, [f"{x.category.__name__}: {x.message}" for x in w]


@pytest.mark.parametrize("name", list(CASES))
def test_dsb_matches_reference_fixture(cuda, name):
    z = load(name)
    X, obs, info, warned = run(name, z)
    assert X.dtype == z["out"].dtype and X.shape == z["out"].shape
    np.testing.assert_array_equal(obs, z["obs_names_out"])
    assert [s for s in warned if not s.startswith("ConvergenceWarning")] == [str(s) for s in z["warnings"]]
    f64 = X.dtype == np.float64
    if "bgmean" not in z:
        tol = 1e-12 if f64 else 1e-6
        np.testing.assert_allclose(X, z["out"], rtol=tol, atol=tol)
        assert info == {}
        return
    m = z["model"]
    rows = np.arange(len(m))
    ok = (info["model"] == m) & (info["n_iter"][rows, m] == z["n_iter"][rows, m])
    assert ok.mean() >= 0.995
    # float64: the device's log/exp and sum orders differ from numpy's in the last bit; on bgmean values up to
    # ~13 that has been measured at up to 2.2e-12 (4e-13 relative)
    np.testing.assert_allclose(info["bgmean"][ok], z["bgmean"][ok], rtol=0, atol=5e-12 if f64 else 1e-5)
    np.testing.assert_allclose(X[ok], z["out"][ok], rtol=0, atol=1e-9 if f64 else 1e-4)
    np.testing.assert_array_equal(info["converged"], z["converged"])


def test_two_calls_are_bit_identical(cuda):
    for name in ("f32", "isotype", "rs"):
        z = load(name)
        a, _, ia, _ = run(name, z)
        b, _, ib, _ = run(name, z)
        np.testing.assert_array_equal(a, b)
        for k in ia:
            np.testing.assert_array_equal(ia[k], ib[k])


def test_global_generator_is_consumed_like_the_reference(cuda):
    cells, empty = synth_citeseq(700, 800, 9, seed=3)
    np.random.seed(1234)
    _, info = mu.prot.pp.dsb(SimpleAnnData(cells.copy()), SimpleAnnData(empty, obs=[f"e{i}" for i in range(800)]),
                             random_state=None, return_info=True)
    after = np.random.get_state()
    np.random.seed(1234)
    ref = background_means(scale(cells, empty), random_state=None)
    expect = np.random.get_state()
    assert after[0] == expect[0] and np.array_equal(after[1], expect[1]) and after[2:] == expect[2:]
    np.testing.assert_array_equal(info["model"], ref["model"])
    np.testing.assert_allclose(info["bgmean"], ref["bgmean"], rtol=0, atol=1e-5)


def test_chunked_draws_match_per_fit_draws(cuda, monkeypatch):
    """The host draws the per-fit blocks chunk by chunk; small chunks must give what one chunk gives."""
    from muon_b200.prot import pp
    cells, empty = synth_citeseq(300, 500, 40, seed=4)
    E = SimpleAnnData(empty, obs=[f"e{i}" for i in range(500)])
    outs = []
    for chunk in (pp._DRAW_CHUNK, 4 * 40 * 7):
        monkeypatch.setattr(pp, "_DRAW_CHUNK", chunk)
        a = SimpleAnnData(cells.copy())
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            _, info = mu.prot.pp.dsb(a, E, random_state=np.random.RandomState(5), return_info=True)
        outs.append((a.X, info["bgmean"]))
    np.testing.assert_array_equal(outs[0][0], outs[1][0])
    np.testing.assert_array_equal(outs[0][1], outs[1][1])


def test_zero_std_control_raises(cuda):
    cells, empty = synth_citeseq(50, 200, 8, seed=5)
    empty = empty.toarray()
    empty[:, 2] = 3.0                   # constant in every empty droplet: std 0, scaled column infinite
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        with pytest.raises(ValueError):
            mu.prot.pp.dsb(SimpleAnnData(cells), SimpleAnnData(empty, obs=[f"e{i}" for i in range(200)]),
                           random_state=0)
        # without denoising the reference never validates: the infinite column is returned as is
        a = SimpleAnnData(cells.copy())
        mu.prot.pp.dsb(a, SimpleAnnData(empty, obs=[f"e{i}" for i in range(200)]), denoise_counts=False)
    assert not np.isfinite(a.X[:, 2]).any() and np.isfinite(np.delete(a.X, 2, axis=1)).all()


def test_p1025_refused(cuda):
    cells, empty = synth_citeseq(10, 20, 1025, seed=6)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        with pytest.raises(NotImplementedError):
            mu.prot.pp.dsb(SimpleAnnData(cells), SimpleAnnData(empty, obs=[f"e{i}" for i in range(20)]))


def test_one_million_cells_sampled_against_oracle(cuda):
    n, P, m = 1_000_000, 200, 200_000
    cells, empty = synth_citeseq(n, m, P, seed=7)
    a = SimpleAnnData(cells, obs=None)
    E = SimpleAnnData(empty, obs=[f"e{i}" for i in range(m)])
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        _, info = mu.prot.pp.dsb(a, E, random_state=17, return_info=True)
    assert a.X.shape == (n, P) and np.isfinite(a.X).all()
    idx = np.sort(np.random.default_rng(0).choice(n, 2000, replace=False))
    ref = background_means(scale(cells[idx], empty), random_state=17)
    ok = ref["model"] == info["model"][idx]
    assert ok.mean() >= 0.995
    np.testing.assert_allclose(info["bgmean"][idx][ok], ref["bgmean"][ok], rtol=0, atol=1e-5)
