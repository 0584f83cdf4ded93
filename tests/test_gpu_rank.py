"""GPU: ``mu.atac.tl.rank_peaks_groups`` against the reference run recorded in tests/golden/rank_small.npz, the
per-peak statistics against the float64 oracle (short and long rows), determinism and the error paths."""
import io
import json
import os
import sys

import numpy as np
import pandas as pd
import pytest
import scipy.sparse as sp

from conftest import GOLDEN
from oracle import rank_ref as R

pytestmark = pytest.mark.gpu
sys.path.insert(0, GOLDEN)
import make_golden_rank as M  # noqa: E402

Z = np.load(os.path.join(GOLDEN, "rank_small.npz"))
CASES = json.load(open(os.path.join(GOLDEN, "rank_signature.json")))["cases"]
X0, LABELS = M.load_counts(Z)
PEAKS = np.array(M.peak_names(M.N_PEAKS))


def fixture_adata(drop=None):
    import muon_b200 as mu
    ad = M.make_adata(X0, M.scaled_layer(X0), LABELS)
    mu.atac.tl.add_peak_annotation(ad, pd.read_csv(io.StringIO(M.annotation_tsv(M.N_PEAKS, drop)), sep="\t"))
    return ad


def check_against_fixture(name, uns, rankby_abs=False):
    groups = uns["names"].dtype.names
    clear_of = {}
    assert json.loads(str(Z[f"{name}|params"])) == json.loads(json.dumps(uns["params"]))
    for g in groups:
        sc = uns["scores"][g]
        want_sc = Z[f"{name}|scores|{g}"]
        assert sc.dtype == np.float32 and len(sc) == len(want_sc)
        names, want_names = np.asarray(uns["names"][g], dtype=str), PEAKS[Z[f"{name}|names|{g}"]]
        # names identical wherever the neighbouring ranking keys are apart by more than float32 rounding
        s64 = want_sc.astype(np.float64)
        if rankby_abs:
            s64 = np.abs(s64)
        gap = np.abs(np.diff(s64)) > 4 * np.finfo(np.float32).eps * np.maximum(np.abs(s64[1:]), 1e-30)
        clear = np.ones(len(s64), bool)
        clear[1:] &= gap
        clear[:-1] &= gap
        if len(s64) < M.N_PEAKS:        # a truncated list: peaks tied with its last score may be cut either way
            clear &= np.abs(s64 - s64[-1]) > 4 * np.finfo(np.float32).eps * max(abs(s64[-1]), 1e-30)
        assert np.array_equal(names[clear], want_names[clear]), g
        clear_of[g] = set(names[clear])
        # scores: float32 within 1 ulp at the same peak
        ulps = np.abs(sc.view(np.int32).astype(np.int64) - want_sc.view(np.int32).astype(np.int64))
        assert np.all(ulps[clear] <= 1), g
        ok = set(np.flatnonzero(clear))
        for key in ("pvals", "pvals_adj"):
            got, want = uns[key][g], Z[f"{name}|{key}|{g}"]
            sel = np.array([i in ok for i in range(len(got))]) & (want >= 1e-250)
            np.testing.assert_allclose(got[sel], want[sel], rtol=1e-9, atol=0, err_msg=f"{name} {key} {g}")
        sel = np.array([i in ok for i in range(len(sc))])
        np.testing.assert_allclose(uns["logfoldchanges"][g][sel], Z[f"{name}|logfoldchanges|{g}"][sel], rtol=0, atol=1e-5)
    for key in ("pts", "pts_rest"):
        if f"{name}|{key}" in Z:
            assert list(uns[key].columns) == list(Z[f"{name}|{key}|columns"])
            np.testing.assert_allclose(uns[key].to_numpy(), Z[f"{name}|{key}"], rtol=1e-14)
        else:
            assert key not in uns
    # the joined annotation, peak by peak (tied peaks may be listed in another order)
    gone = PEAKS[int(Z["unannotated_drop"])] if name == "unannotated" else None
    for key in ("genes", "peak_type", "distance"):
        for g in groups:
            k = f"{name}|{key}|{g}"
            if k in Z:
                mine = [str(x) for x in np.asarray(uns["names"][g], dtype=str) if x != gone]
                theirs = [str(x) for x in PEAKS[Z[f"{name}|names|{g}"]] if x != gone]
                got = [str(x) for x in uns[key][g]]
                assert len(got) == len(Z[k]), (name, key, g)
                keep = clear_of[g]
                mine_d, theirs_d = dict(zip(mine, got)), dict(zip(theirs, Z[k]))
                assert {p: mine_d[p] for p in keep if p in mine_d} == {p: theirs_d[p] for p in keep if p in theirs_d}


@pytest.mark.parametrize("name", list(CASES))
def test_reproduces_reference_run(name, cuda):
    import muon_b200 as mu
    kw = dict(CASES[name])
    drop = int(Z["unannotated_drop"]) if name == "unannotated" else None
    ad = fixture_adata(drop)
    err = str(Z[f"{name}|error"])
    if err:
        import builtins
        with pytest.raises(getattr(builtins, err)) as info:
            mu.atac.tl.rank_peaks_groups(ad, "leiden", **kw)
        assert type(info.value).__name__ == err
    else:
        mu.atac.tl.rank_peaks_groups(ad, "leiden", **kw)
    check_against_fixture(name, ad.uns["rank_genes_groups"], kw.get("rankby_abs", False))


def _stats(X, labels, n_groups, reference=None, groups="all", tie_correct=True):
    import torch

    from muon_b200 import _rank
    cat = pd.Categorical([str(v) for v in labels], categories=[str(i) for i in range(n_groups)])
    plan = _rank.Plan(pd.Series(cat), groups, "rest" if reference is None else reference)
    A = _rank.device_matrix(X)
    st, long_share, _ = _rank.peak_stats(A, plan, np.arange(X.shape[1]), wilcoxon=True, tie_correct=tie_correct)
    torch.cuda.synchronize()
    return plan, st.cpu().numpy(), long_share


def _oracle_stats(X, plan, labels):
    masks = np.stack([np.asarray([str(v) == g for v in labels]) for g in plan.tested + ([plan.reference] if plan.reference
                                                                                         else [])])
    ref = len(plan.tested) if plan.reference is not None else None
    return R.group_stats(X, masks, ref, tie_correct=True)


def _compare_stats(plan, st, want):
    G = len(plan.tested)
    np.testing.assert_array_equal(st[0, :G], want["cnt"][:G])
    np.testing.assert_array_equal(st[3, :G], want["ranksum"][:G])
    np.testing.assert_array_equal(st[4, :G], want["tie"][:G].astype(np.float64))
    np.testing.assert_allclose(st[1, :G], want["sum"][:G], rtol=1e-12, atol=1e-300)
    np.testing.assert_allclose(st[2, :G], want["sumsq"][:G], rtol=1e-12, atol=1e-300)


@pytest.mark.parametrize("layer", ["X", "scaled"])
@pytest.mark.parametrize("reference", [None, "1"])
def test_stats_equal_oracle(layer, reference, cuda):
    labels, X = LABELS, X0
    if layer == "scaled":
        X = M.scaled_layer(X0)
    groups = "all" if reference is None else ["3", "0", "1"]
    plan, st, _ = _stats(X, labels, len(M.SIZES), reference, groups)
    _compare_stats(plan, st, _oracle_stats(np.asarray(X.toarray() if sp.issparse(X) else X), plan, labels))


def test_long_row_matches_oracle(cuda):
    rng = np.random.default_rng(5)
    n = 40_000
    labels = rng.integers(0, 3, size=n)
    dense = np.zeros((n, 3), np.float32)
    dense[:, 0] = rng.integers(1, 50, size=n)                      # stored in every cell: the long-row path
    dense[:, 1] = rng.integers(-3, 4, size=n) * (rng.random(n) < 0.3)
    X = sp.csr_matrix(dense)
    for reference in (None, "2"):
        plan, st, long_share = _stats(X, labels, 3, reference, "all")
        assert long_share > 0.5
        _compare_stats(plan, st, _oracle_stats(dense, plan, labels))


def test_long_and_short_paths_agree(cuda):
    """Rows that fit in shared memory, forced through the global-memory sort: identical bits."""
    import torch

    from muon_b200 import _device, _lib, _rank
    X = X0
    cat = pd.Categorical([str(v) for v in LABELS], categories=[str(i) for i in range(len(M.SIZES))])
    for reference in ("rest", "1"):
        plan = _rank.Plan(pd.Series(cat), "all", reference)
        A = _rank.device_matrix(X)
        short, _, flags = _rank.peak_stats(A, plan, np.arange(X.shape[1]), wilcoxon=True, tie_correct=True)
        T = _device.csr_transpose(A)
        d = X.shape[1]
        K = len(plan.tested) + 1
        out = torch.empty_like(short)
        cap = 2 * _lib.load().mub_rank_shared_capacity(4)
        slice_bytes = _lib.load().mub_rank_workspace_slice_bytes(4, cap)
        ws = torch.empty(8 * slice_bytes, dtype=torch.uint8, device=A.data.device)
        rows = torch.arange(d, dtype=torch.int32, device=A.data.device)
        code, sizes = torch.from_numpy(plan.code).cuda(), torch.from_numpy(plan.sizes).cuda()
        _lib.call("mub_rank_stats_f32", _lib.ptr(T.indptr), _lib.ptr(T.indices), _lib.ptr(T.data), _lib.ptr(code),
                  _lib.ptr(rows), _lib.ptr(rows), d, d, K, _lib.ptr(sizes), plan.n_ranked, flags, cap, _lib.ptr(ws),
                  ws.numel(), _lib.ptr(out), _lib.stream_ptr())
        assert torch.equal(out, short)


def test_all_zero_peak(cuda):
    import muon_b200 as mu
    for kw in ({"method": "wilcoxon"}, {"method": "wilcoxon", "tie_correct": True}, {"method": "t-test"}):
        ad = fixture_adata()
        mu.atac.tl.rank_peaks_groups(ad, "leiden", **kw)
        res = ad.uns["rank_genes_groups"]
        for g in res["names"].dtype.names:
            names = list(res["names"][g])
            for p in PEAKS[-10:]:
                i = names.index(p)
                assert res["scores"][g][i] == 0 and res["pvals"][g][i] == 1


def test_host_and_device_input_and_repeat_calls_identical(cuda):
    import muon_b200 as mu
    from muon_b200 import DeviceCSR
    outs = []
    for kind in ("host", "device", "device"):
        ad = fixture_adata()
        if kind == "device":
            ad.X = DeviceCSR.from_scipy(ad.X)
        mu.atac.tl.rank_peaks_groups(ad, "leiden", method="wilcoxon", tie_correct=True, pts=True)
        outs.append(ad.uns["rank_genes_groups"])
        if kind == "device":
            assert ad.X._t is None                       # no transpose left cached on the caller's matrix
    for o in outs[1:]:
        for key in ("names", "scores", "pvals", "pvals_adj", "logfoldchanges"):
            for g in o[key].dtype.names:
                assert np.array_equal(o[key][g], outs[0][key][g])
        assert np.array_equal(o["pts"].to_numpy(), outs[0]["pts"].to_numpy())
    # a float64 matrix is ranked on its own values; two calls are bit-identical
    a, b = fixture_adata(), fixture_adata()
    for ad in (a, b):
        mu.atac.tl.rank_peaks_groups(ad, "leiden", method="t-test", layer="scaled")
    for key in ("scores", "pvals"):
        for g in a.uns["rank_genes_groups"][key].dtype.names:
            assert np.array_equal(a.uns["rank_genes_groups"][key][g], b.uns["rank_genes_groups"][key][g])


def test_error_paths(cuda):
    import muon_b200 as mu
    ad = fixture_adata()
    labels = np.array(ad.obs["leiden"].astype(str))
    labels[0] = "9"
    ad.obs["single"] = pd.Categorical(labels)
    with pytest.raises(ValueError):
        mu.atac.tl.rank_peaks_groups(ad, "single")
    with pytest.raises(ValueError):
        mu.atac.tl.rank_peaks_groups(ad, "leiden", reference="nope")
    ad.obs["plain"] = labels
    with pytest.raises(ValueError):
        mu.atac.tl.rank_peaks_groups(ad, "plain")
    with pytest.raises(NotImplementedError):
        mu.atac.tl.rank_peaks_groups(ad, "leiden", method="logreg")
    assert "rank_genes_groups" not in ad.uns
