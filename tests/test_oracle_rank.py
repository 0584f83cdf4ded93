"""CPU: the rank_genes_groups restatement against scipy, the peak annotation shims against the reference functions,
the reference's own annotation tests, and the signatures."""
import copy
import io
import json
import os

import numpy as np
import pandas as pd
import pytest
import scipy.sparse as sp
from scipy import stats

from conftest import GOLDEN
from muon_b200 import SimpleAnnData, SimpleMuData
from muon_b200 import _rank
from muon_b200.atac import tl as atl
from oracle import rank_ref as R


def _adata(X, labels, n_groups):
    ad = SimpleAnnData(X, var=[f"p{i}" for i in range(X.shape[1])])
    ad.obs["g"] = pd.Categorical([str(v) for v in labels], categories=[str(i) for i in range(n_groups)])
    return ad


def _random_case(seed=0, n=150, d=40):
    rng = np.random.default_rng(seed)
    labels = rng.integers(0, 3, size=n)
    X = rng.integers(-2, 4, size=(n, d)).astype(np.float64) * (rng.random((n, d)) < 0.5)   # ties, negatives, zeros
    return X, labels


@pytest.mark.parametrize("method", ["t-test", "wilcoxon"])
def test_oracle_scores_equal_scipy(method):
    X, labels = _random_case()
    ad = _adata(sp.csr_matrix(X), labels, 3)
    R.rank_genes_groups(ad, "g", method=method, n_genes=None)
    res = ad.uns["rank_genes_groups"]
    for g in range(3):
        m = labels == g
        if method == "t-test":
            want = stats.ttest_ind(X[m], X[~m], equal_var=False)
        else:
            want = stats.ranksums(X[m], X[~m])
        order = [int(s[1:]) for s in res["names"][str(g)]]
        np.testing.assert_allclose(res["pvals"][str(g)], want.pvalue[order], rtol=1e-12, atol=0)
        np.testing.assert_allclose(res["scores"][str(g)], want.statistic[order].astype(np.float32), rtol=1e-6)


def test_oracle_tie_corrected_z_equals_mannwhitneyu():
    X, labels = _random_case(1)
    ad = _adata(sp.csr_matrix(X), labels, 3)
    R.rank_genes_groups(ad, "g", method="wilcoxon", tie_correct=True)
    res = ad.uns["rank_genes_groups"]
    for g in range(3):
        m = labels == g
        want = stats.mannwhitneyu(X[m], X[~m], use_continuity=False, method="asymptotic")
        order = [int(s[1:]) for s in res["names"][str(g)]]
        np.testing.assert_allclose(res["pvals"][str(g)], want.pvalue[order], rtol=1e-12, atol=0)
    # against a group: ranks over the two groups only
    R.rank_genes_groups(ad, "g", method="wilcoxon", tie_correct=True, reference="2")
    res = ad.uns["rank_genes_groups"]
    assert res["names"].dtype.names == ("0", "1")
    for g in range(2):
        want = stats.mannwhitneyu(X[labels == g], X[labels == 2], use_continuity=False, method="asymptotic")
        order = [int(s[1:]) for s in res["names"][str(g)]]
        np.testing.assert_allclose(res["pvals"][str(g)], want.pvalue[order], rtol=1e-12, atol=0)


def test_tie_term_exact_beyond_int64():
    """A tie block of 2 097 153 = 2^21 + 1 cells: t^3 - t is above 2^63, where int64 arithmetic wraps negative.  The
    ranked-cell limit admits blocks up to 2 642 244 cells, so the oracle must stay exact there."""
    t = 2_097_153
    ranks = np.zeros((t + 3, 2))
    ranks[t:, 0] = [1.0, 2.0, 2.0]                      # column 0: blocks of t, 1 and 2
    ranks[:, 1] = np.arange(t + 3)                      # column 1: no ties
    got = R.tie_term(ranks)
    assert got[0] == t**3 - t + 2**3 - 2 and got[0] > 2**63
    assert got[1] == 0
    X = np.zeros((t + 3, 1))
    X[: t + 1, 0] = 5.0                                 # a stored block of t + 1, next to a zero block of 2
    st = R.group_stats(X, np.stack([np.arange(t + 3) < 4, np.arange(t + 3) >= 4]), None, tie_correct=True)
    want = float((t + 1) ** 3 - (t + 1) + 2**3 - 2)
    assert st["tie"][0, 0] == want and st["tie"][1, 0] == want


def test_bh_and_top_selection():
    import torch
    rng = np.random.default_rng(3)
    p = rng.random((4, 500)) ** 3
    p[:, :20] = p[:, [0]]                               # ties
    got = _rank.adjust(torch.from_numpy(p), "benjamini-hochberg").numpy()
    want = np.stack([stats.false_discovery_control(r) for r in p])
    np.testing.assert_allclose(got, want, rtol=1e-14, atol=0)
    np.testing.assert_allclose(_rank.adjust(torch.from_numpy(p), "bonferroni").numpy(), np.minimum(p * 500, 1.0))
    s = np.array([[0.5, 2.0, 2.0, -3.0, 2.0]])
    assert _rank.top(torch.from_numpy(s), 4, False).numpy().tolist() == [[1, 2, 4, 0]]     # ties: ascending index
    assert _rank.top(torch.from_numpy(s), 2, True).numpy().tolist() == [[3, 1]]


def test_errors_before_device_work():
    X, labels = _random_case()
    ad = _adata(sp.csr_matrix(X), labels, 3)
    with pytest.raises(NotImplementedError):
        atl.rank_peaks_groups(ad, "g", method="logreg")
    with pytest.raises(ValueError):
        atl.rank_peaks_groups(ad, "g", reference="7")
    with pytest.raises(TypeError):
        atl.rank_peaks_groups(ad, "g", not_a_scanpy_argument=1)
    ad.obs["plain"] = labels
    with pytest.raises(ValueError):
        atl.rank_peaks_groups(ad, "plain")
    one = labels.copy()
    one[:] = 0
    one[5] = 1
    ad.obs["one"] = pd.Categorical([str(v) for v in one], categories=["0", "1"])
    with pytest.raises(ValueError):
        atl.rank_peaks_groups(ad, "one")
    with pytest.raises(TypeError):
        atl.rank_peaks_groups(X, "g")
    with pytest.raises(KeyError):
        atl.rank_peaks_groups(SimpleMuData({"rna": ad}), "g")
    many = _adata(sp.csr_matrix(np.ones((2 * (_rank.RANK_MAX_GROUPS + 1), 2))),
                  np.repeat(np.arange(_rank.RANK_MAX_GROUPS + 1), 2), _rank.RANK_MAX_GROUPS + 1)
    with pytest.raises(NotImplementedError):
        atl.rank_peaks_groups(many, "g")


def test_signatures_match_reference():
    import inspect
    ref = json.load(open(os.path.join(GOLDEN, "rank_signature.json")))["signatures"]
    for name, want in ref.items():
        sig = inspect.signature(getattr(atl, name))
        pos = [p for p in sig.parameters.values() if p.kind == p.POSITIONAL_OR_KEYWORD]
        assert [p.name for p in pos] == want["params"], name
        defaults = [repr(p.default) for p in pos[want["required"]:]]
        assert defaults == [repr(eval(d)) for d in want["defaults"]], name   # noqa: S307 -- literals from the fixture
        assert all(p.default is inspect.Parameter.empty for p in pos[:want["required"]])
        extra = [p for p in sig.parameters.values() if p.kind != p.POSITIONAL_OR_KEYWORD]
        assert [p.name for p in extra if p.kind == p.VAR_KEYWORD] == ([want["var_keyword"]] if want["var_keyword"] else [])
        assert all(p.kind in (p.KEYWORD_ONLY, p.VAR_KEYWORD) for p in extra)


# ---- the reference's tests/test_atac_tools.py, on this package -------------------------------------------------------
def test_empty_distance_values():
    tsv = io.StringIO("chrom\tstart\tend\tgene\tdistance\tpeak_type\n"
                      "chr1\t100\t200\t\t\tintergenic\n"
                      "chr1\t300\t400\tGeneA\t-173268\tdistal\n")
    pa = pd.read_csv(tsv, sep="\t")
    peaks = ["chr1:100-200", "chr1:300-400"]
    adata = SimpleAnnData(np.zeros((2, 2)), var=peaks)
    result = atl.add_peak_annotation(adata, pa, return_annotation=True)
    assert result.distance.dtype == pd.Int64Dtype()
    assert result.distance.iloc[0] is pd.NA
    assert result.distance.iloc[1] == -173268
    assert (result.peak == peaks).all()


def test_semicolon_separated_distances():
    tsv = io.StringIO("chrom\tstart\tend\tgene\tdistance\tpeak_type\n"
                      "chr1\t100\t200\tGeneA;GeneB\t-100;200\tpromoter;distal\n")
    pa = pd.read_csv(tsv, sep="\t")
    adata = SimpleAnnData(np.zeros((1, 1)), var=["chr1:100-200"])
    result = atl.add_peak_annotation(adata, pa, return_annotation=True)
    assert result.distance.dtype == np.int64
    assert result.distance.iloc[0] == -100
    assert result.distance.iloc[1] == 200
    assert (result.peak.iloc[0] == result.peak.iloc[1] == adata.var_names).all()


# ---- the host shims against the reference functions ------------------------------------------------------------------
def _reference():
    from oracle._refload import reference_available
    if not reference_available():
        pytest.skip("reference checkout not present")
    return R.load_reference_rank_peaks_groups()


def _uns_equal(a, b):
    assert set(a) == set(b)
    for k in a:
        va, vb = a[k], b[k]
        if isinstance(va, pd.DataFrame):
            pd.testing.assert_frame_equal(va, vb)
        elif isinstance(va, np.ndarray) and va.dtype.names:
            assert va.dtype == vb.dtype and all(np.array_equal(va[f], vb[f]) for f in va.dtype.names)
        elif hasattr(va, "__len__") and not isinstance(va, str):
            assert type(va) is type(vb) and list(va) == list(vb)
        elif isinstance(va, dict):
            _uns_equal(va, vb)
        else:
            assert va == vb


def _annotation_tables():
    import sys
    sys.path.insert(0, GOLDEN)
    import make_golden_rank as M
    full = M.annotation_tsv(M.N_PEAKS)
    plain = "chrom\tstart\tend\tgene\tdistance\tpeak_type\nchr1\t0\t500\tG0\t5\tpromoter\nchr1\t1000\t1500\t\t\tintergenic\n"
    return {"multi": full, "plain": plain}


@pytest.mark.parametrize("table", ["multi", "plain"])
def test_annotation_shims_match_reference(table):
    _, ref_add_genes, ref_add_ann, ref_add_names = _reference()
    tsv = _annotation_tables()[table]
    var = [f"chr1:{1000 * i}-{1000 * i + 500}" for i in range(4)]
    gene_names = pd.DataFrame({"gene_ids": ["G0", "G1", "G7", "G8"]}, index=["Zero", "One", "Seven", "Eight"])
    out = []
    for add_ann, add_names in ((ref_add_ann, ref_add_names), (atl.add_peak_annotation, atl.add_peak_annotation_gene_names)):
        ad = SimpleAnnData(np.zeros((2, 4)), var=var)
        ann = add_ann(ad, pd.read_csv(io.StringIO(tsv), sep="\t"), return_annotation=True)
        renamed = add_names(ad, gene_names=gene_names, return_annotation=True)
        out.append((ann, renamed, copy.deepcopy(ad.uns)))
    pd.testing.assert_frame_equal(out[0][0], out[1][0])
    pd.testing.assert_frame_equal(out[0][1], out[1][1])
    _uns_equal(out[0][2], out[1][2])
    for fn in (ref_add_names, atl.add_peak_annotation_gene_names):
        with pytest.raises(KeyError):
            fn(SimpleAnnData(np.zeros((2, 4)), var=var), gene_names=gene_names)
        with pytest.raises(TypeError):
            fn(np.zeros(3))
        with pytest.raises(ValueError):
            fn(SimpleMuData({"atac": SimpleAnnData(np.zeros((2, 4)), var=var)}))


@pytest.mark.parametrize("flags", [(False, False), (True, False), (True, True)])
@pytest.mark.parametrize("drop", [None, "top"])
def test_add_genes_peaks_groups_matches_reference(flags, drop):
    _, ref_add_genes, ref_add_ann, _ = _reference()
    import sys
    sys.path.insert(0, GOLDEN)
    import make_golden_rank as M
    X, scaled, labels = M.make_data()
    results = []
    for add_ann, add_genes in ((ref_add_ann, ref_add_genes), (atl.add_peak_annotation, atl.add_genes_peaks_groups)):
        ad = M.make_adata(X, scaled, labels)
        R.rank_genes_groups(ad, "leiden", n_genes=30)
        gone = None if drop is None else M.peak_names(X.shape[1]).index(ad.uns["rank_genes_groups"]["names"]["0"][0])
        add_ann(ad, pd.read_csv(io.StringIO(M.annotation_tsv(X.shape[1], gone)), sep="\t"))
        err = None
        try:
            add_genes(ad, add_peak_type=flags[0], add_distance=flags[1])
        except Exception as e:  # noqa: BLE001 -- compared with the reference's exception type
            err = type(e)
        results.append((err, ad.uns))
    assert results[0][0] == results[1][0]
    if drop is not None:
        assert results[0][0] is ValueError
    _uns_equal(results[0][1], results[1][1])
    for fn in (ref_add_genes, atl.add_genes_peaks_groups):
        with pytest.raises(KeyError):
            fn(SimpleAnnData(np.zeros((2, 2))))
