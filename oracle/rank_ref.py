"""float64 numpy / scipy restatement of scanpy's ``rank_genes_groups`` as muon's ``rank_peaks_groups`` calls it
(muon/_atac/tools.py:371), and a loader that runs the reference's ``muon/_atac/tools.py`` with it in place of scanpy.

scanpy is not vendored and not installable here; every item below is recalled from scanpy 1.10 and marked so.
  * [recalled] Signature ``rank_genes_groups(adata, groupby, *, mask_var=None, use_raw=None, groups="all",
    reference="rest", n_genes=None, rankby_abs=False, pts=False, key_added=None, copy=False, method=None,
    corr_method="benjamini-hochberg", tie_correct=False, layer=None, **kwds)``; ``method=None`` is ``"t-test"``.
  * [recalled] ``use_raw=None`` means ``.raw`` when present (and not with a ``layer``); ``n_genes=None`` (or more than
    the peaks) means every tested peak.  Groups follow the user's list, the reference appended when missing from it;
    the reference group gets no results.  A selected group (or the reference) with fewer than 2 cells raises
    ValueError, as does a reference that is not a category.
  * [recalled] Moments in float64: mean, and var = (mean of x^2 - mean^2) * n / (n - 1), x^2 taken in the input dtype.
    Rest = every cell outside the group.  ``logfoldchanges = log2((expm1(m_g) + 1e-9) / (expm1(m_rest) + 1e-9))``,
    expm1(x ln base) with ``uns["log1p"]["base"]``.
  * [recalled] t-test: ``scipy.stats.ttest_ind_from_stats(..., equal_var=False)``; ``t-test_overestim_var`` uses the
    group's n for the rest; NaN score -> 0, NaN p -> 1.
  * [recalled] wilcoxon, rest: ranks (``rankdata``, average ties) over all cells, z = (R_g - n_g (n+1)/2) /
    sqrt(T n_g (n - n_g) (n+1) / 12); against a group r: ranks over g then r, n_g, m_r, n_g + m_r + 1 in the formula;
    T = 1 - sum(t^3 - t) / (N^3 - N) over the ranked cells with ``tie_correct``, else 1; NaN z -> 0;
    p = 2 norm.sf(|z|).
  * [recalled] Benjamini-Hochberg over all tested peaks of a group (NaN p -> 1), or Bonferroni min(p n, 1); the top
    ``n_genes`` by descending score (|score| with ``rankby_abs``) via ``np.argpartition`` then ``np.argsort``.
  * [recalled] ``uns[key_added or "rank_genes_groups"]``: ``params`` (groupby, reference, method, use_raw, layer,
    corr_method) and recarrays names / scores / pvals / pvals_adj / logfoldchanges with dtypes object, float32,
    float64, float64, float32; with ``pts``, DataFrames ``pts`` (every group in order, reference included) and
    ``pts_rest`` (rest only) of the fraction of cells with a stored non-zero.
  * [recalled] A non-categorical ``groupby`` fails (here: ValueError); ``logreg`` is not restated (NotImplementedError).
"""
from __future__ import annotations

import os
import sys
import types

import numpy as np
from scipy import stats

CHUNK = 512


def _dense(X, cols):
    import scipy.sparse as sp
    sub = X[:, cols]
    return np.asarray(sub.toarray() if sp.issparse(sub) else sub)


def tie_term(ranks):
    """sum over tie blocks of t^3 - t, per column of a rank matrix, as exact Python ints (an object array): t^3 wraps
    int64 from t = 2 097 153 on, and the sum of a column exceeds it even earlier."""
    out = np.zeros(ranks.shape[1], dtype=object)
    for j in range(ranks.shape[1]):
        _, t = np.unique(ranks[:, j], return_counts=True)
        out[j] = sum(int(c) ** 3 - int(c) for c in t)
    return out


def bh(p):
    return stats.false_discovery_control(p, method="bh")


def select_top_n(scores, n_top):
    part = np.argpartition(scores, -n_top)[-n_top:]
    return part[np.argsort(scores[part])[::-1]]


def groups_setup(labels, groups, reference):
    import pandas as pd
    if not isinstance(labels.dtype, pd.CategoricalDtype):
        raise ValueError("groupby must be categorical")
    cats = [str(c) for c in labels.cat.categories]
    if reference != "rest" and str(reference) not in cats:
        raise ValueError(f"reference = {reference} needs to be one of groupby = {cats}.")
    if isinstance(groups, str) and groups == "all":
        order = list(cats)
    else:
        order = [str(g) for g in groups]
        if reference != "rest" and str(reference) not in order:
            order.append(str(reference))
    values = np.asarray(labels.astype(str).values, dtype=object)
    valid = np.asarray(labels.notna())
    masks = np.stack([(values == g) & valid for g in order])
    small = [g for g, m in zip(order, masks) if m.sum() < 2]
    if small:
        raise ValueError(f"Could not calculate statistics for groups {', '.join(small)} since they only contain one sample.")
    return order, masks


def group_stats(X, masks, ref=None, tie_correct=True):
    """Per (group, peak) over the groups of ``masks`` (the reference row ``ref`` skipped): stored non-zeros, sums,
    sums of squares (float64 of squares in the input dtype), the Wilcoxon rank sums (ranks over all cells, or over
    g then the reference) and tie terms.  float64 arrays [len(masks)][d]."""
    d = X.shape[1]
    G = len(masks)
    out = {k: np.zeros((G, d)) for k in ("cnt", "sum", "sumsq", "ranksum", "tie")}
    for c0 in range(0, d, CHUNK):
        cols = np.arange(c0, min(d, c0 + CHUNK))
        Xc = _dense(X, cols)
        sq = (Xc * Xc).astype(np.float64)
        if ref is None:
            R = stats.rankdata(Xc, axis=0).astype(np.float64)      # rankdata keeps float32; ranks sum in float64
            T = tie_term(R) if tie_correct else np.zeros(len(cols))
        for g, m in enumerate(masks):
            out["cnt"][g, cols] = (Xc[m] != 0).sum(0)
            out["sum"][g, cols] = Xc[m].astype(np.float64).sum(0)
            out["sumsq"][g, cols] = sq[m].sum(0)
            if ref is None:
                out["ranksum"][g, cols] = R[m].sum(0)
                out["tie"][g, cols] = T
            elif g != ref:
                Rg = stats.rankdata(np.vstack([Xc[m], Xc[masks[ref]]]), axis=0).astype(np.float64)
                out["ranksum"][g, cols] = Rg[: m.sum()].sum(0)
                out["tie"][g, cols] = tie_term(Rg) if tie_correct else 0
    return out


def rank_genes_groups(adata, groupby, *, mask_var=None, use_raw=None, groups="all", reference="rest", n_genes=None,
                      rankby_abs=False, pts=False, key_added=None, copy=False, method=None,
                      corr_method="benjamini-hochberg", tie_correct=False, layer=None, **kwds):
    import pandas as pd
    if method is None:
        method = "t-test"
    if method == "logreg":
        raise NotImplementedError("logreg is not restated")
    if method not in ("t-test", "t-test_overestim_var", "wilcoxon"):
        raise ValueError("bad method")
    if copy:
        adata = adata.copy()
    if use_raw is None:
        use_raw = layer is None and getattr(adata, "raw", None) is not None
    if layer is not None and use_raw:
        raise ValueError("Cannot specify `layer` and have `use_raw=True`.")
    order, masks = groups_setup(adata.obs[groupby], groups, reference)
    if use_raw:
        X, var_names = adata.raw.X, adata.raw.var_names
    elif layer is not None:
        X, var_names = adata.layers[layer], adata.var_names
    else:
        X, var_names = adata.X, adata.var_names
    var_names = np.asarray(var_names, dtype=object)
    if mask_var is not None:
        mv = np.asarray(adata.var[mask_var]) if isinstance(mask_var, str) else np.asarray(mask_var)
        X = X[:, np.flatnonzero(mv)]
        var_names = var_names[mv]
    n, d = X.shape
    n_top = d if n_genes is None or n_genes > d else n_genes
    ref = None if reference == "rest" else order.index(str(reference))
    st = group_stats(X, masks, ref, tie_correct=tie_correct and method == "wilcoxon")
    log1p = adata.uns.get("log1p", {})
    base = log1p.get("base") if isinstance(log1p, dict) else None
    expm1 = (lambda x: np.expm1(x * np.log(base))) if base is not None else np.expm1
    tot = {k: st[k].sum(0) for k in ("cnt", "sum", "sumsq")}
    ns = masks.sum(1)

    def moments(g):
        ng = ns[g]
        mean = st["sum"][g] / ng
        var = (st["sumsq"][g] / ng - mean**2) * (ng / (ng - 1))
        return mean, var, ng

    def rest_moments(g):
        if ref is not None:
            return moments(ref) + (st["cnt"][ref],)
        nr = n - ns[g]
        mean = (tot["sum"] - st["sum"][g]) / nr
        var = ((tot["sumsq"] - st["sumsq"][g]) / nr - mean**2) * (nr / (nr - 1))
        return mean, var, nr, tot["cnt"] - st["cnt"][g]

    res = {k: {} for k in ("names", "scores", "pvals", "pvals_adj", "logfoldchanges")}
    pts_df = np.zeros((len(order), d))
    pts_rest = np.zeros((len(order), d))
    for g, name in enumerate(order):
        mg, vg, ng = moments(g)
        mr, vr, nr, cnt_r = rest_moments(g)
        pts_df[g] = st["cnt"][g] / ng
        if ref is None:
            pts_rest[g] = cnt_r / nr
        if g == ref:
            continue
        with np.errstate(divide="ignore", invalid="ignore"):
            if method == "wilcoxon":
                N = n if ref is None else ng + nr
                T = 1.0 - st["tie"][g] / (float(N) ** 3 - N) if tie_correct else 1.0
                sd = np.sqrt(T * ng * (N - ng) * (N + 1) / 12.0)
                sc = (st["ranksum"][g] - ng * ((N + 1) / 2.0)) / sd
                sc[np.isnan(sc)] = 0
                pv = 2 * stats.norm.sf(np.abs(sc))
            else:
                n2 = ng if method == "t-test_overestim_var" else nr
                sc, pv = stats.ttest_ind_from_stats(mean1=mg, std1=np.sqrt(vg), nobs1=ng, mean2=mr, std2=np.sqrt(vr),
                                                    nobs2=n2, equal_var=False)
                sc = np.asarray(sc, dtype=np.float64)
                pv = np.asarray(pv, dtype=np.float64)
                sc[np.isnan(sc)] = 0
                pv[np.isnan(pv)] = 1
            lfc = np.log2((expm1(mg) + 1e-9) / (expm1(mr) + 1e-9))
        pv[np.isnan(pv)] = 1
        adj = bh(pv) if corr_method == "benjamini-hochberg" else np.minimum(pv * d, 1.0)
        idx = select_top_n(np.abs(sc) if rankby_abs else sc, n_top)
        res["names"][name] = var_names[idx]
        res["scores"][name] = sc[idx]
        res["pvals"][name] = pv[idx]
        res["pvals_adj"][name] = adj[idx]
        res["logfoldchanges"][name] = lfc[idx]
    key = key_added or "rank_genes_groups"
    out = {"params": dict(groupby=groupby, reference=reference, method=method, use_raw=use_raw, layer=layer,
                          corr_method=corr_method)}
    if pts:
        out["pts"] = pd.DataFrame(pts_df.T, index=var_names, columns=order)
        if ref is None:
            out["pts_rest"] = pd.DataFrame(pts_rest.T, index=var_names, columns=order)
    dtypes = {"names": "O", "scores": "float32", "logfoldchanges": "float32", "pvals": "float64", "pvals_adj": "float64"}
    for col in ("logfoldchanges", "names", "pvals", "pvals_adj", "scores"):
        out[col] = pd.DataFrame(res[col]).to_records(index=False, column_dtypes=dtypes[col])
    adata.uns[key] = out
    return adata if copy else None


def load_reference_rank_peaks_groups():
    """The reference's own ``rank_peaks_groups``, ``add_genes_peaks_groups``, ``add_peak_annotation`` and
    ``add_peak_annotation_gene_names`` (muon/_atac/tools.py), executed unmodified with ``scanpy.tl.rank_genes_groups``
    = the restatement above."""
    from . import _refload
    _refload.load_reference_lsi()                        # stubs, package context and tools.py itself
    sc = sys.modules["scanpy"]
    sc.tl = getattr(sc, "tl", None) or types.ModuleType("scanpy.tl")
    sc.tl.rank_genes_groups = rank_genes_groups
    m = sys.modules["_refmuon._atac.tools"]
    return m.rank_peaks_groups, m.add_genes_peaks_groups, m.add_peak_annotation, m.add_peak_annotation_gene_names


def reference_signatures():
    """The four reference signatures, read from the source with ast."""
    import ast

    from ._refload import REF_ROOT
    tree = ast.parse(open(os.path.join(REF_ROOT, "muon/_atac/tools.py")).read())
    out = {}
    for name in ("rank_peaks_groups", "add_genes_peaks_groups", "add_peak_annotation", "add_peak_annotation_gene_names"):
        fn = next(f for f in tree.body if isinstance(f, ast.FunctionDef) and f.name == name)
        params = [a.arg for a in fn.args.args]
        defaults = [ast.unparse(v) for v in fn.args.defaults]
        out[name] = {"params": params, "defaults": defaults, "required": len(params) - len(defaults),
                     "var_keyword": fn.args.kwarg.arg if fn.args.kwarg else None}
    return out
