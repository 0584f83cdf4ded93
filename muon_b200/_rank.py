"""Differential testing of every peak per group on the GPU: scanpy's ``rank_genes_groups`` as muon's
``rank_peaks_groups`` calls it (muon/_atac/tools.py:371).

The statistics come from csrc/rank.cu over the CSR of Aᵀ: one CTA per peak sorts the peak's stored entries by value
(the implicit zeros are one tie block counted from the group sizes, never materialised) and sweeps them once for the
exact rank sums and tie terms, then sorts them by group for fixed-order moments; a second kernel turns those into the
t or z scores, p-values, log fold changes and detection fractions.  The multiple-testing correction and the top-n
selection are torch sorts on the device; only the G x n_genes results come back to the host.

Deliberate divergences from scanpy:
  * Ties in score are ordered by ascending peak index (numpy's argpartition / argsort leave that order unspecified).
  * A non-categorical ``groupby`` raises ValueError (scanpy fails inside pandas' ``.cat`` accessor).
  * ``method="logreg"``, more than ``RANK_MAX_GROUPS`` tested groups and a process group of more than one rank raise
    NotImplementedError before any device work.
"""
from __future__ import annotations

import numpy as np

from ._lib import (RANK_MAX_GROUPS, RANK_OVERESTIM_VAR, RANK_TIE_CORRECT, RANK_VS_GROUP, RANK_WILCOXON, call, load,
                   phase, ptr, stream_ptr)

METHODS = ("t-test", "t-test_overestim_var", "wilcoxon")
CORR_METHODS = ("benjamini-hochberg", "bonferroni")
SHORT_CLASSES = (512, 2048)       # shared-memory size classes below the kernel's capacity (a small row, a small CTA)
LONG_WORKSPACE = 1 << 30          # bytes of workspace slices for rows sorted in global memory
RANKED_CELLS_LIMIT = 2642245      # exact 64-bit tie terms sum(t^3 - t)


class Plan:
    """What a call tests, decided on the host before any device work.

    ``order`` the groups in scanpy's order (the user's list, plus the reference when it is missing from it); ``tested``
    the groups with results (``order`` without the reference); ``code`` [n] int32 = index into ``tested``, G for the
    other ranked cells (rest) or the reference, -1 for cells outside both (against a group); ``sizes`` [G + 1]."""

    def __init__(self, labels, groups, reference):
        import pandas as pd
        if not isinstance(labels.dtype, pd.CategoricalDtype):
            raise ValueError("rank_genes_groups: `groupby` must name a categorical column of `obs`")
        cats = [str(c) for c in labels.cat.categories]
        if reference != "rest" and str(reference) not in cats:
            raise ValueError(f"reference = {reference} needs to be one of groupby = {cats}.")
        if isinstance(groups, str) and groups == "all":
            order = list(cats)
        elif isinstance(groups, (str, int)):
            raise ValueError("Specify a sequence of groups")
        else:
            order = [str(g) for g in groups]
            if reference != "rest" and str(reference) not in order:
                order.append(str(reference))
            unknown = [g for g in order if g not in cats]
            if unknown:
                raise ValueError(f"groups {unknown} are not categories of groupby = {cats}")
        codes = np.asarray(labels.cat.codes, dtype=np.int64)
        counts = np.bincount(codes[codes >= 0], minlength=len(cats))
        pos = {c: i for i, c in enumerate(cats)}
        small = [g for g in order if counts[pos[g]] < 2]
        if small:
            raise ValueError(f"Could not calculate statistics for groups {', '.join(small)} since they only "
                             "contain one sample.")
        self.order = order
        self.reference = None if reference == "rest" else str(reference)
        self.tested = [g for g in order if g != self.reference]
        G = len(self.tested)
        if G > RANK_MAX_GROUPS:
            raise NotImplementedError(f"rank_genes_groups: {G} groups; at most {RANK_MAX_GROUPS} are supported")
        lut = np.full(len(cats) + 1, -1 if self.reference is not None else G, dtype=np.int32)   # last slot: NaN label
        for i, g in enumerate(self.tested):
            lut[pos[g]] = i
        if self.reference is not None:
            lut[pos[self.reference]] = G
        self.code = lut[codes]                          # codes of -1 (NaN) index the last slot
        self.sizes = np.bincount(self.code[self.code >= 0], minlength=G + 1).astype(np.int64)
        self.n_ranked = int(self.sizes.sum())


def _check_use_raw(adata, use_raw, layer):
    if use_raw is not None:
        return bool(use_raw)
    if layer is not None:
        return False
    return getattr(adata, "raw", None) is not None


def _mask_var(adata, mask_var, var_names):
    if mask_var is None:
        return None
    if isinstance(mask_var, str):
        mask_var = np.asarray(adata.var[mask_var])
    mask = np.asarray(mask_var)
    if mask.dtype != bool or mask.shape != (len(var_names),):
        raise ValueError("`mask_var` must be a boolean mask over the variables or the name of a boolean column of `var`")
    return mask


def device_matrix(X):
    """X as a DeviceCSR with float32 or float64 values (a DeviceCSR is used in place, a host matrix uploaded)."""
    import scipy.sparse as sp
    import torch

    from . import _device
    if isinstance(X, _device.DeviceCSR):
        if X.data.dtype in (torch.float32, torch.float64):
            return X
        return X.with_data(X.data.to(torch.float32))
    Xs = X if sp.issparse(X) else sp.csr_matrix(np.asarray(X))
    Xs = sp.csr_matrix(Xs)
    return _device.DeviceCSR.from_scipy(Xs, dtype=np.float64 if Xs.dtype == np.float64 else np.float32)


def peak_stats(A, plan: Plan, peaks, *, wilcoxon: bool, tie_correct: bool = False):
    """(stats [5][G + 1][len(peaks)] float64 of mub_rank_stats over the rows ``peaks`` of Aᵀ, the share of their stored
    entries that took the long-row path, the MUB_RANK_* flags).  Reuses a transpose cached on A, and caches none."""
    import torch

    from . import _device
    _device.require_cuda()
    dev = A.data.device
    if plan.n_ranked >= RANKED_CELLS_LIMIT:
        raise NotImplementedError(f"rank_genes_groups: {plan.n_ranked} ranked cells; fewer than {RANKED_CELLS_LIMIT} "
                                  "are supported")
    with phase("rank.transpose"):
        T = A._t if A._t is not None and A._t.data.dtype == A.data.dtype else _device.csr_transpose(A)
    K = len(plan.tested) + 1
    n_out = len(peaks)
    flags = (RANK_WILCOXON if wilcoxon else 0) | (RANK_VS_GROUP if plan.reference is not None else 0)
    flags |= RANK_TIE_CORRECT if tie_correct else 0
    stats = torch.empty((5, K, n_out), dtype=torch.float64, device=dev)
    if n_out == 0:
        return stats, 0.0, flags
    with phase("rank.stats"):
        code = torch.from_numpy(plan.code).to(dev)
        sizes = torch.from_numpy(plan.sizes).to(dev)
        rows = torch.as_tensor(np.asarray(peaks), dtype=torch.int64, device=dev)
        length = T.indptr[rows + 1] - T.indptr[rows]
        vb = T.data.element_size()
        cap_shared = int(load().mub_rank_shared_capacity(vb))
        fn = "mub_rank_stats_f64" if vb == 8 else "mub_rank_stats_f32"
        lo = -1
        long_entries = 0
        for cap in [c for c in SHORT_CLASSES if c < cap_shared] + [cap_shared, None]:
            sel = (length > lo) if cap is None else (length > lo) & (length <= cap)
            cols = torch.nonzero(sel).flatten()
            lo = cap if cap is not None else lo
            if cols.numel() == 0:
                continue
            r, c = rows[cols].to(torch.int32), cols.to(torch.int32)
            ws, ws_bytes = None, 0
            if cap is None:
                longest = int(length[cols].max())
                long_entries = int(length[cols].sum())
                cap = 1 << (longest - 1).bit_length()
                slice_bytes = int(load().mub_rank_workspace_slice_bytes(vb, cap))
                ws_bytes = max(1, min(cols.numel(), LONG_WORKSPACE // slice_bytes)) * slice_bytes
                ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
            call(fn, ptr(T.indptr), ptr(T.indices), ptr(T.data), ptr(code), ptr(r), ptr(c),
                 int(cols.numel()), n_out, K, ptr(sizes), plan.n_ranked, flags, cap, ptr(ws), ws_bytes, ptr(stats),
                 stream_ptr())
        total = int(length.sum())
    return stats, (long_entries / total if total else 0.0), flags


def score(stats, plan: Plan, flags: int, n_total: int, *, overestim_var=False, log_base=None, with_pts=False):
    """scores, pvals, logfoldchanges [G][n_out], pts [G + 1][n_out], pts_rest [G][n_out] (rest only) from mub_rank_score."""
    import torch
    K, n_out = stats.shape[1], stats.shape[2]
    G = K - 1
    dev = stats.device
    f64 = dict(dtype=torch.float64, device=dev)
    scores, pvals, lfc = (torch.empty((G, n_out), **f64) for _ in range(3))
    pts = torch.zeros((K, n_out), **f64)
    pts_rest = torch.empty((G, n_out), **f64) if with_pts and plan.reference is None else None
    flags |= RANK_OVERESTIM_VAR if overestim_var else 0
    sizes = torch.from_numpy(plan.sizes).to(dev)
    call("mub_rank_score", ptr(stats), K, n_out, ptr(sizes), n_total, flags,
         float(np.log(log_base)) if log_base is not None else 0.0, ptr(scores), ptr(pvals), ptr(lfc), ptr(pts),
         ptr(pts_rest), stream_ptr())
    return scores, pvals, lfc, pts, pts_rest


def adjust(pvals, corr_method: str):
    """Benjamini-Hochberg (scipy.stats.false_discovery_control) or Bonferroni over each row."""
    import torch
    n = pvals.shape[1]
    if corr_method == "bonferroni":
        return torch.clamp(pvals * n, max=1.0)
    order = torch.argsort(pvals, dim=1, stable=True)
    ps = torch.gather(pvals, 1, order) * (n / torch.arange(1, n + 1, dtype=torch.float64, device=pvals.device))
    ps = torch.flip(torch.cummin(torch.flip(ps, [1]), 1).values, [1]).clamp(0.0, 1.0)
    return torch.empty_like(ps).scatter_(1, order, ps)


def top(scores, n: int, rankby_abs: bool):
    """Indices of the n best scores of each row: descending score (|score|), ties by ascending peak index."""
    import torch
    key = scores.abs() if rankby_abs else scores
    return torch.sort(key, dim=1, descending=True, stable=True).indices[:, :n]


def rank_genes_groups(adata, groupby, *, mask_var=None, use_raw=None, groups="all", reference="rest", n_genes=None,
                      rankby_abs=False, pts=False, key_added=None, copy=False, method=None,
                      corr_method="benjamini-hochberg", tie_correct=False, layer=None, **kwds):
    """scanpy's ``rank_genes_groups`` (1.10 semantics) for t-test, t-test_overestim_var and wilcoxon on the GPU.

    Writes ``uns[key_added or "rank_genes_groups"]``: ``params`` and the recarrays ``names``, ``scores``, ``pvals``,
    ``pvals_adj``, ``logfoldchanges`` (one field per tested group), plus ``pts`` / ``pts_rest`` DataFrames with
    ``pts=True``.  Returns the copy with ``copy=True``, else None."""
    import pandas as pd
    import torch

    from . import _dist, _device
    if kwds:
        raise TypeError(f"rank_genes_groups() got unexpected keyword arguments: {sorted(kwds)}")
    if method is None:
        method = "t-test"
    if method == "logreg":
        raise NotImplementedError("rank_genes_groups: method='logreg' is not supported")
    if method not in METHODS:
        raise ValueError(f"Method must be one of {METHODS}.")
    if corr_method not in CORR_METHODS:
        raise ValueError(f"Correction method must be one of {CORR_METHODS}.")
    if _dist.is_distributed() and _dist.world_size() > 1:
        raise NotImplementedError("rank_genes_groups: ranks over cell shards of several processes are not supported")
    if copy:
        adata = adata.copy()
    use_raw = _check_use_raw(adata, use_raw, layer)
    if layer is not None and use_raw:
        raise ValueError("Cannot specify `layer` and have `use_raw=True`.")
    if groupby not in adata.obs.columns:
        raise KeyError(f"groupby = {groupby!r} is not a column of obs")
    plan = Plan(adata.obs[groupby], groups, reference)
    if use_raw:
        X, var_names = adata.raw.X, adata.raw.var_names
    elif layer is not None:
        X, var_names = adata.layers[layer], adata.var_names
    else:
        X, var_names = adata.X, adata.var_names
    mask = _mask_var(adata, mask_var, var_names)
    peaks = np.arange(X.shape[1]) if mask is None else np.flatnonzero(mask)
    names_all = np.asarray(var_names, dtype=object)[peaks]
    n_tested = len(peaks)
    n_top = n_tested if n_genes is None or n_genes > n_tested else int(n_genes)
    log1p = adata.uns.get("log1p", {}) if hasattr(adata.uns, "get") else {}
    base = log1p.get("base") if isinstance(log1p, dict) else None

    A = device_matrix(X)
    if isinstance(A, _device.DeviceCSR) and (A.row0 != 0 or A.n_total != A.shape[0]):
        raise NotImplementedError("rank_genes_groups: a cell shard of a larger matrix cannot be ranked on its own")
    stats, _, flags = peak_stats(A, plan, peaks, wilcoxon=method == "wilcoxon", tie_correct=tie_correct)
    with phase("rank.score"):
        scores, pvals, lfc, pts_t, pts_rest_t = score(stats, plan, flags, A.shape[0],
                                                      overestim_var=method == "t-test_overestim_var", log_base=base,
                                                      with_pts=pts)
        adj = adjust(pvals, corr_method)
        idx = top(scores, n_top, rankby_abs)
        picked = torch.stack([torch.gather(t, 1, idx) for t in (scores, pvals, adj, lfc)])
    with phase("rank.assemble"):
        picked = picked.cpu().numpy()
        idx = idx.cpu().numpy()
        G = len(plan.tested)
        dtypes = {"names": "O", "scores": "float32", "logfoldchanges": "float32", "pvals": "float64",
                  "pvals_adj": "float64"}
        cols = {"names": [names_all[idx[g]] for g in range(G)], "scores": picked[0], "pvals": picked[1],
                "pvals_adj": picked[2], "logfoldchanges": picked[3]}
        key = key_added or "rank_genes_groups"
        out = {"params": dict(groupby=groupby, reference=reference, method=method, use_raw=use_raw, layer=layer,
                              corr_method=corr_method)}
        if pts:
            rowof = {g: i for i, g in enumerate(plan.tested)}
            if plan.reference is not None:
                rowof[plan.reference] = G
            P = pts_t.cpu().numpy()
            out["pts"] = pd.DataFrame(P[[rowof[g] for g in plan.order]].T, index=names_all, columns=plan.order)
            if pts_rest_t is not None:
                out["pts_rest"] = pd.DataFrame(pts_rest_t.cpu().numpy().T, index=names_all, columns=plan.order)
        for col in ("logfoldchanges", "names", "pvals", "pvals_adj", "scores"):      # what DataFrame.to_records makes
            out[col] = np.rec.fromarrays([np.asarray(a, dtype=dtypes[col]) for a in cols[col]],
                                         dtype=[(g, dtypes[col]) for g in plan.tested])
        adata.uns[key] = out
    return adata if copy else None
