"""``mu.atac.tl`` -- ATAC tools.  ``lsi`` and ``rank_peaks_groups`` run on the GPU; the peak annotation helpers are pandas."""
from __future__ import annotations

import numpy as np

from .._containers import is_anndata, is_mudata


def lsi(data, scale_embeddings=True, n_comps=50, *, tol: float = 1e-5, seed: int = 0, return_info: bool = False):
    """Run Latent Semantic Indexing -- drop-in for ``muon.atac.tl.lsi``
    (reference muon/_atac/tools.py:29-71).

    Writes ``adata.obsm["X_lsi"]`` (n x k; z-scored left singular vectors when
    ``scale_embeddings``), ``adata.uns["lsi"]["stdev"]`` (singular values / sqrt(n-1)) and
    ``adata.varm["LSI"]`` (d x k right singular vectors), components in descending order,
    signs arbitrary (as with ARPACK).  Returns ``None``.

    The truncated SVD is a block Golub-Kahan-Lanczos iteration (``_lsi.py``) whose passes over
    the matrix are the CUDA SpMM kernels; ``tol`` (keyword-only, not in the reference) is the
    relative residual at which the k triplets are accepted -- the default makes singular values
    agree with ``scipy.sparse.linalg.svds`` to ~1e-7 and gap-resolved vectors to ~1e-5.
    """
    import torch

    from .. import _device, _dist
    from .._lib import phase
    from .._lsi import CsrOperator, truncated_svd

    if is_anndata(data):
        adata = data
    elif is_mudata(data) and "atac" in data.mod:
        adata = data.mod["atac"]
    else:
        raise TypeError("Expected AnnData or MuData object with 'atac' modality")

    X = adata.X
    n_comps = min(n_comps, X.shape[1])  # tools.py:50
    resident = isinstance(X, _device.DeviceCSR)
    if resident:
        A = X
        if A.data.dtype != torch.float32:
            A = A.with_data(A.data.to(torch.float32))
    else:
        import scipy.sparse as sp
        Xs = X if sp.issparse(X) else sp.csr_matrix(np.asarray(X))
        Xs = Xs.tocsr()  # row order inside a row is irrelevant to the SpMM kernels
        # tfidf() may have left a device twin of this matrix.  It is used only if EVERY host element still equals
        # what was downloaded; that check (a threaded read pass over the host arrays, GIL released) runs on a helper
        # thread while the device already works on the twin, and a mismatch discards that work for a fresh upload.
        cand = _device.resident_candidate(Xs)
        check = None
        if cand is not None:
            from concurrent.futures import ThreadPoolExecutor
            A = cand[0]
            pool = ThreadPoolExecutor(1)
            check = pool.submit(_device.resident_valid, Xs, cand[1])
            pool.shutdown(wait=False)
        else:
            A = _device.DeviceCSR.from_scipy(Xs, dtype=np.float32)
    n_total = A.n_total
    if n_comps >= min(n_total, A.shape[1]):  # svds' own requirement, scipy _svds.py:40-44
        if not resident and check is not None:
            check.result()
        raise ValueError(f"`k` must be an integer satisfying `0 < k < min(A.shape)` (k={n_comps})")

    P = _device.pad_width(min(n_comps + 8, 128) if n_comps + 8 <= 128 else n_comps)

    def solve(A):
        op = CsrOperator(A, P)
        return truncated_svd(op, n_comps, P, tol=tol, seed=seed)

    U, s, V, info = solve(A)
    if not resident:
        if check is not None and not check.result():          # the host matrix was edited after tfidf(): start over
            A._tp = None
            _device.release_resident(Xs)
            del U, s, V
            A = _device.DeviceCSR.from_scipy(Xs, dtype=np.float32)
            U, s, V, info = solve(A)
        # the matrix on the device is a hidden copy (fresh upload or the twin left by tfidf): do not leave the
        # 8 B/nnz transposed panels cached on it; a DeviceCSR the caller owns keeps them for the next call (mofa)
        A._tp = None
    if not info.converged:
        from warnings import warn
        warn(f"lsi: stopped after {info.passes} passes at relative residual {max(info.residuals):.1e} > tol={tol:g} "
             "(clustered singular values around the k-th component?); the leading components are still accurate")

    # post-processing of tools.py:60-65 on the device (moments allreduced over cell shards)
    with phase("lsi.post_and_d2h"):
        emb = U
        if scale_embeddings:
            mom = torch.stack([U.sum(0, dtype=torch.float64), (U.to(torch.float64) ** 2).sum(0)])
            _dist.all_reduce_sum_(mom)
            mean = mom[0] / n_total
            std = (mom[1] / n_total - mean**2).clamp_min(0).sqrt()     # numpy std, ddof=0
            emb = ((U.to(torch.float64) - mean) / std).to(torch.float32)
        stdev = s / np.sqrt(n_total - 1)

        out_dtype = np.float32 if resident or X.dtype == np.float32 else np.float64
        adata.obsm["X_lsi"] = _device.to_host(emb.contiguous()).astype(out_dtype, copy=False)
        adata.uns["lsi"] = {"stdev": stdev.cpu().numpy().astype(out_dtype, copy=False)}
        adata.varm["LSI"] = _device.to_host(V.contiguous()).astype(out_dtype, copy=False)
    if return_info:
        return info
    return None


def _atac_of(data):
    if is_anndata(data):
        return data
    if is_mudata(data) and "atac" in data.mod:
        return data.mod["atac"]
    raise TypeError("Expected AnnData or MuData object with 'atac' modality")


def add_peak_annotation(data, annotation, sep="\t", return_annotation=False):
    """Store a peak annotation table in ``uns["atac"]["peak_annotation"]`` -- drop-in for
    ``muon.atac.tl.add_peak_annotation`` (reference muon/_atac/tools.py:83-165).  Host-only (pandas).

    ``annotation`` is a DataFrame or a path read with ``sep``; it needs ``gene``, ``distance`` and ``peak_type`` and
    either ``peak`` (``chrX_1_2`` is rewritten ``chrX:1-2``) or ``chrom``/``start``/``end``.  Rows listing several genes
    as ``;``-separated strings become one row per gene.  The stored table is indexed by gene, with ``peak``,
    ``distance`` (integers where every value is one) and ``peak_type``; missing strings become ``""``."""
    import pandas as pd

    adata = _atac_of(data)
    table = annotation if isinstance(annotation, pd.DataFrame) else pd.read_csv(annotation, sep=sep)
    table = table.convert_dtypes()
    if "peak" in table.columns:
        table["peak"] = table["peak"].str.replace("_", ":", n=1).str.replace("_", "-", n=1)
    elif {"chrom", "start", "end"} <= set(table.columns):
        table["peak"] = (table["chrom"].astype(str) + ":" + table["start"].astype(str) + "-"
                         + table["end"].astype(str))
    else:
        raise AttributeError("Peak annotation does not in contain neighter peak column nor chrom, start, and end "
                             "columns.")
    if pd.api.types.is_string_dtype(table["distance"]):
        # one row per gene of the ';'-separated lists, aligned on the peak
        by_peak = table.set_index("peak")
        parts = [by_peak["gene"].str.split(";").explode(),
                 by_peak["distance"].str.split(";").explode().astype(int),
                 by_peak["peak_type"].str.split(";").explode()]
        table = pd.concat(parts, axis=1).reset_index()
    else:
        table = table[["peak", "gene", "distance", "peak_type"]]
    try:
        table["distance"] = table["distance"].astype(int)
    except ValueError:          # missing distances (intergenic rows) keep the nullable integer type
        pass
    for name in ("peak", "gene", "peak_type"):
        table[name] = table[name].fillna("").astype(object)
    table = table.set_index("gene")
    adata.uns.setdefault("atac", dict())
    adata.uns["atac"]["peak_annotation"] = table
    if return_annotation:
        return table


def add_peak_annotation_gene_names(data, gene_names=None, join_on=None, return_annotation=False):
    """Re-index the peak annotation on gene names -- drop-in for ``muon.atac.tl.add_peak_annotation_gene_names``
    (reference muon/_atac/tools.py:168-247).  Host-only (pandas).

    ``gene_names`` is indexed by gene name and holds the annotation's current index in column ``join_on`` (default
    ``gene_ids``); for a MuData it defaults to ``mod["rna"].var``.  When no annotation key is found in that column but
    some are gene names already, the index is only renamed ``gene_name``."""
    if is_anndata(data):
        adata = data
    elif is_mudata(data) and "atac" in data.mod:
        adata = data.mod["atac"]
        if gene_names is None:
            if "rna" not in data.mod:
                raise ValueError("There is no .mod['rna'] modality. Provide `gene_names` as a pd.DataFrame.")
            gene_names = data.mod["rna"].var
    else:
        raise TypeError("Expected AnnData or MuData object with 'atac' modality")
    if "peak_annotation" not in adata.uns.get("atac", {}):
        raise KeyError("There is no peak annotation yet. Run muon.atac.tl.add_peak_annotation first.")
    ann = adata.uns["atac"]["peak_annotation"]
    join_on = "gene_ids" if join_on is None else join_on
    id_to_name = gene_names.loc[:, [join_on]].rename_axis("gene_name").reset_index(drop=False).set_index(join_on)
    if len(np.intersect1d(ann.index.values, id_to_name.index.values)) == 0:
        if len(np.intersect1d(ann.index.values, gene_names.index.values)) != 0:
            ann.index.names = ["gene_name"]
            adata.uns["atac"]["peak_annotation"] = ann
        return ann if return_annotation else None
    ann = ann.join(id_to_name).rename_axis(join_on).reset_index(drop=False)
    ann.loc[ann["gene_name"].isnull(), "gene_name"] = ""
    ann = ann.set_index("gene_name")
    adata.uns["atac"]["peak_annotation"] = ann
    if return_annotation:
        return ann


def add_genes_peaks_groups(data, add_peak_type=False, add_distance=False):
    """Join the annotated genes onto the ranked peaks -- drop-in for ``muon.atac.tl.add_genes_peaks_groups``
    (reference muon/_atac/tools.py:251-334).  Host-only (pandas).

    Needs ``uns["rank_genes_groups"]`` and ``uns["atac"]["peak_annotation"]``.  For each group, the ranked names are
    inner-joined to the annotation in rank order and the genes of a peak joined with ``", "``: ``genes`` is a recarray
    (one field per group); ``peak_type`` / ``distance`` (dicts of arrays) are added on request.  A ranked peak missing
    from the annotation leaves the groups with unequal lengths, and building ``genes`` raises ValueError."""
    import pandas as pd

    adata = _atac_of(data)
    if "rank_genes_groups" not in adata.uns:
        raise KeyError("There is no .uns['rank_genes_groups'] yet. Run sc.tl.rank_genes_groups first.")
    if "peak_annotation" not in adata.uns.get("atac", {}):
        raise KeyError("There is no peak annotation yet. Run muon.atac.pp.add_peak_annotation first.")
    annotation = adata.uns["atac"]["peak_annotation"]
    if "peak" not in annotation.columns:
        raise KeyError("Peak annotation has to contain 'peak' column.")
    result = adata.uns["rank_genes_groups"]
    gene_col = annotation.index.name
    extra = [("peak_type", add_peak_type), ("distance", add_distance)]
    for name, wanted in extra:
        if wanted:
            if name not in annotation.columns:
                raise KeyError(f"Peak annotation has to contain '{name}' column.")
            result[name] = {}
    if add_distance:
        annotation.distance = annotation.distance.astype(str)      # joined as strings (stored back, as the reference)
    keep = [gene_col] + [name for name, wanted in extra if wanted]
    by_peak = annotation.reset_index(drop=False).loc[:, ["peak", *keep]].set_index("peak")
    genes = {}
    for group in result["names"].dtype.names:
        ranked = pd.DataFrame(result["names"][group]).rename({0: "peak"}, axis=1)
        joined = ranked.join(by_peak, on="peak", how="inner", sort=False).groupby("peak", sort=False).agg(", ".join)
        genes[group] = joined[gene_col].values
        for name, wanted in extra:
            if wanted:
                result[name][group] = joined[name].values
    result["genes"] = genes
    result["genes"] = pd.DataFrame(genes).to_records(index=False)


def rank_peaks_groups(data, groupby, add_peak_type=False, add_distance=False, **kwargs):
    """Rank peaks per group and name their genes -- drop-in for ``muon.atac.tl.rank_peaks_groups``
    (reference muon/_atac/tools.py:337-373): ``rank_genes_groups`` on the GPU (``muon_b200._rank``), then
    ``add_genes_peaks_groups``.

    ``kwargs`` are those of scanpy's ``rank_genes_groups`` (``mask_var, use_raw, groups, reference, n_genes,
    rankby_abs, pts, key_added, copy, method, corr_method, tie_correct, layer``); any other name raises TypeError.
    ``method`` is ``"t-test"`` (default), ``"t-test_overestim_var"`` or ``"wilcoxon"``; ``"logreg"`` raises
    NotImplementedError.  A MuData's ``mod["atac"]`` is used without a membership check (KeyError when missing)."""
    from .._rank import rank_genes_groups

    if is_anndata(data):
        adata = data
    elif is_mudata(data):
        adata = data.mod["atac"]
    else:
        raise TypeError("Expected AnnData or MuData object with 'atac' modality")
    rank_genes_groups(adata, groupby, **kwargs)
    add_genes_peaks_groups(adata, add_peak_type=add_peak_type, add_distance=add_distance)
