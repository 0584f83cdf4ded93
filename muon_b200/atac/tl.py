"""``mu.atac.tl`` -- ATAC tools.  ``lsi``, ``rank_peaks_groups``, the fragments-file tools (``count_fragments_features``,
``tss_enrichment``, ``nucleosome_signal``) and ``scan_sequences`` run on the GPU; the peak annotation helpers,
``locate_fragments``, ``locate_file``, ``locate_genome`` and ``get_sequences`` are host-only."""
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


# ---- the fragments file (muon/_atac/tools.py:640-1201) -----------------------------------------------------------------
def _new_anndata(X, obs, var):
    from .._containers import SimpleAnnData, _real
    cls = _real("AnnData", "anndata") or SimpleAnnData
    return cls(X=X, obs=obs, var=var)


def _gene_annotation_from_rna(data):
    """Gene coordinates from ``mod["rna"].var["interval"]`` (``chr:start-end``), as muon/_rna/utils.py:7-37 builds
    them: Chromosome, Start, End, gene_id, gene_name, indexed like ``var``."""
    import pandas as pd
    var = data.mod["rna"].var
    parts = [str(s).replace(":", "-", 1).split("-") for s in var["interval"]]
    table = pd.DataFrame(parts, columns=["Chromosome", "Start", "End"], index=var.index)
    table["gene_id"] = var["gene_ids"].values
    table["gene_name"] = var.index.values
    table = table.loc[~table["Start"].isnull()]
    table["Start"] = table["Start"].astype(int)
    table["End"] = table["End"].astype(int)
    return table


def _features_or_rna(data, features):
    if features is not None:
        return features
    if is_mudata(data) and "rna" in data.mod and "interval" in data.mod["rna"].var.columns:
        return _gene_annotation_from_rna(data)
    raise ValueError("Argument `features` is required. It should be a BED-like DataFrame with gene coordinates and "
                     "names.")


def _fragments_path(adata):
    if "files" not in adata.uns or "fragments" not in adata.uns["files"]:
        raise KeyError("There is no fragments file located yet. Run muon.atac.tl.locate_fragments first.")
    return adata.uns["files"]["fragments"]


def _integral(v, what):
    """A fetch bound as int64: integral floats are accepted (the default extension 2e3 makes them floats)."""
    a = np.asarray(v, dtype=np.float64) if np.asarray(v).dtype.kind == "f" else np.asarray(v)
    if a.dtype.kind == "f":
        if not np.all(np.isfinite(a)) or not np.all(a == np.floor(a)):
            raise TypeError(f"{what} must be integral")
    return a.astype(np.int64)


def _check_fetch(contig, lo, hi):
    """pysam's refusals of a region, before any device work: start > stop, start < 0."""
    bad = np.flatnonzero(lo > hi)
    if len(bad):
        i = bad[0]
        raise ValueError(f"invalid coordinates: start ({lo[i]}) > stop ({hi[i]})")
    bad = np.flatnonzero(lo < 0)
    if len(bad):
        raise ValueError(f"start out of range ({lo[bad[0]]})")
    if np.any(hi > (1 << 31) - 1):
        raise NotImplementedError("fetch bounds beyond int32 are not supported")


def _barcode_rows(adata, barcodes):
    """Barcode -> obs row as the reference's dict builds it: the ``barcodes`` column when it exists, else obs_names;
    a repeated barcode maps to its last row."""
    keys = adata.obs.loc[:, barcodes] if barcodes and barcodes in adata.obs.columns else adata.obs.index
    if len(keys) > (1 << 31) - 1:
        raise NotImplementedError("more than 2^31 - 1 cells")
    return {k: v for v, k in enumerate(keys)}


def _device():
    import torch
    if not torch.cuda.is_available():
        from .._lib import MuonB200Error
        raise MuonB200Error("the fragments tools run on a CUDA device and none is available")
    return torch.device("cuda", torch.cuda.current_device())


def locate_fragments(data, fragments, return_fragments=False):
    """Record the fragments file in ``uns["files"]["fragments"]`` -- drop-in for ``muon.atac.tl.locate_fragments``
    (reference muon/_atac/tools.py:640-690).  Like the reference, any exception is printed and the call returns None.

    Deliberate divergence: the path is recorded when the file opens; neither pysam nor a ``.tbi`` index is needed.
    ``return_fragments=True`` returns ``pysam.TabixFile(fragments, parser=pysam.asBed())``, which does need pysam."""
    try:
        adata = _atac_of(data)
        with open(fragments, "rb"):
            pass
        if "files" not in adata.uns:
            adata.uns["files"] = dict()
        adata.uns["files"]["fragments"] = fragments
        if return_fragments:
            try:
                import pysam
            except ImportError:
                raise ImportError("pysam is not available. It is required to return a connection to the fragments "
                                  "file. Install pysam from PyPI (`pip install pysam`).")
            return pysam.TabixFile(fragments, parser=pysam.asBed())
    except Exception as e:   # noqa: BLE001 -- the reference prints every failure
        print(e)


def count_fragments_features(data, features=None, stranded=False, extend_upstream=2e3, extend_downstream=0,
                             count_reads=True, *, chunk_bytes=None):
    """Count the fragments overlapping each feature -- drop-in for ``muon.atac.tl.count_fragments_features``
    (reference muon/_atac/tools.py:746-891).  Returns a cells x features AnnData (``obs`` = the ATAC obs, ``var`` =
    ``features``) whose X is a canonical int64 CSR: duplicates summed, indices sorted (the reference returns a CSC with
    duplicate, unsorted entries; the two are equal once densified).

    The whole file is parsed on the device (``muon_b200._fragments``); one warp per feature window counts the
    overlapping fragments.  Each fragment adds ``int(score)`` (``count_reads``) or 1.  The window is ``[start -
    extend_upstream, end + extend_downstream)`` for every feature: as in the reference, ``stranded`` is replaced by
    whether a ``Strand`` column exists and the strand is read from the chromosome column, so no feature is ever
    treated as on the ``-`` strand, and a ``Strand`` column with ``stranded=False`` raises KeyError.  A window starting
    below 0 or on a contig the file lacks raises ValueError, as pysam's fetch does.  Non-unique ``obs_names`` raise
    ValueError.  ``chunk_bytes`` (keyword-only) sets the text per device chunk."""
    import warnings

    from .. import _fragments as F

    adata = _atac_of(data)
    features = _features_or_rna(data, features)
    path = _fragments_path(adata)
    if count_reads:
        warnings.warn("From v0.2, by default, unique fragments will be counted instead of reads. See muon#110 for "
                      "details.", FutureWarning, stacklevel=2)
    names = [str(c).lower() for c in features.columns.values]
    for col in ("start", "end"):
        if col not in names:
            raise ValueError(f"No column with feature {col}s could be found")
    chrom = next((c for c in ("chromosome", "chrom", "chr") if c in names), None)
    if chrom is None:
        raise ValueError("No column with chromosome for features could be found")
    column = {key: features.columns.values[names.index(key)] for key in ("start", "end", chrom)}
    strand_col = None
    if stranded:
        if "strand" not in names:
            raise ValueError("No column with strand for features could be found")
        strand_col = column[chrom]                       # the reference reads the strand from the chromosome column
    stranded = "Strand" in features.columns
    if stranded and strand_col is None and features.shape[0]:
        raise KeyError(None)
    contig = [str(c) for c in features[column[chrom]].values]
    start = _integral(features[column["start"]].values, "start")
    end = _integral(features[column["end"]].values, "end")
    minus = np.asarray(features[strand_col].values == "-", dtype=bool) if stranded else np.zeros(len(contig), bool)
    up, down = extend_upstream, extend_downstream
    lo = np.where(minus, _integral(start - down, "start"), _integral(start - up, "start"))
    hi = np.where(minus, _integral(end + up, "end"), _integral(end + down, "end"))
    _check_fetch(contig, lo, hi)
    if not adata.obs.index.is_unique:
        raise ValueError("count_fragments_features needs unique obs_names")
    index_of = _barcode_rows(adata, None)

    device = _device()
    R = F.read_records(path, index_of, device, chunk_bytes=chunk_bytes or F.CHUNK_BYTES)
    missing = [c for c in dict.fromkeys(contig) if c not in R.contigs]
    if missing:
        raise ValueError(f"could not create iterator for region '{missing[0]}': contig not in the fragments file")
    X = F.count_matrix(R, list(zip(contig, lo.tolist(), hi.tolist())), adata.n_obs, count_reads, device)
    return _new_anndata(X, adata.obs, features)


def tss_enrichment(data, features=None, extend_upstream=1000, extend_downstream=1000, n_tss=2000, return_tss=True,
                   random_state=None, barcodes=None, *, use_index=True, chunk_bytes=None):
    """TSS enrichment per cell (ENCODE) -- drop-in for ``muon.atac.tl.tss_enrichment`` (reference
    muon/_atac/tools.py:894-1106).  Adds ``obs["tss_score"]`` and returns (``return_tss``) an AnnData whose X is the
    cells x positions pileup divided by each cell's flank mean (float64) and whose ``var`` holds ``TSS_position``.

    More than ``n_tss`` features are sampled with ``features.sample(n=n_tss, random_state=random_state)``, as in the
    reference; features on contigs the file lacks are dropped.  Fragments with score s add s to the positions they
    cover in ``[Start - extend_upstream, Start + extend_downstream]``.  Flanks are the first and last 100 positions,
    the centre the middle 1001 (empty, hence NaN scores, when the region is exactly 1001 wide; ValueError when it is
    narrower); a zero flank mean is replaced by the mean over cells.

    With ``<file>.tbi`` present (``use_index``, keyword-only) only the windows are read, through the tabix linear
    index; otherwise the whole file is parsed.  The pileup is an exact int64 difference array on the device."""
    import warnings

    import pandas as pd

    from .. import _fragments as F

    adata = _atac_of(data)
    features = _features_or_rna(data, features)
    if features.shape[0] > n_tss:
        features = features.sample(n=n_tss, random_state=random_state)
    path = _fragments_path(adata)
    n = adata.n_obs
    width = extend_downstream + extend_upstream + 1
    index_of = _barcode_rows(adata, barcodes)
    device = _device()
    tbi = F.contigs_of(path) if use_index else None
    R = None
    if tbi is not None:
        chromosomes = list(tbi)
    else:
        R = F.read_records(path, index_of, device, chunk_bytes=chunk_bytes or F.CHUNK_BYTES)
        chromosomes = list(R.contigs)
    features = features[features.Chromosome.isin(chromosomes)]
    contig = [str(c) for c in features.Chromosome.values]
    tss_start = np.asarray(features.Start.values, dtype=np.int64)
    lo, hi = tss_start - extend_upstream, tss_start + extend_downstream
    _check_fetch(contig, lo, hi)
    if width < 1001:
        raise ValueError(f"`center_size` (1001) must smaller than the piled up region ({width}).")
    if R is None:
        text = F.indexed_text(path, list(zip(contig, lo.tolist(), hi.tolist())), tbi)
        chunks = F.text_chunks([text] if text else [], chunk_bytes or F.CHUNK_BYTES) if text is not None else None
        if chunks is None:
            R = F.read_records(path, index_of, device, chunk_bytes=chunk_bytes or F.CHUNK_BYTES)
        else:
            R = F.parse_chunks(chunks, F.BarcodeTable(index_of, device), device)
    diff, sums, center_n = F.tss_pileup(R, list(zip(contig, tss_start.tolist())), n, extend_upstream,
                                        extend_downstream, device)
    sums = sums.cpu().numpy()
    flank = sums[:, 0].astype(np.float64) / 200
    flank[flank == 0] = flank.mean()
    with np.errstate(invalid="ignore", divide="ignore"):
        center = sums[:, 1].astype(np.float64) / center_n
        if center_n == 0:
            warnings.warn("Mean of empty slice.", RuntimeWarning, stacklevel=2)
        scores = center / flank
    X = F.tss_scale(diff, n, width, flank, device).cpu().numpy() if return_tss else None
    adata.obs["tss_score"] = scores
    if return_tss:
        anno = pd.DataFrame({"TSS_position": range(-extend_upstream, extend_downstream + 1)})
        anno.index = anno.index.astype(str)
        return _new_anndata(X, adata.obs.copy(), anno)
    return None


def nucleosome_signal(data, n=None, nucleosome_free_upper_bound=147, mononuleosomal_upper_bound=294, barcodes=None,
                      *, chunk_bytes=None):
    """Ratio of mono-nucleosomal to nucleosome-free fragments per cell -- drop-in for ``muon.atac.tl.nucleosome_signal``
    (reference muon/_atac/tools.py:1109-1201).  Writes ``obs["nucleosome_signal"]`` and returns None.

    The first ``n`` records of the file (default ``n_obs * 1e4``) are counted, those of barcodes outside obs
    included; a fragment shorter than ``nucleosome_free_upper_bound`` is nucleosome-free, else one shorter than
    ``mononuleosomal_upper_bound`` is mono-nucleosomal.  Cells with no nucleosome-free fragment get one more of each.
    A file with fewer than ``n`` records raises StopIteration, as the reference's ``next()`` does.  Reading stops as
    soon as ``n`` records are parsed."""
    from .. import _fragments as F

    adata = _atac_of(data)
    path = _fragments_path(adata)
    index_of = _barcode_rows(adata, barcodes)
    n = int(adata.n_obs * 1e4) if n is None else int(n)
    mat = np.zeros((adata.n_obs, 2), dtype=np.int64)
    if n > 0:
        device = _device()
        R = F.read_records(path, index_of, device, max_records=n, chunk_bytes=chunk_bytes or F.CHUNK_BYTES)
        if R.n < n:
            raise StopIteration
        mat += F.nucleosome_counts(R, n, adata.n_obs, nucleosome_free_upper_bound, mononuleosomal_upper_bound,
                                   device).cpu().numpy()
    mat[mat[:, 0] == 0, :] += 1
    adata.obs["nucleosome_signal"] = mat[:, 1] / mat[:, 0]
    return None


# ---- sequences and motifs (muon/_atac/tools.py:381-618) ------------------------------------------------------------------
def _parse_motif_ids(filename=None):
    """The motif_id -> tf_gene_name table (reference muon/_atac/tools.py:381-389), indexed by ``motif_id``.
    ``filename=None`` reads ``motif_to_gene.txt`` of the JASPAR database bundled with an importable ``muon`` package;
    without one it raises FileNotFoundError."""
    from .._motifs import parse_motif_ids
    return parse_motif_ids(filename)


def _parse_motif_matrices(files=None, background=4, pseudocount=0.0001):
    """Log-odds matrices of ``.pfm`` count files (reference muon/_atac/tools.py:392-416): ``{"motifs": ids,
    "matrices": [float64 (4, L) arrays]}``, with ids ``os.path.basename(f).rstrip(".pfm")`` (a character-set strip, as
    in the reference).  ``files=None`` globs the JASPAR database bundled with an importable ``muon`` package; without
    one it raises FileNotFoundError: pass ``files=``.  A file that is not 4 rows (A, C, G, T) of counts raises
    ValueError; so does a background that is not 4 frequencies summing to 1."""
    from .._motifs import parse_motif_matrices
    return parse_motif_matrices(files, background, pseudocount)


def _prepare_motif_scanner(matrices=None, background=4, pvalue=0.0001, max_hits=10):
    """A ``MotifScanner`` (reference muon/_atac/tools.py:419-443): the log-odds tables, per-motif lengths and
    p-value thresholds, uploaded once to the current CUDA device.  ``max_hits`` is MOODS' lookahead window size; it
    does not change results and is ignored.  ``pvalue`` outside (0, 1] raises ValueError; motifs longer than 64
    columns raise NotImplementedError."""
    from .._motifs import prepare_motif_scanner
    return prepare_motif_scanner(matrices, background, pvalue, max_hits)


def scan_sequences(sequences, motif_scanner=None, matrices=None, motifs=None, motif_meta=None, background=4,
                   pvalue=0.0001, max_hits=10):
    """Scan sequences for motif hits on the GPU -- drop-in for ``muon.atac.tl.scan_sequences`` (reference
    muon/_atac/tools.py:446-517).

    Returns a DataFrame with one row per hit, ordered by sequence, then motif (list order), then position:
    ``sequence`` (the caller's own ``str`` objects, not copies), ``motif_id``, ``position`` (0-based window start,
    int64) and ``score`` (float64); with ``motif_meta`` it is left-joined on ``motif_id`` (``motif_id, sequence,
    position, score, tf_gene_name``).  Without a scanner or matrices the JASPAR database bundled with an importable
    ``muon`` package is used, with its motif_to_gene table as ``motif_meta``.  Custom matrices with ``motif_meta=None``
    get that table too when ``muon`` is importable; otherwise the join is skipped with a UserWarning.

    Only the forward strand is scanned, as in the reference.  A window is scored as the float64 sum of its columns in
    order; ``a/c/g/t`` score like ``A/C/G/T`` and a window holding any other character (N, IUPAC codes) is not scored.
    A hit is ``score >= threshold``.  ``motif_scanner`` must be a ``MotifScanner`` from ``_prepare_motif_scanner``
    (anything else, such as a MOODS scanner, raises TypeError: there is no CPU scanner); ``max_hits`` is ignored.
    Zero hits raise ValueError, as the reference does when it names the columns of an empty frame.  Under pandas >= 3
    the reference's frame converts ``sequence`` to the ``str`` dtype, copying every sequence; here it stays an object
    column of the caller's strings."""
    from .._motifs import scan_sequences as scan
    return scan(sequences, motif_scanner, matrices, motifs, motif_meta, background, pvalue, max_hits)


def get_sequences(data, bed, fasta_file, bed_file=None):
    """Sequences of BED intervals from a FASTA file -- drop-in for ``muon.atac.tl.get_sequences`` (reference
    muon/_atac/tools.py:520-566), without pybedtools.

    The genome is ``uns["files"]["genome"]`` when set (``fasta_file`` is then ignored), else ``fasta_file`` is
    recorded there first.  ``bed_file`` is read when given (``bed`` must then be None); ``bed=None`` uses the
    features, named ``chrX:NNN-NNN``.  One sequence per interval (0-based, half-open), case preserved; an interval
    past the end of its contig, or on a contig missing from the FASTA, is skipped with a warning, so the list can be
    shorter than the intervals (as with bedtools).  Start > end raises ValueError.  The FASTA is read through
    ``<fasta>.fai`` when present, else indexed in memory (no ``.fai`` is written); compressed FASTA raises
    NotImplementedError and lines of uneven width inside a record raise ValueError."""
    from .._motifs import get_fasta

    adata = _atac_of(data)
    if "files" not in adata.uns or "genome" not in adata.uns["files"]:
        if fasta_file is not None:
            locate_genome(adata, fasta_file)
        else:
            raise FileNotFoundError("Genome file has to be provided with `fasta_file` or located using "
                                    "`muon.atac.tl.locate_genome`.")
    else:
        fasta_file = adata.uns["files"]["genome"]
    if bed_file is not None:
        assert bed is None
        with open(bed_file) as fh:
            bed = fh.read()
    elif bed is None:
        bed = "\n".join([i.replace(":", "-", 1).replace("-", "\t", 2) for i in adata.var.index.values])
    return get_fasta(bed, fasta_file)


def locate_file(data, key, file):
    """Record ``file`` in ``uns["files"][key]`` -- drop-in for ``muon.atac.tl.locate_file`` (reference
    muon/_atac/tools.py:569-596).  A missing file raises FileNotFoundError."""
    import os
    adata = _atac_of(data)
    if not os.path.exists(file):
        raise FileNotFoundError(f"File {file} does not exist")
    if "files" not in adata.uns:
        adata.uns["files"] = dict()
    adata.uns["files"][key] = file


def locate_genome(data, fasta_file):
    """Record the genome FASTA in ``uns["files"]["genome"]`` -- drop-in for ``muon.atac.tl.locate_genome``
    (reference muon/_atac/tools.py:599-618)."""
    _atac_of(data)
    locate_file(data, "genome", fasta_file)
