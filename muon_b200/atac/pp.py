"""``mu.atac.pp`` -- ATAC preprocessing: ``tfidf``, ``binarize`` and ``scopen``."""
from __future__ import annotations

from typing import Optional, Union
from warnings import warn

import numpy as np

from .._containers import is_anndata, is_mudata, view_to_actual


def _canonical_csr(X):
    """Host-side canonicalisation matching what scipy's matmul does to the reference's output
    pattern (SURVEY App. A.3): duplicates summed, explicit zeros dropped, indices sorted."""
    X = X.copy()
    X.sum_duplicates()
    X.eliminate_zeros()
    X.sort_indices()
    return X


def tfidf(
    data,
    log_tf: bool = True,
    log_idf: bool = True,
    log_tfidf: bool = False,
    scale_factor: Union[int, float] = 1e4,
    inplace: bool = True,
    copy: bool = False,
    from_layer: Optional[str] = None,
    to_layer: Optional[str] = None,
):
    """Transform peak counts with TF-IDF -- drop-in for ``muon.atac.pp.tfidf``
    (reference muon/_atac/preproc.py:16-129; same arguments, errors, and slot rebinding).

    TF: counts normalised by the total per cell; IDF: number of cells over the total per peak;
    by default ``log1p(TF * scale_factor) * log1p(IDF)`` is stored.

    The arithmetic runs on the GPU (fused two-pass CSR kernel, ``csrc/tfidf.cu``) in the
    floating dtype of the counts (float32 stays float32, float64 stays float64, integer counts
    are computed in float64 like the reference).  ``adata.X`` may be a scipy sparse matrix, a
    dense ndarray (result is a ``csr_matrix`` exactly like the reference, preproc.py:113-114)
    or a device-resident :class:`muon_b200.DeviceCSR`, in which case the result stays in HBM.
    """
    from .. import _device

    if is_anndata(data):
        adata = data
    elif is_mudata(data) and "atac" in data.mod:
        adata = data.mod["atac"]
    else:
        raise TypeError("Expected AnnData or MuData object with 'atac' modality")

    if log_tfidf and (log_tf or log_idf):
        raise AttributeError(
            "When returning log(TF*IDF), applying neither log(TF) nor log(IDF) is possible.")
    if copy and not inplace:
        raise ValueError("`copy=True` cannot be used with `inplace=False`.")
    if to_layer is not None and not inplace:
        raise ValueError(f"`to_layer='{str(to_layer)}'` cannot be used with `inplace=False`.")

    if copy:
        adata = adata.copy()
    view_to_actual(adata)

    counts = adata.X if from_layer is None else adata.layers[from_layer]
    if to_layer is not None and to_layer in adata.layers:
        warn(f"Existing layer '{str(to_layer)}' will be overwritten")

    if isinstance(counts, _device.DeviceCSR):
        from .._lib import phase
        with phase("tfidf"):
            res = _device.tfidf_csr(counts, log_tf, log_idf, log_tfidf, scale_factor)
    else:
        import scipy.sparse as sp
        X = counts if sp.isspmatrix_csr(counts) else sp.csr_matrix(counts)
        cdt = X.dtype if X.dtype in (np.float32, np.float64) else np.float64  # ints -> f64, App. A.2
        # The device never touches the sparsity pattern, so the result reuses the host index arrays -- but only
        # when it REPLACES the matrix it was computed from (adata.X = res).  If source and result both stay
        # alive (inplace=False, layers) they get their own arrays, like the reference's np.dot(dia, counts).
        replaces_source = inplace and from_layer is None and to_layer is None and X is counts
        res = None
        for attempt in range(2):
            if cdt == np.float32 and X.indices.dtype in (np.int32, np.int64) and X.nnz > 0:
                got = _device.tfidf_from_host(X, log_tf, log_idf, log_tfidf, scale_factor)   # pipelined with the copies
                if got is not None:
                    out, values, fps = got
                    res = sp.csr_matrix(X.shape, dtype=np.float32)
                    res.data = values
                    res.indices = X.indices if replaces_source else X.indices.copy()
                    res.indptr = X.indptr if replaces_source else X.indptr.copy()
                    res.has_sorted_indices = True
                    _device.remember_resident(res, out, fps)  # lets lsi() skip the re-upload
                    break
            else:
                dev = _device.DeviceCSR.from_scipy(X, dtype=cdt)
                # the kernel itself verifies canonical form while it reduces (no host scan of 6e9 nnz)
                out = _device.tfidf_csr(dev, log_tf, log_idf, log_tfidf, scale_factor, inplace_values=True,
                                        check_canonical=(attempt == 0))
                if out is not None:
                    res = out.get(indptr_host=X.indptr if replaces_source else X.indptr.copy(),
                                  indices_host=X.indices if replaces_source else X.indices.copy())
                    break
            X = _canonical_csr(X)
            replaces_source = False

    if not inplace:
        return res
    if to_layer is not None:
        adata.layers[to_layer] = res
    else:
        adata.X = res
    if copy:
        return adata


def binarize(data):
    """Transform peak counts to the binary matrix (all the non-zero values become 1) -- drop-in for
    ``muon.atac.pp.binarize`` (reference muon/_atac/preproc.py:132-152): a true in-place write of ``X``.

    Host matrices are edited with numpy exactly like the reference; a device-resident
    :class:`muon_b200.DeviceCSR` is edited in HBM.  ``tfidf`` on binarized counts can also be done in one
    fused pass on the device with ``muon_b200._device.tfidf_csr(A, binarize=True)`` (MUB_TFIDF_BINARIZE)."""
    from .. import _device
    if is_anndata(data):
        adata = data
    elif is_mudata(data) and "atac" in data.mod:
        adata = data.mod["atac"]
    else:
        raise TypeError("Expected AnnData or MuData object with 'atac' modality")
    X = adata.X
    if isinstance(X, _device.DeviceCSR):
        X.data.copy_((X.data != 0).to(X.data.dtype))
        X._t = None
        X._tp = None
        return
    import scipy.sparse as sp
    if sp.issparse(X):
        X.data[X.data != 0] = 1
    else:
        X[X != 0] = 1


def scopen(data, n_components: int = 30, max_iter: int = 500, min_rho: float = 0.0, max_rho: float = 0.5,
           alpha: int = 1, verbose: bool = False):
    """Impute peak accessibility with scOpen (Li et al., 2019) -- drop-in for ``muon.atac.pp.scopen`` (reference
    muon/_atac/preproc.py:155-236; same arguments, prints and slots).

    Fills ``obsm["X_scopen"]`` (cells x n_components), ``varm["scopen"]`` (peaks x n_components) and replaces ``X``
    by the imputed accessibility, a dense float64 cells x peaks matrix in [0, 1].  The bounded NMF runs on the GPU
    on the sparse pattern of ``X`` (see ``muon_b200._scopen``); at most 64 components are supported."""
    from .._scopen import scopen as _scopen
    return _scopen(data, n_components=n_components, max_iter=max_iter, min_rho=min_rho, max_rho=max_rho,
                   alpha=alpha, verbose=verbose)
