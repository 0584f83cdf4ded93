"""``mu.tl`` -- multimodal tools.  ``mofa`` (SURVEY section 8, rows a9-a11), ``snf``, ``umap``, ``leiden``, ``louvain``
and ``ica`` run on the GPU."""
from __future__ import annotations


def mofa(data, *args, **kwargs):
    """Multi-Omics Factor Analysis -- drop-in for ``muon.tl.mofa`` (muon/_core/tools.py:290-708)."""
    from ._mofa import mofa as _impl
    return _impl(data, *args, **kwargs)


def umap(mdata, *args, **kwargs):
    """UMAP layout of the neighbour graph on the GPU -- drop-in for ``muon.tl.umap`` (muon/_core/tools.py:1209-1362)."""
    from ._umap import umap as _impl
    return _impl(mdata, *args, **kwargs)


def leiden(data, *args, **kwargs):
    """Multiplex Leiden clustering on the GPU -- drop-in for ``muon.tl.leiden`` (muon/_core/tools.py:1057)."""
    from ._leiden import leiden as _impl
    return _impl(data, *args, **kwargs)


def louvain(data, *args, **kwargs):
    """Multiplex Louvain clustering on the GPU -- drop-in for ``muon.tl.louvain`` (muon/_core/tools.py:1133)."""
    from ._leiden import louvain as _impl
    return _impl(data, *args, **kwargs)


def snf(mdata, *args, **kwargs):
    """Similarity network fusion on the GPU -- drop-in for ``muon.tl.snf`` (muon/_core/tools.py:716-920)."""
    from ._snf import snf as _impl
    return _impl(mdata, *args, **kwargs)


def ica(data, *args, **kwargs):
    """Independent component analysis (FastICA) of an ``obsm`` basis on the GPU -- drop-in for ``muon.tl.ica``
    (muon/_core/tools.py:1365-1386)."""
    from ._ica import ica as _impl
    return _impl(data, *args, **kwargs)
