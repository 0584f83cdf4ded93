"""muon_b200 -- H100-native (sm_90a) drop-in for muon's sparse hot path.

    import muon_b200 as mu
    mu.atac.pp.tfidf(adata)      # muon/_atac/preproc.py:16
    mu.atac.tl.lsi(adata)        # muon/_atac/tools.py:29
    mu.tl.mofa(mdata)            # muon/_core/tools.py:290
    mu.pp.neighbors(mdata)       # muon/_core/preproc.py:264  (WNN; first version, exact search)
    mu.prot.pp.dsb(mdata, raw)   # muon/_prot/preproc.py:17   (DSB; per-cell mixture fits on the GPU)
    mu.tl.snf(mdata)             # muon/_core/tools.py:716   (similarity network fusion; float64 diffusion on the GPU)
    mu.tl.umap(mdata)            # muon/_core/tools.py:1209  (UMAP layout; Jacobi SGD epochs on the GPU)
    mu.atac.tl.rank_peaks_groups(atac, "leiden")   # muon/_atac/tools.py:337  (t-test / Wilcoxon per peak on the GPU)
    mu.atac.tl.scan_sequences(seqs)                # muon/_atac/tools.py:446  (motif hits; every window scored on the GPU)

Same signatures and AnnData/MuData slot semantics as the reference; the arithmetic runs in
hand-written CUDA kernels behind the C ABI in include/muon_b200.h.  There is no CPU fallback.
"""
from . import atac, pp, prot, tl  # noqa: F401
from ._containers import SimpleAnnData, SimpleMuData  # noqa: F401
from ._device import DeviceCSR, release_all_resident, release_resident, trim_host_cache  # noqa: F401

__version__ = "0.1.0"
