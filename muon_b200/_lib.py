"""ctypes binding of ``libmuon_b200.so`` (the C ABI declared in include/muon_b200.h).

The library is built in-tree by ``python __graft_entry__.py build`` (``make -C
muon_b200/csrc``).  There is deliberately NO fallback: if the shared object is missing or a
call fails, the product path raises.  torch is used by callers for device memory and
streams only; pointers cross this boundary as plain integers.
"""
from __future__ import annotations

import ctypes as C
import os
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("MUON_B200_LIB") or os.path.join(_HERE, "csrc", "libmuon_b200.so")   # override: A/B builds

_lock = threading.Lock()
_lib = None

i64, i32, u32, u64, f32, f64, vp = C.c_int64, C.c_int32, C.c_uint32, C.c_uint64, C.c_float, C.c_double, C.c_void_p

# name -> argtypes (restype is int unless noted).  Keep in sync with include/muon_b200.h;
# tests/test_cabi.py parses the header and checks every declared symbol is listed and exported.
SIGNATURES = {
    "mub_version": [],
    "mub_device_info": [C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(i64)],
    "mub_tfidf_reduce_f32": [vp, vp, vp, i64, i32, vp, vp, vp, u32, vp],
    "mub_tfidf_reduce_f64": [vp, vp, vp, i64, i32, vp, vp, vp, u32, vp],
    "mub_tfidf_reduce_tiled_f32": [vp, vp, vp, i64, i32, vp, vp, vp, u32, vp, vp, i32, i64, vp, vp],
    "mub_csr_transpose_fill_tiled": [vp, vp, vp, i64, i32, vp, vp, vp, vp, vp, vp],
    "mub_tfidf_tile_rows": [],
    "mub_tfidf_idf_f32": [vp, i32, f64, u32, vp, vp],
    "mub_tfidf_idf_f64": [vp, i32, f64, u32, vp, vp],
    "mub_tfidf_apply_f32": [vp, vp, vp, vp, i64, i32, vp, vp, f32, u32, vp],
    "mub_tfidf_apply_f64": [vp, vp, vp, vp, i64, i32, vp, vp, f64, u32, vp],
    "mub_spmm_csr_f32": [vp, vp, vp, i64, i64, vp, i32, vp, i32, vp, u32, vp],
    "mub_csr_transpose_count": [vp, i64, i32, vp, vp],
    "mub_csr_transpose_fill": [vp, vp, vp, i64, i32, i64, vp, vp, vp, vp, vp],
    "mub_csr_transpose_fill_f64": [vp, vp, vp, i64, i32, i64, vp, vp, vp, vp, vp],
    "mub_gram_f32": [vp, vp, i64, i32, i32, vp, vp, vp],
    "mub_csr_transpose_fill_pairs": [vp, vp, vp, i64, i32, i64, vp, vp, vp, vp],
    "mub_spmm_csrp_f32": [vp, vp, i64, i64, vp, i32, vp, i32, vp, u32, vp],
    "mub_csrp_row_stats_f32": [vp, vp, i64, vp, vp, vp],
    "mub_csr_select_count": [vp, vp, i64, i32, vp, i64, vp, vp, vp],
    "mub_csr_select_fill_f32": [vp, vp, vp, i32, vp, i64, vp, vp, vp, vp, vp],
    "mub_mofa_update_w_f32": [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, i64, i32, i32, i32, i32, vp],
    "mub_mofa_update_z_f32": [vp, vp, vp, vp, vp, vp, i64, i32, i32, i32, vp],
    "mub_mofa_tau_f32": [vp, vp, vp, f64, vp, vp, vp, vp, f64, vp, i64, i32, i32, vp],
    "mub_mofa_pseudo_f32": [vp, vp, vp, i64, i32, i32, vp],
    "mub_mofa_loglik_f32": [vp, vp, i64, i32, i32, vp, vp],
    "mub_mofa_lowrank_rows_f32": [vp, i64, vp, i64, vp, vp, i32, i32, vp, i32, vp, vp],
    "mub_mofa_lowrank_cols_f32": [vp, i64, vp, i64, vp, vp, i32, i32, vp, vp, vp],
    "mub_mofa_nnz_rows_f32": [vp, vp, vp, i64, vp, vp, vp, vp, i32, i32, vp, vp, vp],
    "mub_mofa_nnz_cols_f32": [vp, vp, i64, vp, vp, vp, vp, i32, i32, vp, vp, vp],
    "mub_knn_l2_f32": [vp, i64, vp, i64, i32, i32, i32, vp, vp, vp],
    "mub_knn_l2_tc_f32": [vp, i64, vp, i64, i32, i32, i32, vp, vp, vp, C.c_size_t, vp, vp],
    "mub_wnn_bandwidth_f32": [vp, vp, vp, vp, vp, i64, i32, i32, i32, f64, vp, vp, vp, i64, vp, i32, i32, vp],
    "mub_wnn_affinity_topk_f32": [i32, vp, vp, vp, vp, vp, vp, i64, i32, i32, vp, vp, vp, vp],
    "mub_f32_to_f16_scaled": [vp, i64, f32, vp, vp],
    "mub_spmm_csr_h16": [vp, vp, vp, i64, i64, vp, i32, vp, i32, f32, vp, u32, vp],
    "mub_spmm_csrp_h16": [vp, vp, i64, i64, vp, i32, vp, i32, f32, vp, u32, vp],
    "mub_stager_create": [C.c_size_t, i32, i32, C.POINTER(vp)],
    "mub_stager_destroy": [vp],
    "mub_stager_h2d": [vp, vp, vp, C.c_size_t, i32, i32, C.POINTER(u64), C.POINTER(i32), vp],
    "mub_stager_d2h": [vp, vp, vp, C.c_size_t, C.POINTER(u64), vp],
    "mub_u8_to_f32": [vp, i64, vp, vp],
    "mub_host_fingerprint": [vp, vp, C.c_size_t, i32, C.POINTER(u64)],
    "mub_device_fingerprint": [vp, i64, vp, vp],
    "mub_synth_count": [i64, i64, i32, vp, vp, vp, vp, u64, vp, vp],
    "mub_synth_fill": [i64, i64, i32, vp, vp, vp, vp, u64, vp, vp, vp, vp],
    "mub_dsb_moments_f32": [vp, vp, vp, i64, i32, f32, vp, vp, vp, vp],
    "mub_dsb_moments_f64": [vp, vp, vp, i64, i32, f64, vp, vp, vp, vp],
    "mub_dsb_fit_f32": [vp, vp, vp, i64, i32, f32, vp, vp, u32, vp, i64, i64, vp, vp, vp, vp, vp, vp, vp],
    "mub_dsb_fit_f64": [vp, vp, vp, i64, i32, f64, vp, vp, u32, vp, i64, i64, vp, vp, vp, vp, vp, vp, vp],
    "mub_dsb_cross_f32": [vp, i64, i32, vp, vp, i32, vp, vp, vp],
    "mub_dsb_cross_f64": [vp, i64, i32, vp, vp, i32, vp, vp, vp],
    "mub_dsb_apply_f32": [vp, i64, i32, vp, vp, i32, vp, f64, vp, f64, f64, u32, vp],
    "mub_dsb_apply_f64": [vp, i64, i32, vp, vp, i32, vp, f64, vp, f64, f64, u32, vp],
    "mub_umap_epoch_f32": [vp, vp, vp, vp, vp, vp, i64, i32, vp, vp, f32, f32, f32, f32, i32, i32, u32, u32, u32, vp],
    "mub_philox4x32_10": [vp, i64, u32, u32, vp, vp],
    "mub_leiden_scan": [i32, vp, vp, vp, vp, i64, i32, f64, vp, vp, vp, vp, vp, u64, vp, vp, vp, vp, i64, vp, vp, vp,
                        vp, vp, vp, vp],
    "mub_leiden_max_shared_degree": [],
    "mub_leiden_apply": [i32, i64, vp, vp, u64, u64, vp, vp, vp],
    "mub_leiden_totals": [i64, i32, vp, vp, i64, vp, vp, vp],
    "mub_leiden_segment_sum": [i64, vp, vp, i64, vp, vp],
    "mub_leiden_internal": [i64, vp, vp, vp, vp, vp, vp],
    "mub_rank_stats_f32": [vp, vp, vp, vp, vp, vp, i32, i32, i32, vp, i64, u32, i32, vp, i64, vp, vp],
    "mub_rank_stats_f64": [vp, vp, vp, vp, vp, vp, i32, i32, i32, vp, i64, u32, i32, vp, i64, vp, vp],
    "mub_rank_score": [vp, i32, i32, vp, i64, u32, f64, vp, vp, vp, vp, vp, vp],
    "mub_frag_newline_count": [vp, i64, vp, vp],
    "mub_frag_newline_fill": [vp, i64, vp, vp, vp],
    "mub_frag_barcode_table": [vp, vp, i32, vp, vp, i64, vp],
    "mub_frag_parse": [vp, vp, i64, i64, vp, vp, vp, vp, vp, i64, vp, vp, vp, vp, vp, vp, vp],
    "mub_frag_overlap": [vp, vp, vp, vp, vp, vp, vp, vp, i32, i64, i32, i32, vp, vp, vp, vp, vp, vp],
    "mub_frag_tss_pileup": [vp, vp, vp, vp, vp, vp, vp, vp, i32, i64, i32, vp, vp],
    "mub_frag_tss_rows": [vp, i64, i32, i32, i32, i32, vp, vp],
    "mub_frag_tss_scale": [vp, i64, i32, vp, vp, vp],
    "mub_frag_nucleosome": [vp, vp, vp, i64, f64, f64, vp, vp],
    "mub_snf_symmetrise_f64": [vp, i64, vp],
    "mub_snf_densify_f64": [vp, vp, vp, i64, vp, vp],
    "mub_snf_select_f64": [vp, vp, i64, i32, i32, vp, vp, vp, vp],
    "mub_snf_affinity_f64": [vp, i64, vp, i32, f64, f64, vp, vp],
    "mub_snf_rowsum_f64": [vp, i64, vp, vp],
    "mub_snf_average_f64": [C.POINTER(vp), C.POINTER(vp), i32, f64, i64, vp, vp],
    "mub_snf_dominate_f64": [vp, vp, vp, i64, vp, vp, vp],
    "mub_snf_diffuse_f64": [vp, vp, vp, i64, vp, vp, vp, i32, vp],
    "mub_motif_encode": [vp, i64, vp],
    "mub_motif_count": [vp, vp, vp, vp, i64, vp, vp, vp, vp, i32, i32, vp, vp],
    "mub_motif_fill": [vp, vp, vp, vp, i64, vp, vp, vp, vp, i32, i32, vp, vp, vp, vp, vp, vp, vp],
}
SPECIAL_RESTYPE = {
    "mub_last_error": ([], C.c_char_p),
    "mub_gram_workspace_bytes": ([i64, i32], C.c_size_t),
    "mub_wnn_bandwidth_workspace_bytes": ([i32, i32], C.c_size_t),
    "mub_knn_l2_tc_workspace_bytes": ([i64, i64, i32], C.c_size_t),
    "mub_dsb_moments_workspace_bytes": ([i64, i32], C.c_size_t),
    "mub_dsb_cross_workspace_bytes": ([i64, i32, i32], C.c_size_t),
    "mub_rank_shared_capacity": ([i32], i32),
    "mub_rank_workspace_slice_bytes": ([i32, i32], i64),
    "mub_frag_tile_bytes": ([], i64),
}

TFIDF_LOG_TF, TFIDF_LOG_IDF, TFIDF_LOG_TFIDF, TFIDF_NO_SCALE, TFIDF_BINARIZE = 1, 2, 4, 8, 16
SPMM_ROWS_SORTED = 1
DSB_STANDARDIZE, DSB_FIT, DSB_CLIP = 1, 2, 1
DSB_MAX_PROTEINS, DSB_MAX_CONTROLS = 1024, 14
UMAP_MAX_COMPONENTS = 16
LEIDEN_MAX_LAYERS = 4
RANK_WILCOXON, RANK_VS_GROUP, RANK_TIE_CORRECT, RANK_OVERESTIM_VAR = 1, 2, 4, 8
RANK_MAX_GROUPS = 1024
SNF_MAX_NEIGHBORS, SNF_MAX_MODALITIES, SNF_MAX_CELLS = 255, 16, 1048576
SNF_SELECT_SMALLEST, SNF_SELECT_LARGEST, SNF_SELECT_DIST, SNF_SELECT_CONN = 0, 1, 2, 3
SNF_DIFFUSE_TRANSPOSED, SNF_DIFFUSE_SYMMETRIC = 0, 1
MOTIF_MAX_LEN, MOTIF_TILE, MOTIF_CODES, MOTIF_GROUP_COLS = 64, 512, 5, 512


class MuonB200Error(RuntimeError):
    pass


def load():
    """Load (once) and return the ctypes library; raise loudly if it is not built."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.isfile(LIB_PATH):
            raise MuonB200Error(
                f"{LIB_PATH} is missing: build the CUDA extension first "
                "(python __graft_entry__.py build, or make -C muon_b200/csrc). "
                "muon_b200 has no CPU fallback.")
        lib = C.CDLL(LIB_PATH)
        for name, argtypes in SIGNATURES.items():
            fn = getattr(lib, name)
            fn.argtypes = argtypes
            fn.restype = C.c_int
        for name, (argtypes, restype) in SPECIAL_RESTYPE.items():
            fn = getattr(lib, name)
            fn.argtypes = argtypes
            fn.restype = restype
        _lib = lib
    return _lib


# kernels launched per successful call (for the benchmark's gpu_launches claim)
KERNELS_PER_CALL = {"mub_csr_transpose_fill_tiled": 2, "mub_csr_transpose_fill": 2, "mub_csr_transpose_fill_f64": 2, "mub_csr_transpose_fill_pairs": 2, "mub_gram_f32": 2, "mub_version": 0, "mub_device_info": 0,
                    "mub_tfidf_tile_rows": 0, "mub_stager_create": 0, "mub_stager_destroy": 0, "mub_stager_h2d": 0, "mub_stager_d2h": 0, "mub_host_fingerprint": 0,
                    "mub_dsb_moments_f32": 4, "mub_dsb_moments_f64": 4, "mub_dsb_cross_f32": 2, "mub_dsb_cross_f64": 2,
                    "mub_leiden_max_shared_degree": 0,
                    "mub_snf_affinity_f64": 2, "mub_snf_dominate_f64": 2}
LAUNCHES = 0          # running count of kernels launched through this binding
PROFILE = None        # None, or dict name -> list[(start_event, end_event)] filled by call()


def call(name: str, *args):
    """Call an int-returning entry point and raise MuonB200Error with mub_last_error() on failure."""
    global LAUNCHES
    lib = load()
    if PROFILE is not None:
        import torch
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        rc = getattr(lib, name)(*args)
        e1.record()
        PROFILE.setdefault(name, []).append((e0, e1))
    else:
        rc = getattr(lib, name)(*args)
    LAUNCHES += KERNELS_PER_CALL.get(name, 1)
    if rc != 0:
        msg = lib.mub_last_error()
        raise MuonB200Error(f"{name} failed (rc={rc}): {msg.decode() if msg else '?'}")


def ptr(t):
    """Device (or host) pointer of a torch tensor / None as an integer for ctypes."""
    return None if t is None else t.data_ptr()


def stream_ptr():
    import torch
    return torch.cuda.current_stream().cuda_stream


# ---- optional coarse phase timing (bench.py --breakdown): synchronising, so never on by default
import contextlib
import time as _time

PHASES = None   # None, or dict name -> seconds
NVTX = os.environ.get("MUON_B200_NVTX", "0") == "1"   # NVTX ranges around the phases (readable nsys timelines)


@contextlib.contextmanager
def phase(name: str):
    if PHASES is None:
        if NVTX:
            import torch
            torch.cuda.nvtx.range_push(name)
            try:
                yield
            finally:
                torch.cuda.nvtx.range_pop()
            return
        yield
        return
    import torch
    torch.cuda.synchronize()
    t0 = _time.perf_counter()
    try:
        yield
    finally:
        torch.cuda.synchronize()
        PHASES[name] = PHASES.get(name, 0.0) + _time.perf_counter() - t0
