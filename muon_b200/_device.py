"""Device-resident CSR container and thin wrappers over the C-ABI kernels.

torch supplies device memory, streams and (in ``_dist``) NCCL; every numerical kernel on
the hot path is a call into ``libmuon_b200.so``.  Nothing here has a CPU fallback.
"""
from __future__ import annotations

import os
from typing import Optional

import numpy as np
import torch

from . import _dist
from ._lib import (TFIDF_BINARIZE, TFIDF_LOG_IDF, TFIDF_LOG_TF, TFIDF_LOG_TFIDF, TFIDF_NO_SCALE, MuonB200Error, call, load, ptr,
                   stream_ptr)

PAD_WIDTHS = (32, 64, 128)


def require_cuda():
    if not torch.cuda.is_available():
        raise MuonB200Error("muon_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
    load()


def pad_width(l: int) -> int:
    for p in PAD_WIDTHS:
        if l <= p:
            return p
    raise NotImplementedError(f"dense block width {l} > 128 is not supported yet")


# ---- host <-> device transfers: native staging engine (csrc/staging.cu) ---------------------------------
_STAGE_BYTES = int(os.environ.get("MUON_B200_STAGE_MB", "64")) << 20
_STAGE_BUFS = int(os.environ.get("MUON_B200_STAGE_BUFS", "4"))
HOST_TIMES = None     # None, or dict name -> seconds of host wall time (bench.py's e2e breakdown)


class _timed:
    def __init__(self, name):
        self.name = name

    def __enter__(self):
        if HOST_TIMES is not None:
            import time
            self.t0 = time.perf_counter()

    def __exit__(self, *exc):
        if HOST_TIMES is not None:
            import time
            HOST_TIMES[self.name] = HOST_TIMES.get(self.name, 0.0) + time.perf_counter() - self.t0


def copy_threads() -> int:
    """Host threads that fill / drain the pinned staging ring: $MUON_B200_COPY_THREADS, else half the cores this
    process may use divided by the ranks sharing the host (torchrun's LOCAL_WORLD_SIZE), clamped to [4, 16]:
    many concurrent copy streams contend for the host's memory system, so more threads can be slower
    (profiles/staging_probe.py measures it)."""
    env = os.environ.get("MUON_B200_COPY_THREADS")
    if env:
        return max(1, int(env))
    try:
        cores = len(os.sched_getaffinity(0))
    except Exception:
        cores = os.cpu_count() or 8
    local = max(1, int(os.environ.get("LOCAL_WORLD_SIZE", "1")))
    return int(min(16, max(4, cores // (2 * local))))


class Stager:
    """ctypes handle on a ``mub_stager`` (ring of pinned buffers + host thread pool).  ``pool_only`` builds the
    thread pool without pinned buffers (host fingerprints only; works without a CUDA device)."""

    def __init__(self, pool_only: bool = False, threads: Optional[int] = None):
        import ctypes as C
        self._C = C
        self.handle = C.c_void_p()
        self.pool_only = pool_only
        call("mub_stager_create", _STAGE_BYTES, 0 if pool_only else _STAGE_BUFS, threads or copy_threads(),
             C.byref(self.handle))

    def __del__(self):
        try:
            if self.handle:
                load().mub_stager_destroy(self.handle)
                self.handle = None
        except Exception:
            pass

    def h2d(self, src: np.ndarray, dst: torch.Tensor, narrow=False, want_hash: bool = False, stream=None):
        """src: contiguous 1-D host array -> dst (device tensor of the same length).  ``narrow``: True / 1 = int64 ->
        int32 (dst int32); 2 = float32 -> uint8 for count data (dst uint8; returns False instead of raising if a
        value is not an integer in [0, 255] -- the caller resends the block as float32)."""
        C = self._C
        h, ov = C.c_uint64(0), C.c_int32(0)
        assert src.flags.c_contiguous and dst.is_contiguous() and src.shape[0] == dst.numel()
        mode = int(narrow)
        eb = src.itemsize if src.itemsize in (4, 8) else 1
        n = src.shape[0] if eb != 1 else src.nbytes
        st = torch.cuda.current_stream().cuda_stream if stream is None else stream.cuda_stream
        with _timed("h2d_s"):
            call("mub_stager_h2d", self.handle, src.ctypes.data, dst.data_ptr(), n, eb, mode,
                 C.byref(h) if want_hash else None, C.byref(ov), st)
        if HOST_TIMES is not None:
            HOST_TIMES["h2d_bytes"] = HOST_TIMES.get("h2d_bytes", 0) + dst.numel() * dst.element_size()
        if mode == 2:
            return not ov.value
        if ov.value:
            raise MuonB200Error("column index does not fit int32 (n_vars >= 2^31 is not supported)")
        return h.value if want_hash else None

    def d2h(self, src: torch.Tensor, dst: np.ndarray, want_hash: bool = False, stream=None):
        C = self._C
        h = C.c_uint64(0)
        nbytes = src.numel() * src.element_size()
        assert dst.flags.c_contiguous and dst.nbytes == nbytes and src.is_contiguous()
        st = torch.cuda.current_stream().cuda_stream if stream is None else stream.cuda_stream
        with _timed("d2h_s"):
            call("mub_stager_d2h", self.handle, src.data_ptr(), dst.ctypes.data, nbytes, C.byref(h) if want_hash else None, st)
        if HOST_TIMES is not None:
            HOST_TIMES["d2h_bytes"] = HOST_TIMES.get("d2h_bytes", 0) + nbytes
        return h.value if want_hash else None

    def fingerprint(self, a: np.ndarray) -> int:
        """Position-dependent 64-bit fingerprint of a host array of 4-byte elements (or int64, read as int32)."""
        C = self._C
        a = np.ascontiguousarray(a).reshape(-1)
        if a.itemsize not in (4, 8):
            raise ValueError("fingerprint: 4-byte elements or int64 only")
        if a.itemsize == 8 and a.dtype != np.int64:
            a = a.view(np.uint32)
        h = C.c_uint64(0)
        with _timed("fingerprint_s"):
            call("mub_host_fingerprint", self.handle, a.ctypes.data, a.shape[0], a.itemsize, C.byref(h))
        return h.value


_STAGER = None
_POOL_ONLY = None


def stager() -> Stager:
    global _STAGER
    if _STAGER is None:
        _STAGER = Stager()
    return _STAGER


def host_pool() -> Stager:
    """Thread pool for host fingerprints (the full stager when one exists)."""
    global _POOL_ONLY
    if _STAGER is not None:
        return _STAGER
    if _POOL_ONLY is None:
        _POOL_ONLY = Stager(pool_only=True)
    return _POOL_ONLY


def device_fingerprint(t: torch.Tensor) -> int:
    """The stager's fingerprint of a contiguous device tensor of 4-byte elements."""
    assert t.is_contiguous() and t.element_size() == 4
    out = torch.zeros(1, dtype=torch.int64, device=t.device)
    call("mub_device_fingerprint", ptr(t), t.numel(), ptr(out), stream_ptr())
    return int(out[0]) & 0xFFFFFFFFFFFFFFFF


def device_fingerprints(t: torch.Tensor, ranges) -> list:
    """Fingerprints of the slices t[k0:k1] (positions counted from each slice's start), one host sync for all."""
    assert t.is_contiguous() and t.element_size() == 4 and t.dim() == 1
    out = torch.zeros(max(len(ranges), 1), dtype=torch.int64, device=t.device)
    for i, (k0, k1) in enumerate(ranges):
        call("mub_device_fingerprint", ptr(t) + 4 * k0, k1 - k0, ptr(out) + 8 * i, stream_ptr())
    return [int(v) & 0xFFFFFFFFFFFFFFFF for v in out.tolist()][:len(ranges)]


class _HostArena:
    """Recycles large host result arrays.  Fresh anonymous memory is expensive here twice over -- the first touch
    of every page while the download is written into it and the unmapping when the array dies -- so blocks are kept and handed out again once NOTHING references them any more (the arrays we
    return are views whose ``base`` is the block, so a live result, or any view of it a caller holds, pins it).
    At most $MUON_B200_HOST_CACHE_GB (default 64) are retained; ``trim()`` returns them to the OS."""

    def __init__(self):
        self.blocks = []
        self.cap = int(float(os.environ.get("MUON_B200_HOST_CACHE_GB", "64")) * 2**30)

    def empty(self, n: int, dtype) -> np.ndarray:
        import sys
        dt = np.dtype(dtype)
        nbytes = int(n) * dt.itemsize
        if nbytes < (64 << 20):
            return np.empty(n, dtype=dt)
        for b in self.blocks:
            if nbytes <= b.nbytes <= 2 * nbytes and sys.getrefcount(b) == 3:      # list + loop variable + argument
                return b[:nbytes].view(dt)
        b = np.empty(nbytes, dtype=np.uint8)
        if sum(x.nbytes for x in self.blocks) + nbytes <= self.cap:
            self.blocks.append(b)
        return b[:nbytes].view(dt)

    def trim(self):
        self.blocks = []


_ARENA = _HostArena()


def trim_host_cache():
    """Give the retained host result buffers back to the OS."""
    _ARENA.trim()


_SMALL = 8 << 20


def to_device(arr, device, dtype=None) -> torch.Tensor:
    """Host array -> device tensor of numpy dtype ``dtype`` (default: unchanged).

    Small arrays go through torch; large pageable arrays through the native stager (pinned ring filled by a
    thread pool while the previous chunk is on the bus; scipy's int64 indices are narrowed to int32 on the host
    inside that copy).  Any other dtype change happens on the device after the upload."""
    if isinstance(arr, torch.Tensor):
        if arr.device.type == "cuda":
            tgt = arr.dtype if dtype is None else getattr(torch, np.dtype(dtype).name)
            return arr if arr.dtype == tgt else arr.to(tgt)
        arr = arr.numpy()
    a = np.ascontiguousarray(arr)
    tgt_np = np.dtype(a.dtype if dtype is None else dtype)
    tgt = getattr(torch, tgt_np.name)
    if a.nbytes <= _SMALL:
        if not a.flags.writeable:
            a = a.copy()
        out = torch.from_numpy(a).to(device, non_blocking=False)
        return out if out.dtype == tgt else out.to(tgt)
    flat = a.reshape(-1)
    if a.dtype == np.int64 and tgt_np == np.int32:
        out = torch.empty(a.shape, dtype=torch.int32, device=device)
        stager().h2d(flat, out.reshape(-1), narrow=True)
        return out
    raw = torch.empty(a.shape, dtype=getattr(torch, a.dtype.name), device=device)
    stager().h2d(flat, raw.reshape(-1))
    if raw.dtype == tgt:
        return raw
    out = raw.to(tgt)
    del raw
    return out


def to_host(t: torch.Tensor, out: Optional[np.ndarray] = None) -> np.ndarray:
    """Device tensor -> numpy array (native stager for large transfers)."""
    np_dt = np.dtype(str(t.dtype).split(".")[1])
    if out is None:
        out = np.empty(tuple(t.shape), dtype=np_dt)
    nbytes = t.numel() * t.element_size()
    if nbytes <= _SMALL:
        torch.from_numpy(out.reshape(-1)).copy_(t.reshape(-1))
        return out
    stager().d2h(t.contiguous().reshape(-1), out.reshape(-1))
    return out


class DeviceCSR:
    """CSR matrix resident in HBM: ``indptr`` int64 [n+1], ``indices`` int32 [nnz], ``data`` [nnz].

    Quacks enough like a scipy matrix (``shape``, ``dtype``, ``nnz``, ``get()``) that it can sit
    in ``adata.X`` between ``tfidf`` and ``lsi`` so that the matrix never leaves the GPU.
    ``row0``/``n_total`` describe a cell shard of a larger matrix (one shard per rank).
    """

    def __init__(self, indptr, indices, data, shape, row0: int = 0, n_total: Optional[int] = None,
                 sorted_indices: bool = True):
        self.indptr, self.indices, self.data = indptr, indices, data
        self.sorted_indices = sorted_indices
        self.shape = (int(shape[0]), int(shape[1]))
        self.row0 = int(row0)
        self._n_total = int(n_total) if n_total is not None else None
        self._t = None  # cached transpose (DeviceCSR of A^T), invalidated when data is rebound
        assert indptr.dtype == torch.int64 and indices.dtype == torch.int32
        assert indptr.numel() == self.shape[0] + 1

    @property
    def n_total(self) -> int:
        """Number of cells of the whole (possibly sharded) matrix: explicit, else the sum of the
        shard heights over the process group, else the local height."""
        if self._n_total is None:
            if _dist.is_distributed():
                t = torch.tensor([self.shape[0]], dtype=torch.int64, device=self.data.device)
                self._n_total = int(_dist.all_reduce_sum_(t)[0])
            else:
                self._n_total = self.shape[0]
        return self._n_total

    # -- scipy-ish surface -------------------------------------------------------------
    @property
    def dtype(self):
        return np.dtype(np.float32 if self.data.dtype == torch.float32 else np.float64)

    @property
    def nnz(self) -> int:
        return int(self.data.numel())

    @property
    def device(self):
        return self.data.device

    def with_data(self, data) -> "DeviceCSR":
        """Same sparsity pattern (shared index tensors), new values."""
        return DeviceCSR(self.indptr, self.indices, data, self.shape, self.row0, self._n_total,
                         self.sorted_indices)

    def copy(self) -> "DeviceCSR":
        return self.with_data(self.data.clone())

    @classmethod
    def from_scipy(cls, X, device=None, dtype=None) -> "DeviceCSR":
        """Upload a canonical scipy CSR (or any object exposing indptr/indices/data/shape)."""
        require_cuda()
        device = torch.device("cuda", torch.cuda.current_device()) if device is None else device
        data = X.data
        if dtype is None:
            dtype = np.float32 if data.dtype == np.float32 else (np.float64 if data.dtype == np.float64 else np.float32)
        return cls(to_device(X.indptr, device, np.int64), to_device(X.indices, device, np.int32),
                   to_device(data, device, dtype), X.shape)

    @classmethod
    def from_scipy_shard(cls, X, world: Optional[int] = None, rank: Optional[int] = None, device=None) -> "DeviceCSR":
        """Upload this rank's row block of a host CSR that every rank can see (e.g. memory-mapped), the blocks cut so
        that all ranks hold about the same number of stored entries (``_dist.balanced_row_range``).  The result
        carries ``row0`` / ``n_total`` like the shards of the synthetic generator."""
        r0, r1 = _dist.balanced_row_range(X.indptr, world, rank)
        sub = X[r0:r1]
        out = cls.from_scipy(sub, device=device)
        out.row0, out._n_total = int(r0), int(X.shape[0])
        return out

    def get(self, indptr_host=None, indices_host=None):
        """Download as scipy.sparse.csr_matrix.  Host index arrays may be passed to be reused
        (the sparsity pattern is never modified on the device)."""
        import scipy.sparse as sp
        data = to_host(self.data)
        indptr = to_host(self.indptr) if indptr_host is None else indptr_host
        indices = to_host(self.indices) if indices_host is None else indices_host
        # scipy's (data, indices, indptr) constructor scans the index arrays (min/max to pick an index
        # dtype): ~30 s for 6e9 int64 indices.  The arrays are known-good, so attach them to an empty matrix.
        if indices.dtype != indptr.dtype:
            if self.nnz < 2**31 - 1 and max(self.shape) < 2**31 - 1:
                indptr = indptr.astype(np.int32) if indptr.dtype != np.int32 else indptr
                indices = indices.astype(np.int32) if indices.dtype != np.int32 else indices
            else:
                indices = indices.astype(np.int64) if indices.dtype != np.int64 else indices
                indptr = indptr.astype(np.int64) if indptr.dtype != np.int64 else indptr
        m = sp.csr_matrix(self.shape, dtype=data.dtype)
        m.data, m.indices, m.indptr = data, indices, indptr
        m.has_sorted_indices = bool(self.sorted_indices)
        return m

    # -- transpose (cached) --------------------------------------------------------------
    def transpose(self) -> "DeviceCSR":
        if self._t is None:
            self._t = csr_transpose(self)
        return self._t

    def transpose_panels(self, pad: int = 64, side_stream: bool = False) -> "TransposedPanels":
        key = ("panels", pad)
        if getattr(self, "_tp", None) is None or self._tp[0] != key:
            self._tp = (key, TransposedPanels(self, pad, side_stream))
        return self._tp[1]


class DevicePairs:
    """CSR whose entries are interleaved 8-byte {int32 index, float32 value} pairs (``pairs``: int32 [nnz, 2]).
    Used for the transposed row panels: one scattered store per non-zero when building, one 8-byte load per
    entry when multiplying."""

    def __init__(self, indptr, pairs, shape):
        self.indptr, self.pairs = indptr, pairs
        self.shape = (int(shape[0]), int(shape[1]))
        self.sorted_indices = False

    @property
    def nnz(self) -> int:
        return int(self.pairs.shape[0])

    @property
    def indices(self):
        return self.pairs[:, 0]

    @property
    def data(self):
        return self.pairs[:, 1].view(torch.float32)


# ------------------------------------------------------------------------------------------
N_CHUNKS = 16          # row chunks of the per-(chunk, column) entry counts; panel sets of 1/2/4/8/16 panels nest in them
_TILE_ROWS = None


def tile_rows() -> int:
    global _TILE_ROWS
    if _TILE_ROWS is None:
        _TILE_ROWS = int(load().mub_tfidf_tile_rows())
    return _TILE_ROWS


def chunk_bounds(n: int, align: Optional[int] = None) -> list:
    """Row boundaries of the N_CHUNKS row chunks of an n-row shard: i*n/16 rounded up to a multiple of the tiled
    reduce kernel's block height (so that no CTA straddles a chunk), last = n.  The transposed row panels
    (TransposedPanels) are unions of consecutive chunks, which lets them reuse the entry counts the TF-IDF
    reduce pass produces."""
    align = tile_rows() if align is None else align
    b = [min(n, -(-round(i * n / N_CHUNKS) // align) * align) for i in range(N_CHUNKS)] + [n]
    for i in range(1, len(b)):
        b[i] = max(b[i], b[i - 1])
    return b


def tiled_reduce_enabled() -> bool:
    return os.environ.get("MUON_B200_TFIDF_TILED", "1") != "0"


def tfidf_csr(A: DeviceCSR, log_tf=True, log_idf=True, log_tfidf=False, scale_factor=1e4,
              inplace_values=False, check_canonical=False, binarize=False) -> Optional[DeviceCSR]:
    """K1: two fused passes (reduce, apply).  Column sums are allreduced across cell shards
    (muon/_atac/preproc.py:92-119; multi-GPU plan SURVEY section 8e)."""
    require_cuda()
    n, d = A.shape
    sfx = "f32" if A.data.dtype == torch.float32 else "f64"
    flags = (TFIDF_LOG_TF if log_tf else 0) | (TFIDF_LOG_IDF if log_idf else 0) | (TFIDF_LOG_TFIDF if log_tfidf else 0)
    if scale_factor is None or scale_factor == 0 or scale_factor == 1:
        flags |= TFIDF_NO_SCALE
        scale_factor = 1.0
    if binarize:
        flags |= TFIDF_BINARIZE
    dev, dt = A.data.device, A.data.dtype
    row_sum = torch.empty(n, dtype=dt, device=dev)
    col_sum = torch.zeros(d, dtype=dt, device=dev)
    st = stream_ptr()
    status = torch.zeros(1, dtype=torch.int32, device=dev) if check_canonical else None
    counts = None
    if sfx == "f32" and A.sorted_indices and tiled_reduce_enabled() and n > 0:
        # shared-memory tiled pass: column sums + the transposition's entry counts, ~30x fewer global atomics
        st_t = torch.zeros(1, dtype=torch.int32, device=dev)
        bounds = chunk_bounds(n)
        counts = torch.zeros((N_CHUNKS, d), dtype=torch.int32, device=dev)
        cb = torch.tensor(bounds, dtype=torch.int64, device=dev)
        rb_counts = torch.empty((-(-n // tile_rows()), d), dtype=torch.int16, device=dev)      # uint16 entries per (512-row block, column)
        call("mub_tfidf_reduce_tiled_f32", ptr(A.indptr), ptr(A.indices), ptr(A.data), n, d, ptr(row_sum), ptr(col_sum),
             ptr(st_t), flags, ptr(counts), ptr(cb), N_CHUNKS, 0, ptr(rb_counts), st)
        bad = int(st_t[0])
        if check_canonical and bad != 0:
            return None  # caller canonicalises (duplicates / explicit zeros / unsorted rows) and retries
        if bad & 1:      # a row is not sorted after all: the tiled sums are invalid, take the order-agnostic kernel
            A.sorted_indices = False
            counts = None
            col_sum.zero_()
    if counts is None:
        call(f"mub_tfidf_reduce_{sfx}", ptr(A.indptr), ptr(A.indices), ptr(A.data), n, d, ptr(row_sum), ptr(col_sum),
             ptr(status), flags, st)
        if check_canonical and int(status[0]) != 0:
            return None  # caller canonicalises (duplicates / explicit zeros / unsorted rows) and retries
    _dist.all_reduce_sum_(col_sum)
    idf = torch.empty(d, dtype=dt, device=dev)
    call(f"mub_tfidf_idf_{sfx}", ptr(col_sum), d, float(A.n_total), flags, ptr(idf), st)
    out = A.data if inplace_values else torch.empty_like(A.data)
    call(f"mub_tfidf_apply_{sfx}", ptr(A.indptr), ptr(A.indices), ptr(A.data), ptr(out), n, d, ptr(row_sum),
         ptr(idf), float(scale_factor), flags, st)
    res = A.with_data(out)
    res._aux = {"row_sum": row_sum, "col_sum": col_sum, "idf": idf}
    if counts is not None:
        res._aux["col_counts"] = (bounds, counts)
        res._aux["rb_counts"] = rb_counts
    return res


def csr_transpose(A: DeviceCSR, row0: int = 0, row1: Optional[int] = None, k0: Optional[int] = None,
                  k1: Optional[int] = None, pairs: bool = False, col_count: Optional[torch.Tensor] = None,
                  rb_counts: Optional[torch.Tensor] = None, scratch: Optional[dict] = None):
    """Build the CSR of (A[row0:row1])^T on the device (count -> scan -> atomic-cursor fill).
    Row indices stored in the result are local to the panel (0 .. row1-row0).  ``k0``/``k1`` are the
    non-zero offsets of the row range if the caller already knows them (avoids a host sync)."""
    require_cuda()
    assert A.data.dtype == torch.float32, "transpose: float32 values only"
    n, d = A.shape
    row1 = n if row1 is None else row1
    dev = A.data.device
    st = stream_ptr()
    if k0 is None or k1 is None:
        if row0 == 0 and row1 == n:
            k0, k1 = 0, A.nnz
        else:
            k0, k1 = int(A.indptr[row0]), int(A.indptr[row1])
    nnz = k1 - k0
    t_count = torch.zeros(d + 1, dtype=torch.int64, device=dev)
    if col_count is not None:      # entries per column of this row range, known from the TF-IDF reduce pass
        t_count[1:] = col_count
    else:
        call("mub_csr_transpose_count", ptr(A.indices) + 4 * k0, nnz, d, ptr(t_count), st)
    t_indptr = torch.cumsum(t_count, 0)
    cursor = torch.empty(max(d, 1), dtype=torch.int64, device=dev)
    if pairs and rb_counts is not None and col_count is not None and row0 % tile_rows() == 0:
        # atomic-free fill: write offsets of every 512-row block from the scanned per-block counts (transpose.cu)
        t_pairs = torch.empty((nnz, 2), dtype=torch.int32, device=dev)
        nb = -(-(row1 - row0) // tile_rows())
        if scratch.get("base") is None or scratch["base"].numel() < nb * d:
            scratch["base"] = torch.empty(nb * d, dtype=torch.int32, device=dev)
        if scratch.get("status") is None:
            scratch["status"] = torch.zeros(1, dtype=torch.int32, device=dev)
        call("mub_csr_transpose_fill_tiled", ptr(A.indptr) + 8 * row0, ptr(A.indices), ptr(A.data), row1 - row0, d,
             ptr(rb_counts) + 2 * (row0 // tile_rows()) * d, ptr(t_indptr), ptr(scratch["base"]), ptr(t_pairs),
             ptr(scratch["status"]), st)
        return DevicePairs(t_indptr, t_pairs, (d, row1 - row0))
    if pairs:
        t_pairs = torch.empty((nnz, 2), dtype=torch.int32, device=dev)
        call("mub_csr_transpose_fill_pairs", ptr(A.indptr) + 8 * row0, ptr(A.indices), ptr(A.data), row1 - row0, d, 0,
             ptr(t_indptr), ptr(cursor), ptr(t_pairs), st)
        return DevicePairs(t_indptr, t_pairs, (d, row1 - row0))
    t_indices = torch.empty(nnz, dtype=torch.int32, device=dev)
    t_data = torch.empty(nnz, dtype=torch.float32, device=dev)
    # indptr values are absolute offsets into indices/data, so only the indptr pointer is shifted;
    # slots claimed from `cursor` are panel-local, so the outputs are not
    call("mub_csr_transpose_fill", ptr(A.indptr) + 8 * row0, ptr(A.indices), ptr(A.data), row1 - row0, d, 0,
         ptr(t_indptr), ptr(cursor), ptr(t_indices), ptr(t_data), st)
    return DeviceCSR(t_indptr, t_indices, t_data, (d, row1 - row0), n_total=d, sorted_indices=False)


class TransposedPanels:
    """A^T as a list of row-panel transposes.  A^T Y gathers rows of Y (n x P); when n*P*4 bytes
    exceed what stays resident in L2 the gathers fall through to HBM, so the cells are cut into
    panels whose slice of Y fits in L2 and the products are accumulated panel by panel."""

    # bytes of the gathered operand per panel (H100 L2: 50 MB, shared with the CSR stream)
    L2_BUDGET = int(os.environ.get("MUON_B200_L2_BUDGET_MB", "16")) << 20

    def __init__(self, A: DeviceCSR, pad: int = 64, side_stream: bool = False):
        n = A.shape[0]
        rows = max(1, self.L2_BUDGET // (4 * pad))
        n_panels = max(1, -(-n // rows))
        counts, rb = None, None
        if n_panels <= N_CHUNKS:
            # 1, 2, 4, 8 or 16 panels, each a union of consecutive row chunks (see chunk_bounds): the entry counts
            # per (chunk, column) left behind by the TF-IDF reduce pass then replace the counting pass
            n_panels = 1 << (n_panels - 1).bit_length()
            cb = chunk_bounds(n)
            per = N_CHUNKS // n_panels
            bounds = [cb[i * per] for i in range(n_panels)] + [n]
            aux = getattr(A, "_aux", None) or {}
            if "col_counts" in aux and list(aux["col_counts"][0]) == cb:
                cc = aux["col_counts"][1]
                counts = [cc[i * per:(i + 1) * per].sum(0, dtype=torch.int64) for i in range(n_panels)]
                # the tiled fill lists every transposed row in ascending cell order, so A^T Y sums in the same
                # order on every run (the atomic-cursor fill's order follows slot claims); MUON_B200_FILL_TILED=0
                # selects the atomic-cursor fill
                if os.environ.get("MUON_B200_FILL_TILED", "1") == "1" and not side_stream:
                    rb = aux.get("rb_counts")
        else:
            bounds = [round(i * n / n_panels) for i in range(n_panels + 1)]
        self.counts_reused = counts is not None
        self.tiled_fill = False
        self.shape = (A.shape[1], n)
        # non-zero offsets of the panel boundaries: one small D2H up front, no host syncs afterwards
        ks = A.indptr[torch.tensor(bounds, device=A.indptr.device)].tolist()
        self.ready = None
        if side_stream:
            # build on a second stream so that the first A*V product (main stream) overlaps it;
            # consumers call wait() before touching the panels
            main = torch.cuda.current_stream()
            side = torch.cuda.Stream()
            side.wait_stream(main)
            with torch.cuda.stream(side):
                self.panels = [(bounds[i], bounds[i + 1], csr_transpose(A, bounds[i], bounds[i + 1], ks[i], ks[i + 1], pairs=True,
                                                                        col_count=counts[i] if counts else None))
                               for i in range(n_panels)]
                self.ready = side.record_event()
            for _, _, T in self.panels:           # memory is consumed on the main stream later on
                for t in (T.indptr, T.pairs):
                    t.record_stream(main)
        else:
            scratch = {}
            build = lambda rbc: [(bounds[i], bounds[i + 1], csr_transpose(A, bounds[i], bounds[i + 1], ks[i], ks[i + 1], pairs=True,  # noqa: E731
                                                                          col_count=counts[i] if counts else None, rb_counts=rbc,
                                                                          scratch=scratch))
                                 for i in range(n_panels) if bounds[i + 1] > bounds[i]]
            self.panels = build(rb)
            if rb is not None:
                if int(scratch["status"][0]) == 0:
                    self.tiled_fill = True
                else:          # counts and pattern disagree (the matrix was modified after tfidf): atomic-cursor fill
                    self.panels = build(None)

    def wait(self):
        if self.ready is not None:
            torch.cuda.current_stream().wait_event(self.ready)
            self.ready = None

    def spmm(self, Y: torch.Tensor, dynamic=True, half: bool = False, row_chunks: int = 1, on_chunk=None) -> torch.Tensor:
        """A^T Y accumulated panel by panel.  ``half``: round Y to IEEE half first (see ``spmm_h16``).
        ``row_chunks`` > 1 computes the result in that many blocks of output rows (peaks), each finished over all
        panels before the next starts, and hands every finished block to ``on_chunk`` (the multi-GPU driver starts
        its allreduce there, under the next block's product)."""
        self.wait()
        d, P = self.shape[0], Y.shape[1]
        Yh = to_half_scaled(Y) if half else None
        out = torch.empty((d, P), dtype=torch.float32, device=Y.device)
        row_chunks = max(1, min(int(row_chunks), d))
        cuts = [round(i * d / row_chunks) for i in range(row_chunks + 1)]
        for j0, j1 in zip(cuts[:-1], cuts[1:]):
            first = True
            for r0, r1, T in self.panels:
                if half:
                    spmm_h16(T, Yh[r0:r1], out=out, accumulate=not first, dynamic=dynamic, rows=(j0, j1))
                else:
                    spmm(T, Y[r0:r1], out=out, accumulate=not first, dynamic=dynamic, rows=(j0, j1))
                first = False
            if on_chunk is not None:
                on_chunk(out[j0:j1])
        return out

    def spmm_rowblocks(self, Y: torch.Tensor, blocks) -> torch.Tensor:
        """Rows ``blocks`` = [(j0, j1), ...] of A^T Y only, stacked into a compact (sum of block heights) x P buffer
        (fp32 operand).  Used for the sampled residual check of the LSI driver: 1/16 of the rows costs 1/16 of a pass."""
        self.wait()
        P = Y.shape[1]
        total = sum(j1 - j0 for j0, j1 in blocks)
        out = torch.empty((total, P), dtype=torch.float32, device=Y.device)
        o0 = 0
        for j0, j1 in blocks:
            first = True
            for r0, r1, T in self.panels:
                spmm(T, Y[r0:r1], out=out, accumulate=not first, dynamic=False, rows=(j0, j1, o0))
                first = False
            o0 += j1 - j0
        return out


def _row_range(rows, n):
    """``rows`` of spmm / spmm_h16: None = all rows; (j0, j1) = that row range written to the same rows of ``out``;
    (j0, j1, o0) = written to out rows starting at o0 (a compact buffer of sampled rows)."""
    if rows is None:
        return 0, n, 0
    if len(rows) == 2:
        return rows[0], rows[1], rows[0]
    return rows


def sample_row_blocks(d: int, fraction: int = 16, n_blocks: int = 4):
    """``n_blocks`` evenly spaced contiguous row blocks covering 1/``fraction`` of d rows -> list of (j0, j1)."""
    bs = max(1, d // (fraction * n_blocks))
    out, last = [], 0
    for i in range(n_blocks):
        j0 = max(last, (i * d) // n_blocks)
        j1 = min(d, j0 + bs)
        if j1 > j0:
            out.append((j0, j1))
            last = j1
    return out


HALF_SCALE = 32768.0     # 2^15: orthonormal columns (|x| <= 1) stay finite and leave the subnormal range of IEEE half


def to_half_scaled(B: torch.Tensor, scale: float = HALF_SCALE) -> torch.Tensor:
    """fp32 dense operand -> IEEE half of (B * scale), same shape (one fused kernel, 6 B per element)."""
    assert B.dtype == torch.float32 and B.is_contiguous() and B.numel() % 4 == 0
    out = torch.empty(B.shape, dtype=torch.float16, device=B.device)
    call("mub_f32_to_f16_scaled", ptr(B), B.numel(), float(scale), ptr(out), stream_ptr())
    return out


def spmm_h16(A, Bh: torch.Tensor, out: Optional[torch.Tensor] = None, accumulate=False, dynamic=True,
             scale: float = HALF_SCALE, rows=None) -> torch.Tensor:
    """C[n x P] (+)= A @ (Bh / scale) with the dense operand stored as IEEE half (``to_half_scaled``): half the
    bytes per non-zero through the L2 -> L1 gather path that bounds the fp32 kernel; fp32 products and sums."""
    n, d = A.shape
    P = Bh.shape[1]
    assert Bh.shape[0] == d and Bh.dtype == torch.float16 and Bh.is_contiguous(), (Bh.shape, d, Bh.dtype)
    if out is None:
        assert not accumulate
        out = torch.empty((n, P), dtype=torch.float32, device=Bh.device)
    counter = torch.zeros(1, dtype=torch.int64, device=Bh.device) if dynamic else None
    j0, j1, o0 = _row_range(rows, n)                    # matrix rows [j0, j1) -> out rows [o0, o0 + j1 - j0)
    if isinstance(A, DevicePairs):
        call("mub_spmm_csrp_h16", ptr(A.indptr) + 8 * j0, ptr(A.pairs), j1 - j0, d, ptr(Bh), P, ptr(out) + 4 * P * o0,
             1 if accumulate else 0, 1.0 / scale, ptr(counter), stream_ptr())
    else:
        call("mub_spmm_csr_h16", ptr(A.indptr) + 8 * j0, ptr(A.indices), ptr(A.data), j1 - j0, d, ptr(Bh), P,
             ptr(out) + 4 * P * o0, 1 if accumulate else 0, 1.0 / scale, ptr(counter), stream_ptr())
    return out


def spmm(A: DeviceCSR, B: torch.Tensor, out: Optional[torch.Tensor] = None, accumulate=False,
         dynamic=True, algo: Optional[str] = None, rows=None) -> torch.Tensor:
    """K2/K3: C[n x P] (+)= A @ B[d x P];  P = B.shape[1] must be 32, 64 or 128.

    algo: "rowwarp" (v1: warp per row, B gathered from L2), "panel" (v2: B column panels staged in
    shared memory by TMA; needs sorted column indices) or None = $MUON_B200_SPMM or auto."""
    n, d = A.shape
    P = B.shape[1]
    assert B.shape[0] == d and B.dtype == torch.float32 and B.is_contiguous(), (B.shape, d, B.dtype)
    if out is None:
        assert not accumulate
        out = torch.empty((n, P), dtype=torch.float32, device=B.device)
    j0, j1, o0 = _row_range(rows, n)                    # matrix rows [j0, j1) -> out rows [o0, o0 + j1 - j0)
    if isinstance(A, DevicePairs):
        counter = torch.zeros(1, dtype=torch.int64, device=B.device) if dynamic else None
        call("mub_spmm_csrp_f32", ptr(A.indptr) + 8 * j0, ptr(A.pairs), j1 - j0, d, ptr(B), P, ptr(out) + 4 * P * o0,
             1 if accumulate else 0, ptr(counter), stream_ptr())
        return out
    if algo is None:
        algo = os.environ.get("MUON_B200_SPMM", "auto")
    if algo == "auto":
        algo = "rowwarp"   # the panel kernel is correct but not yet faster (DESIGN.md section 4)
    if algo == "panel":
        if not A.sorted_indices:
            raise MuonB200Error("spmm(algo='panel') needs sorted column indices")
        call("mub_spmm_csr_panel_f32", ptr(A.indptr), ptr(A.indices), ptr(A.data), n, d, ptr(B), P, ptr(out),
             1 if accumulate else 0, stream_ptr())
        return out
    counter = torch.zeros(1, dtype=torch.int64, device=B.device) if dynamic else None
    call("mub_spmm_csr_f32", ptr(A.indptr) + 8 * j0, ptr(A.indices), ptr(A.data), j1 - j0, d, ptr(B), P,
         ptr(out) + 4 * P * o0, 1 if accumulate else 0, ptr(counter), stream_ptr())
    return out


def gram(Y: torch.Tensor, l: Optional[int] = None, weights: Optional[torch.Tensor] = None,
         reduce=True) -> torch.Tensor:
    """K4: G[l x l] = Y^T diag(w) Y in float64 (allreduced over cell shards if ``reduce``)."""
    lib = load()
    n, P = Y.shape
    l = P if l is None else l
    assert Y.dtype == torch.float32 and Y.is_contiguous()
    ws = torch.empty(max(int(lib.mub_gram_workspace_bytes(n, P)), 4), dtype=torch.uint8, device=Y.device)
    G = torch.empty((l, l), dtype=torch.float64, device=Y.device)
    call("mub_gram_f32", ptr(Y), ptr(weights), n, P, l, ptr(G), ptr(ws), stream_ptr())
    if reduce:
        _dist.all_reduce_sum_(G)
    return G


# ------------------------------------------------------------------------------------------
# Host path of tfidf(): pageable scipy CSR in, pageable scipy CSR out (the reference's contract,
# muon/_atac/preproc.py:86-129), with the device work hidden under the transfers:
#   upload    row block b+1 is staged/uploaded on a copy stream while the reduce kernel runs on block b
#             (int64 indices -> int32 and float32 counts -> uint8 inside the staging copy)
#   download  one apply launch over all rows, then one staged download into a recycled host buffer
# Fingerprints of what crossed the bus are taken on the device copies afterwards (csrc/staging.cu).
_BLOCK_NNZ = int(os.environ.get("MUON_B200_BLOCK_NNZ", str(192 << 20)))


def _row_blocks(indptr_host: np.ndarray, block_nnz: int, align: int = 1):
    """Cut rows into consecutive blocks of about ``block_nnz`` stored entries -> list of (r0, r1, k0, k1); cuts are
    multiples of ``align`` rows."""
    n = indptr_host.shape[0] - 1
    nnz = int(indptr_host[-1])
    if n == 0:
        return []
    nb = max(1, -(-nnz // max(block_nnz, 1)))
    targets = (np.arange(1, nb, dtype=np.float64) * (nnz / nb)).astype(np.int64)
    inner = np.searchsorted(indptr_host, targets, side="left")
    inner = np.minimum(n, -(-inner // align) * align)
    cuts = np.unique(np.concatenate([[0], inner, [n]]))
    return [(int(a), int(b), int(indptr_host[a]), int(indptr_host[b])) for a, b in zip(cuts[:-1], cuts[1:]) if b > a]


def tfidf_from_host(X, log_tf=True, log_idf=True, log_tfidf=False, scale_factor=1e4):
    """float32 scipy CSR on the host -> (DeviceCSR holding the TF-IDF values, host value array, fingerprints),
    or None if the input is not canonical (the caller canonicalises and retries).

    Same kernels as ``tfidf_csr``; the host<->device copies are pipelined with them as described above."""
    require_cuda()
    assert X.data.dtype == np.float32
    n, d = X.shape
    dev = torch.device("cuda", torch.cuda.current_device())
    flags = (TFIDF_LOG_TF if log_tf else 0) | (TFIDF_LOG_IDF if log_idf else 0) | (TFIDF_LOG_TFIDF if log_tfidf else 0)
    if scale_factor is None or scale_factor == 0 or scale_factor == 1:
        flags |= TFIDF_NO_SCALE
        scale_factor = 1.0
    indptr_h = np.ascontiguousarray(X.indptr)
    indices_h = np.ascontiguousarray(X.indices)
    data_h = np.ascontiguousarray(X.data)
    nnz = int(indptr_h[-1]) if indptr_h.shape[0] else 0
    tiled = tiled_reduce_enabled()
    blocks = _row_blocks(indptr_h, _BLOCK_NNZ, tile_rows() if tiled else 1)
    st = stager()
    main = torch.cuda.current_stream()
    side = torch.cuda.Stream()
    indptr = to_device(indptr_h, dev, np.int64)
    indices = torch.empty(nnz, dtype=torch.int32, device=dev)
    data = torch.empty(nnz, dtype=torch.float32, device=dev)
    row_sum = torch.empty(n, dtype=torch.float32, device=dev)
    col_sum = torch.zeros(d, dtype=torch.float32, device=dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    bounds = chunk_bounds(n) if tiled else None
    counts = torch.zeros((N_CHUNKS, d), dtype=torch.int32, device=dev) if tiled else None
    cb = torch.tensor(bounds, dtype=torch.int64, device=dev) if tiled else None
    rb_counts = torch.empty((-(-n // tile_rows()), d), dtype=torch.int16, device=dev) if tiled else None
    side.wait_stream(main)                      # allocations above are ordered on the main stream
    narrow = indices_h.dtype == np.int64
    assert narrow or indices_h.dtype == np.int32, indices_h.dtype
    # peak counts are small integers stored as float32: they cross the bus as uint8 (a quarter of the bytes) and are
    # widened on the device; the first block that holds anything else switches this off for the rest of the matrix
    as_u8 = os.environ.get("MUON_B200_COUNTS_U8", "1") != "0"
    tmp8 = torch.empty(max(k1 - k0 for (_, _, k0, k1) in blocks), dtype=torch.uint8, device=dev) if (as_u8 and blocks) else None
    if tmp8 is not None:
        tmp8.record_stream(side)
    for (r0, r1, k0, k1) in blocks:
        st.h2d(indices_h[k0:k1], indices[k0:k1], narrow=narrow, stream=side)
        if as_u8 and st.h2d(data_h[k0:k1], tmp8[:k1 - k0], narrow=2, stream=side):
            call("mub_u8_to_f32", ptr(tmp8), k1 - k0, ptr(data) + 4 * k0, side.cuda_stream)
        else:
            as_u8 = False
            st.h2d(data_h[k0:k1], data[k0:k1], stream=side)
        main.wait_event(side.record_event())
        if tiled:      # host matrices must be canonical anyway (checked here): sorted rows, so the tiled pass applies
            call("mub_tfidf_reduce_tiled_f32", ptr(indptr) + 8 * r0, ptr(indices), ptr(data), r1 - r0, d, ptr(row_sum) + 4 * r0,
                 ptr(col_sum), ptr(status), flags, ptr(counts), ptr(cb), N_CHUNKS, r0, ptr(rb_counts), main.cuda_stream)
        else:
            call("mub_tfidf_reduce_f32", ptr(indptr) + 8 * r0, ptr(indices), ptr(data), r1 - r0, d, ptr(row_sum) + 4 * r0,
                 ptr(col_sum), ptr(status), flags, main.cuda_stream)
    for t in (indices, data):
        t.record_stream(side)
    if int(status[0]) != 0:                     # duplicates / explicit zeros / unsorted rows (also syncs the upload)
        return None
    _dist.all_reduce_sum_(col_sum)
    idf = torch.empty(d, dtype=torch.float32, device=dev)
    n_total = n
    if _dist.is_distributed():
        t = torch.tensor([n], dtype=torch.int64, device=dev)
        n_total = int(_dist.all_reduce_sum_(t)[0])
    call("mub_tfidf_idf_f32", ptr(col_sum), d, float(n_total), flags, ptr(idf), main.cuda_stream)
    with _timed("alloc_out_s"):
        out_h = _ARENA.empty(nnz, np.float32)

    # apply over all rows, then ONE download call: every d2h call drains its pipeline before it
    # returns, so downloading block by block (to overlap the apply kernels) cost more in bubbles than it hid
    if blocks:
        call("mub_tfidf_apply_f32", ptr(indptr), ptr(indices), ptr(data), ptr(data), n, d, ptr(row_sum), ptr(idf),
             float(scale_factor), flags, main.cuda_stream)
        side.wait_event(main.record_event())
        st.d2h(data, out_h, stream=side)
    main.wait_stream(side)
    # fingerprints of what crossed the bus, taken on the device copies (HBM-bound) instead of
    # inside the host-side staging loops
    ranges = [(k0, k1) for (_, _, k0, k1) in blocks]
    fp_idx = device_fingerprints(indices, ranges)
    fp_out = device_fingerprints(data, ranges)
    res = DeviceCSR(indptr, indices, data, (n, d), n_total=n_total)
    res._aux = {"row_sum": row_sum, "col_sum": col_sum, "idf": idf}
    if tiled:
        res._aux["col_counts"] = (bounds, counts)
        res._aux["rb_counts"] = rb_counts
    fps = {"blocks": [(k0, k1) for (_, _, k0, k1) in blocks], "indices": fp_idx, "data": fp_out,
           "indptr": host_pool().fingerprint(indptr_h.astype(np.int64, copy=False).view(np.uint32)) if n else 0}
    return res, out_h, fps


# ------------------------------------------------------------------------------------------
# Device twins.  A host matrix produced by tfidf() keeps a handle on the DeviceCSR it was downloaded from so
# that a following lsi()/mofa() on the same AnnData skips the 48 GB re-upload.  The twin is used only after
# EVERY element of the host matrix's data, indices and indptr has been re-fingerprinted (position-dependent,
# csrc/staging.cu) and found equal to what crossed the bus -- one threaded read pass over the host arrays, no
# device work -- so any host-side edit between the two calls (values, order, a single index) falls back to a
# fresh upload.  $MUON_B200_RESIDENT=0 disables twins; release_resident() / release_all_resident() free the HBM
# explicitly (a twin otherwise lives as long as the host matrix it is attached to).
_RESIDENT_ATTR = "_mub_resident"
_RESIDENT_REGISTRY = None


def resident_enabled() -> bool:
    return os.environ.get("MUON_B200_RESIDENT", "1") != "0"


def remember_resident(host_matrix, dev: "DeviceCSR", fingerprints: dict):
    global _RESIDENT_REGISTRY
    if not resident_enabled():
        return
    try:
        setattr(host_matrix, _RESIDENT_ATTR, (dev, fingerprints))
    except Exception:
        return
    import weakref
    if _RESIDENT_REGISTRY is None:
        _RESIDENT_REGISTRY = {}
    key = id(host_matrix)                 # scipy matrices are not hashable: registry keyed by id, entries die with the matrix
    _RESIDENT_REGISTRY[key] = weakref.ref(host_matrix, lambda _r, k=key: _RESIDENT_REGISTRY.pop(k, None))


def release_resident(obj) -> bool:
    """Drop the device twin attached to a host matrix (or to ``adata.X`` / every layer of an AnnData-like
    object).  Returns True if something was released."""
    done = False
    for m in [obj, getattr(obj, "X", None)] + list(getattr(obj, "layers", {}).values() if hasattr(obj, "layers") else []):
        if m is not None and getattr(m, _RESIDENT_ATTR, None) is not None:
            try:
                delattr(m, _RESIDENT_ATTR)
                done = True
            except Exception:
                pass
    return done


def release_all_resident() -> int:
    """Drop every live device twin (e.g. before a memory-hungry mofa()/neighbors() call)."""
    n = 0
    if _RESIDENT_REGISTRY is not None:
        for ref in list(_RESIDENT_REGISTRY.values()):
            m = ref()
            if m is not None:
                n += bool(release_resident(m))
    return n


def resident_candidate(host_matrix):
    """The device twin attached to a host matrix and its fingerprints, after the cheap checks (shape, nnz, dtypes);
    None if there is none.  The twin may only be USED once ``resident_valid`` has confirmed it."""
    rec = getattr(host_matrix, _RESIDENT_ATTR, None)
    if rec is None or not resident_enabled():
        return None
    try:
        dev, fps = rec
        if not isinstance(dev, DeviceCSR) or tuple(dev.shape) != tuple(host_matrix.shape) or dev.nnz != host_matrix.nnz:
            return None
        if host_matrix.data.dtype != np.float32 or dev.data.dtype != torch.float32:
            return None
        if host_matrix.indices.dtype not in (np.int32, np.int64) or host_matrix.indptr.shape[0] != dev.shape[0] + 1:
            return None
        return dev, fps
    except Exception:
        return None


def resident_valid(host_matrix, fps) -> bool:
    """Re-fingerprint every element of the host matrix (threaded read pass, no device work; the GIL is released, so
    this can run on a helper thread under device work) and compare with what crossed the bus."""
    try:
        pool = host_pool()
        indptr = np.ascontiguousarray(host_matrix.indptr).astype(np.int64, copy=False)
        if pool.fingerprint(indptr.view(np.uint32)) != fps["indptr"]:
            return False
        idx, dat = np.ascontiguousarray(host_matrix.indices), np.ascontiguousarray(host_matrix.data)
        for (k0, k1), hi, hd in zip(fps["blocks"], fps["indices"], fps["data"]):
            if pool.fingerprint(dat[k0:k1]) != hd or pool.fingerprint(idx[k0:k1]) != hi:
                return False
        return True
    except Exception:
        return False


def recall_resident(host_matrix) -> Optional["DeviceCSR"]:
    cand = resident_candidate(host_matrix)
    if cand is None:
        return None
    return cand[0] if resident_valid(host_matrix, cand[1]) else None


def knn_l2(X: torch.Tensor, k: int, Y: Optional[torch.Tensor] = None, algo: Optional[str] = None,
           query_chunk: Optional[int] = None):
    """Exact k nearest neighbours in Euclidean distance (rows of Y closest to each row of X; Y defaults to X).
    Returns (indices int32 [n x k], distances float32 [n x k]), ascending, ties by lower index.  Groundwork for
    the WNN row (reference muon/_core/preproc.py:520-528).

    algo: "simt" (fp32 CUDA-core kernel), "tc" (wgmma TF32 candidate pass + fp32 re-rank, same result; falls back
    to "simt" -- another GPU kernel, not the host -- if a query has too many points inside the TF32 error band)
    or None = $MUON_B200_KNN, default "tc"."""
    require_cuda()
    Y = X if Y is None else Y
    assert X.dtype == torch.float32 and Y.dtype == torch.float32 and X.is_contiguous() and Y.is_contiguous()
    assert X.shape[1] == Y.shape[1]
    if query_chunk is not None and X.shape[0] > query_chunk:
        # bounded workspace ("low_memory"): the queries in blocks, every block against all of Y -- same result
        parts = [knn_l2(X[q0:q0 + query_chunk], k, Y, algo) for q0 in range(0, X.shape[0], query_chunk)]
        return torch.cat([p[0] for p in parts]), torch.cat([p[1] for p in parts])
    nq, d = X.shape
    idx = torch.empty((nq, k), dtype=torch.int32, device=X.device)
    dist = torch.empty((nq, k), dtype=torch.float32, device=X.device)
    algo = os.environ.get("MUON_B200_KNN", "tc") if algo is None else algo
    if algo == "tc" and d <= 128 and k <= 512:
        nbytes = int(load().mub_knn_l2_tc_workspace_bytes(nq, Y.shape[0], d))
        ws = torch.empty(max(nbytes, 4), dtype=torch.uint8, device=X.device)
        status = torch.zeros(1, dtype=torch.int32, device=X.device)
        call("mub_knn_l2_tc_f32", ptr(X), nq, ptr(Y), Y.shape[0], d, d, k, ptr(idx), ptr(dist), ptr(ws), nbytes,
             ptr(status), stream_ptr())
        st = int(status[0])
        if st == 0:
            return idx, dist
        # st & 2: error band too crowded for some query -> exact SIMT kernel below
    elif algo not in ("simt", "tc"):
        raise ValueError(f"unknown kNN algorithm {algo!r}")
    if k > 320:
        raise NotImplementedError(f"knn_l2: k = {k} > 320 needs the tensor-core path, which declined this input (more than 896 "
                                  "points inside a query's TF32 error band, or d > 128); the fp32 SIMT kernel supports k <= 320")
    call("mub_knn_l2_f32", ptr(X), nq, ptr(Y), Y.shape[0], d, d, k, ptr(idx), ptr(dist), stream_ptr())
    return idx, dist
