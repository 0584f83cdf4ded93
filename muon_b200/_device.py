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
from ._lib import (SPMM_ROWS_SORTED, TFIDF_BINARIZE, TFIDF_LOG_IDF, TFIDF_LOG_TF, TFIDF_LOG_TFIDF, TFIDF_NO_SCALE,
                   MuonB200Error, call, load, ptr, stream_ptr)

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
                   to_device(data, device, dtype), X.shape,
                   sorted_indices=bool(getattr(X, "has_sorted_indices", False)))

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

    def transpose_panels(self, pad: int = 64) -> "TransposedPanels":
        key = ("panels", pad)
        if getattr(self, "_tp", None) is None or self._tp[0] != key:
            self._tp = (key, TransposedPanels(self, pad))
        return self._tp[1]


class DevicePairs:
    """CSR whose entries are interleaved 8-byte {int32 index, float32 value} pairs (``pairs``: int32 [nnz, 2]).
    Used for the transposed row panels: one scattered store per non-zero when building, one 8-byte load per
    entry when multiplying.  ``sorted_indices``: every row lists its columns in ascending order."""

    def __init__(self, indptr, pairs, shape, sorted_indices: bool = False):
        self.indptr, self.pairs = indptr, pairs
        self.shape = (int(shape[0]), int(shape[1]))
        self.sorted_indices = sorted_indices

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


class _EntryCounts:
    """The entry counts of an n x d matrix that TransposedPanels reads from ``A._aux``: ``col_counts`` =
    (chunk_bounds(n), int32 [N_CHUNKS][d] per (row chunk, column)) and ``rb_counts`` = uint16 [ceil(n / 512)][d] per
    (512-row block, column), held as int16.  The tiled TF-IDF reduce pass leaves them as a side product."""

    def __init__(self, n: int, d: int, device):
        self.bounds = chunk_bounds(n)
        self.counts = torch.zeros((N_CHUNKS, d), dtype=torch.int32, device=device)
        self._bounds_dev = torch.tensor(self.bounds, dtype=torch.int64, device=device)
        self.rb_counts = torch.empty((-(-n // tile_rows()), d), dtype=torch.int16, device=device)

    def reduce(self, A: DeviceCSR, row_sum, col_sum, status, flags: int, r0: int = 0, r1: Optional[int] = None,
               stream=None):
        """The tiled reduce pass (shared-memory tiles, ~30x fewer global atomics than mub_tfidf_reduce_f32) over rows
        [r0, r1) of A, float32 values, r0 a multiple of the tile height: their sums into row_sum[r0:r1], their column
        sums added to col_sum, their entry counts into these buffers, the canonical-form verdict ORed into status.
        Bit0 of the verdict (a row not sorted) means none of the sums or counts are valid."""
        n, d = A.shape
        r1 = n if r1 is None else r1
        call("mub_tfidf_reduce_tiled_f32", ptr(A.indptr) + 8 * r0, ptr(A.indices), ptr(A.data), r1 - r0, d,
             ptr(row_sum) + 4 * r0, ptr(col_sum), ptr(status), flags, ptr(self.counts), ptr(self._bounds_dev), N_CHUNKS,
             r0, ptr(self.rb_counts), stream_ptr() if stream is None else stream)

    def record(self, A: DeviceCSR):
        """Attach the counts to A: its transposed panels then skip the counting pass and take the tiled fill."""
        aux = getattr(A, "_aux", None) or {}
        aux.update({"col_counts": (self.bounds, self.counts), "rb_counts": self.rb_counts})
        A._aux = aux


def _tfidf_flags(log_tf, log_idf, log_tfidf, scale_factor, binarize=False):
    """The TF-IDF kernels' flag word and the scale factor they apply (1.0 when there is none)."""
    flags = (TFIDF_LOG_TF if log_tf else 0) | (TFIDF_LOG_IDF if log_idf else 0) | (TFIDF_LOG_TFIDF if log_tfidf else 0)
    if scale_factor is None or scale_factor == 0 or scale_factor == 1:
        flags |= TFIDF_NO_SCALE
        scale_factor = 1.0
    if binarize:
        flags |= TFIDF_BINARIZE
    return flags, scale_factor


def tfidf_csr(A: DeviceCSR, log_tf=True, log_idf=True, log_tfidf=False, scale_factor=1e4,
              inplace_values=False, check_canonical=False, binarize=False) -> Optional[DeviceCSR]:
    """K1: two fused passes (reduce, apply).  Column sums are allreduced across cell shards
    (muon/_atac/preproc.py:92-119; multi-GPU plan SURVEY section 8e).  float32 values with sorted rows take the tiled
    reduce pass, and the result carries the entry counts of its transposition; anything else takes the order-agnostic
    kernel and carries none."""
    require_cuda()
    n, d = A.shape
    sfx = "f32" if A.data.dtype == torch.float32 else "f64"
    flags, scale_factor = _tfidf_flags(log_tf, log_idf, log_tfidf, scale_factor, binarize)
    dev, dt = A.data.device, A.data.dtype
    row_sum = torch.empty(n, dtype=dt, device=dev)
    col_sum = torch.zeros(d, dtype=dt, device=dev)
    st = stream_ptr()
    status = torch.zeros(1, dtype=torch.int32, device=dev) if check_canonical else None
    counts = None
    if sfx == "f32" and A.sorted_indices and n > 0:
        st_t = torch.zeros(1, dtype=torch.int32, device=dev)
        counts = _EntryCounts(n, d, dev)
        counts.reduce(A, row_sum, col_sum, st_t, flags, stream=st)
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
        counts.record(res)
    return res


def row_range(rows, n: int):
    """(lo, hi) if ``rows`` (None = all n rows, else a 1-D integer array) is the ascending range lo, lo+1, ..., hi-1,
    else None.  An empty list is the empty range (0, 0)."""
    if rows is None:
        return 0, n
    r = np.asarray(rows)
    if r.size == 0:
        return 0, 0
    lo = int(r[0])
    return (lo, lo + r.size) if np.array_equal(r, np.arange(lo, lo + r.size)) else None


def select_is_view(rows, col_mask, n: int) -> bool:
    """True when ``csr_select(A, rows, col_mask)`` of an n-row A returns a view of A's arrays (nothing copied): no
    column mask and the rows an ascending range.  Otherwise the selected entries are gathered into new arrays."""
    return col_mask is None and row_range(rows, n) is not None


def attach_block_counts(A: DeviceCSR) -> DeviceCSR:
    """Give A the per-(row chunk, column) and per-(512-row block, column) entry counts that TransposedPanels needs for
    the deterministic tiled fill: the TF-IDF reduce pass run with flags = 0, its sums discarded.  A matrix whose rows
    are not sorted, or whose values are not float32, is left without counts (its panels then take the atomic-cursor
    fill)."""
    n, d = A.shape
    if not A.sorted_indices or n == 0 or d == 0 or A.data.dtype != torch.float32:
        return A
    dev = A.data.device
    counts = _EntryCounts(n, d, dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    counts.reduce(A, torch.empty(n, dtype=torch.float32, device=dev), torch.zeros(d, dtype=torch.float32, device=dev),
                  status, 0)
    if int(status[0]) & 1:
        A.sorted_indices = False
    else:
        counts.record(A)
    return A


def csr_select(A: DeviceCSR, rows=None, col_mask=None) -> DeviceCSR:
    """``A[rows][:, col_mask]`` on the device (csrc/select.cu), as a new DeviceCSR with float32 values.

    ``rows``: source row of every output row (int array, any order, repeats allowed; None = all rows).  ``col_mask``:
    boolean per column of A (None = keep all); the kept columns are renumbered in order, so sorted rows stay sorted.
    An ascending row range without a column mask is a view: ``indices`` / ``data`` are narrowed, not copied, and only
    ``indptr`` is rebased (8 B per row).  Anything else is counted, scanned and filled into new arrays (8 B per kept
    entry).  ``select_is_view`` states the rule.  With ``rows=None`` the result keeps A's shard position (``row0``,
    ``n_total``); any other row selection is a matrix of its own (row0 = 0, n_total = its height).  Every result
    carries the entry counts of the deterministic transposition fill (``attach_block_counts``)."""
    require_cuda()
    assert A.data.dtype == torch.float32, "csr_select: float32 values only (convert fp64 first)"
    n_src, d = A.shape
    dev = A.data.device
    st = stream_ptr()
    col_map, d_out = None, d
    if col_mask is not None:
        mask = np.asarray(col_mask.cpu() if isinstance(col_mask, torch.Tensor) else col_mask, dtype=bool).reshape(-1)
        if mask.shape[0] != d:
            raise ValueError(f"csr_select: col_mask has {mask.shape[0]} entries, the matrix {d} columns")
        cmap = np.full(d, -1, dtype=np.int32)
        d_out = int(mask.sum())
        cmap[mask] = np.arange(d_out, dtype=np.int32)
        col_map = torch.from_numpy(cmap).to(dev)
    r_host = None
    if rows is not None:
        r_host = np.asarray(rows.cpu() if isinstance(rows, torch.Tensor) else rows).reshape(-1)
        if r_host.size and r_host.dtype.kind not in "iu":
            raise TypeError(f"csr_select: rows must be integers, got {r_host.dtype}")
        r_host = r_host.astype(np.int64, copy=False)
        if r_host.size and (int(r_host.min()) < 0 or int(r_host.max()) >= n_src):
            raise IndexError(f"csr_select: row ids must lie in [0, {n_src}), got [{int(r_host.min())}, {int(r_host.max())}]")
    n_out = n_src if r_host is None else int(r_host.size)
    # every row, in order: the same cells, so the same place in a cell-sharded matrix
    shard = {"row0": A.row0, "n_total": A._n_total} if r_host is None else {"row0": 0, "n_total": n_out}
    if select_is_view(r_host, col_mask, n_src):
        lo, hi = row_range(r_host, n_src)
        k0, k1 = (int(x) for x in A.indptr[[lo, hi]].tolist())
        out = DeviceCSR(A.indptr[lo:hi + 1] - k0, A.indices[k0:k1], A.data[k0:k1], (n_out, d),
                        sorted_indices=A.sorted_indices, **shard)
        return attach_block_counts(out)
    if n_out == 0:
        return DeviceCSR(torch.zeros(1, dtype=torch.int64, device=dev), torch.empty(0, dtype=torch.int32, device=dev),
                         torch.empty(0, dtype=torch.float32, device=dev), (0, d_out), sorted_indices=A.sorted_indices,
                         **shard)
    rows_dev = None if r_host is None else torch.from_numpy(np.ascontiguousarray(r_host)).to(dev)
    lens = torch.zeros(n_out + 1, dtype=torch.int64, device=dev)
    call("mub_csr_select_count", ptr(A.indptr), ptr(A.indices), n_src, d, ptr(rows_dev), n_out, ptr(col_map),
         ptr(lens) + 8, st)
    indptr = torch.cumsum(lens, 0)
    del lens
    nnz = int(indptr[-1])
    indices = torch.empty(nnz, dtype=torch.int32, device=dev)
    data = torch.empty(nnz, dtype=torch.float32, device=dev)
    call("mub_csr_select_fill_f32", ptr(A.indptr), ptr(A.indices), ptr(A.data), d, ptr(rows_dev), n_out, ptr(col_map),
         ptr(indptr), ptr(indices), ptr(data), st)
    out = DeviceCSR(indptr, indices, data, (n_out, d_out), sorted_indices=A.sorted_indices, **shard)
    return attach_block_counts(out)


def _transposed_indptr(A: DeviceCSR, k0: int, k1: int, col_count: Optional[torch.Tensor]) -> torch.Tensor:
    """Row offsets of the transpose of the rows of A that hold the non-zeros [k0, k1): scanned from ``col_count`` (their
    entries per column) when it is known, else from a counting pass."""
    d = A.shape[1]
    t_count = torch.zeros(d + 1, dtype=torch.int64, device=A.data.device)
    if col_count is not None:
        t_count[1:] = col_count
    else:
        call("mub_csr_transpose_count", ptr(A.indices) + 4 * k0, k1 - k0, d, ptr(t_count), stream_ptr())
    return torch.cumsum(t_count, 0)


def csr_transpose(A: DeviceCSR) -> DeviceCSR:
    """The CSR of A^T on the device (count -> scan -> atomic-cursor fill).  The order of the entries inside a transposed
    row follows the fill's slot claims."""
    require_cuda()
    assert A.data.dtype in (torch.float32, torch.float64), "transpose: float32 or float64 values only"
    n, d = A.shape
    dev = A.data.device
    t_indptr = _transposed_indptr(A, 0, A.nnz, None)
    cursor = torch.empty(max(d, 1), dtype=torch.int64, device=dev)
    t_indices = torch.empty(A.nnz, dtype=torch.int32, device=dev)
    t_data = torch.empty(A.nnz, dtype=A.data.dtype, device=dev)
    call("mub_csr_transpose_fill_f64" if A.data.dtype == torch.float64 else "mub_csr_transpose_fill", ptr(A.indptr),
         ptr(A.indices), ptr(A.data), n, d, 0, ptr(t_indptr), ptr(cursor), ptr(t_indices), ptr(t_data), stream_ptr())
    return DeviceCSR(t_indptr, t_indices, t_data, (d, n), n_total=d, sorted_indices=False)


class TransposedPanels:
    """A^T as a list of row-panel transposes.  A^T Y gathers rows of Y (n x P); when n*P*4 bytes
    exceed what stays resident in L2 the gathers fall through to HBM, so the cells are cut into
    panels whose slice of Y fits in L2 and the products are accumulated panel by panel."""

    # bytes of the gathered operand per panel (H100 L2: 50 MB, shared with the CSR stream)
    L2_BUDGET = int(os.environ.get("MUON_B200_L2_BUDGET_MB", "16")) << 20

    def __init__(self, A: DeviceCSR, pad: int = 64):
        n, d = A.shape
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
                # order on every run (the atomic-cursor fill's order follows slot claims)
                rb = aux.get("rb_counts")
        else:
            bounds = [round(i * n / n_panels) for i in range(n_panels + 1)]
        self.counts_reused = counts is not None
        self.tiled_fill = False
        self.shape = (d, n)
        # non-zero offsets of the panel boundaries: one small D2H up front, no host syncs afterwards
        ks = A.indptr[torch.tensor(bounds, device=A.indptr.device)].tolist()
        spans = [(bounds[i], bounds[i + 1], ks[i], ks[i + 1], counts[i] if counts else None)
                 for i in range(n_panels) if bounds[i + 1] > bounds[i]]
        if rb is not None:
            # the scanned write offsets of the largest panel's 512-row blocks, reused by every panel
            nb = max((-(-(r1 - r0) // tile_rows()) for r0, r1, *_ in spans), default=0)
            tiled = (rb, torch.empty(nb * d, dtype=torch.int32, device=A.data.device),
                     torch.zeros(1, dtype=torch.int32, device=A.data.device))
            self.panels = [self._panel(A, *s, tiled=tiled) for s in spans]
            self.tiled_fill = int(tiled[2][0]) == 0
        if not self.tiled_fill:    # no per-block counts, or they disagree with the pattern (A modified after tfidf)
            self.panels = [self._panel(A, *s) for s in spans]

    @staticmethod
    def _panel(A: DeviceCSR, r0: int, r1: int, k0: int, k1: int, col_count: Optional[torch.Tensor], tiled=None):
        """(r0, r1, (A[r0:r1])^T) in the pairs layout, row indices local to the panel; k0/k1: the non-zero offsets of
        rows r0 and r1.  ``tiled`` = (per-block counts, write-offset buffer, status word) selects the tiled fill, which
        sets bit0 of the status word if the pattern disagrees with the counts; None the atomic-cursor fill."""
        d = A.shape[1]
        dev, st = A.data.device, stream_ptr()
        t_indptr = _transposed_indptr(A, k0, k1, col_count)
        t_pairs = torch.empty((k1 - k0, 2), dtype=torch.int32, device=dev)
        # indptr values are absolute offsets into indices/data, so only the indptr pointer is shifted
        if tiled is not None:
            rb, base, status = tiled
            call("mub_csr_transpose_fill_tiled", ptr(A.indptr) + 8 * r0, ptr(A.indices), ptr(A.data), r1 - r0, d,
                 ptr(rb) + 2 * (r0 // tile_rows()) * d, ptr(t_indptr), ptr(base), ptr(t_pairs), ptr(status), st)
        else:
            cursor = torch.empty(max(d, 1), dtype=torch.int64, device=dev)
            call("mub_csr_transpose_fill_pairs", ptr(A.indptr) + 8 * r0, ptr(A.indices), ptr(A.data), r1 - r0, d, 0,
                 ptr(t_indptr), ptr(cursor), ptr(t_pairs), st)
        # the tiled fill lists every transposed row in ascending cell order (it is only kept if its status is clear)
        return r0, r1, DevicePairs(t_indptr, t_pairs, (d, r1 - r0), sorted_indices=tiled is not None)

    def spmm(self, Y: torch.Tensor, dynamic=True, half: bool = False) -> torch.Tensor:
        """A^T Y accumulated panel by panel.  ``half``: round Y to IEEE half first (see ``spmm``)."""
        d, P = self.shape[0], Y.shape[1]
        if half:
            Y = to_half_scaled(Y)
        out = torch.empty((d, P), dtype=torch.float32, device=Y.device)
        for i, (r0, r1, T) in enumerate(self.panels):
            spmm(T, Y[r0:r1], out=out, accumulate=i > 0, dynamic=dynamic)
        return out

    def spmm_rowblocks(self, Y: torch.Tensor, blocks) -> torch.Tensor:
        """Rows ``blocks`` = [(j0, j1), ...] of A^T Y only, stacked into a compact (sum of block heights) x P buffer
        (fp32 operand).  Used for the sampled residual check of the LSI driver: 1/16 of the rows costs 1/16 of a pass."""
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
    """``rows`` of spmm: None = all rows; (j0, j1) = that row range written to the same rows of ``out``;
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


def spmm(A, B: torch.Tensor, out: Optional[torch.Tensor] = None, accumulate=False, dynamic=True, rows=None,
         scale: float = HALF_SCALE) -> torch.Tensor:
    """K2/K3: C[n x P] (+)= A @ B[d x P];  P = B.shape[1] must be 32, 64 or 128.  A is a ``DeviceCSR`` or
    ``DevicePairs``.  B is float32, or float16 holding B * ``scale`` (``to_half_scaled``): half the bytes per non-zero
    through the L2 -> L1 gather path that bounds the fp32 operand; products and sums stay fp32.  A matrix whose rows
    are sorted (``A.sorted_indices``) is flagged so to the library, which then runs a fp32 product of at least one
    128-row band per SM with the tiled kernel (B staged in shared memory), on CSR arrays and on pairs alike;
    everything else takes the row-warp kernel (``dynamic``: rows claimed from an atomic counter).  Both give the same
    bits."""
    n, d = A.shape
    P = B.shape[1]
    assert B.shape[0] == d and B.dtype in (torch.float32, torch.float16) and B.is_contiguous(), (B.shape, d, B.dtype)
    if out is None:
        assert not accumulate
        out = torch.empty((n, P), dtype=torch.float32, device=B.device)
    flags = SPMM_ROWS_SORTED if A.sorted_indices else 0
    counter = torch.zeros(1, dtype=torch.int64, device=B.device) if dynamic else None
    j0, j1, o0 = _row_range(rows, n)                    # matrix rows [j0, j1) -> out rows [o0, o0 + j1 - j0)
    pairs = isinstance(A, DevicePairs)
    operands = [ptr(A.indptr) + 8 * j0] + ([ptr(A.pairs)] if pairs else [ptr(A.indices), ptr(A.data)])
    operands += [j1 - j0, d, ptr(B), P, ptr(out) + 4 * P * o0, 1 if accumulate else 0]
    if B.dtype == torch.float16:
        call("mub_spmm_csrp_h16" if pairs else "mub_spmm_csr_h16", *operands, 1.0 / scale, ptr(counter), flags,
             stream_ptr())
    else:
        call("mub_spmm_csrp_f32" if pairs else "mub_spmm_csr_f32", *operands, ptr(counter), flags, stream_ptr())
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


def _row_blocks(indptr_host: np.ndarray, block_nnz: int, align: int):
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
    flags, scale_factor = _tfidf_flags(log_tf, log_idf, log_tfidf, scale_factor)
    indptr_h = np.ascontiguousarray(X.indptr)
    indices_h = np.ascontiguousarray(X.indices)
    data_h = np.ascontiguousarray(X.data)
    nnz = int(indptr_h[-1]) if indptr_h.shape[0] else 0
    blocks = _row_blocks(indptr_h, _BLOCK_NNZ, tile_rows())
    st = stager()
    main = torch.cuda.current_stream()
    side = torch.cuda.Stream()
    indptr = to_device(indptr_h, dev, np.int64)
    indices = torch.empty(nnz, dtype=torch.int32, device=dev)
    data = torch.empty(nnz, dtype=torch.float32, device=dev)
    res = DeviceCSR(indptr, indices, data, (n, d))
    row_sum = torch.empty(n, dtype=torch.float32, device=dev)
    col_sum = torch.zeros(d, dtype=torch.float32, device=dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    counts = _EntryCounts(n, d, dev)
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
        # host matrices must be canonical anyway (checked here): sorted rows, so the tiled pass applies
        counts.reduce(res, row_sum, col_sum, status, flags, r0, r1, main.cuda_stream)
    for t in (indices, data):
        t.record_stream(side)
    if int(status[0]) != 0:                     # duplicates / explicit zeros / unsorted rows (also syncs the upload)
        return None
    _dist.all_reduce_sum_(col_sum)
    idf = torch.empty(d, dtype=torch.float32, device=dev)
    call("mub_tfidf_idf_f32", ptr(col_sum), d, float(res.n_total), flags, ptr(idf), main.cuda_stream)
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
    res._aux = {"row_sum": row_sum, "col_sum": col_sum, "idf": idf}
    counts.record(res)
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
