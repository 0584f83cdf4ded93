"""``mu.atac.pp.scopen`` -- scOpen's imputation of ATAC accessibility: bounded NMF of the scaled peak pattern on the GPU.

The reference (muon/_atac/preproc.py:155-236) builds the dense peaks x cells matrix X[p, c] = s_c where
count(c, p) > 0, with s_c = 1 / (1 - rho_c) and rho_c a linear map of log10 of the cell's open regions onto
[min_rho, max_rho], and hands it to ``scopen.MF.non_negative_factorization``: a fork of sklearn's coordinate-descent
NMF.  X is a binary pattern times one scale per cell, so both products of an iteration, X Ht and X^T W, are sparse
gather-sums of O(nnz k), and nothing of size peaks x cells exists on the device except one block of the imputed
output at a time.  csrc/scopen.cu holds the passes:

  * pattern  entries > 0 per cell (duplicates summed first), then their columns in stored order; the transposed
             pattern is ``_device.csr_transpose`` with every row sorted, so each peak's sum runs in cell order;
  * init     NNDSVD from the exact top-k SVD of X, computed by ``_lsi.truncated_svd`` on the fp32 pattern with
             data s_c; the NNDSVD factors are formed on the host in float64, line for line as sklearn's
             ``_initialize_nmf`` does;
  * fit      per iteration W then H, each a float64 Gram (k x k), a pattern SpMM and a coordinate-descent sweep
             (csrc/scopen.cu, one row per warp, components in order); the host reads one violation per sweep;
  * impute   clip(W H, 0, 1) block by block of peak rows into the preallocated float64 host array.

The solver contract lives in this module alone.  Items marked [recalled] come from scOpen's MF.py as remembered, not
as read (the package is not a dependency of this project); each is a named constant here so that it can be
corrected in one place:
  * [recalled] the fork's defaults: init "nndsvd" with eps = 1e-6 truncation (INIT_EPS), solver "cd",
    tol = 1e-4 (TOL), l1_ratio = 0, and the pre-1.0 regularisation "both", unscaled: l2_reg_W = l2_reg_H = alpha;
  * [recalled] the bound: every coordinate update is projected onto [0, UPPER] = [0, 1]; the projected-gradient
    violation stays sklearn's (min(0, grad) where the coordinate is 0, else grad);
  * [recalled] a non-finite scale is rejected by the solver's input validation (NOT_FINITE).
Everything else follows sklearn's ``_fit_coordinate_descent``: stop when violation / violation_at_iteration_1 <= tol,
or when the first violation is 0; reaching ``max_iter`` with tol > 0 warns (NOT_CONVERGED).

Divergences (DESIGN.md section 8): the SVD of the init is the exact top-k one (to the fp32 Krylov driver's
tolerance) instead of sklearn's unseeded ``randomized_svd``, so a call is deterministic; every sum of the fit is
float64 in a fixed order, so two calls return the same bits.  Refused with NotImplementedError before any device
work: n_components > 64, more than 2^31 - 1 cells or peaks, and a fit larger than free device memory.
"""
from __future__ import annotations

import numbers
import time
import warnings

import numpy as np

from ._lib import SCOPEN_MAX_COMPONENTS
from .prot.pp import ConvergenceWarning

TOL = 1e-4                 # [recalled] the fork's default tol
INIT_EPS = 1e-6            # [recalled] NNDSVD truncation: entries below it are set to 0
UPPER = 1.0                # [recalled] the fork's bound on every coordinate of W and H
SVD_TOL = 1e-5             # relative residual of the init's singular triplets (fp32 Krylov driver)
SVD_SEED = 0
MAX_DIM = 2**31 - 1        # int32 indices of the pattern
IMPUTE_BLOCK_BYTES = 256 << 20

NOT_FINITE = "Input contains NaN, infinity or a value too large for dtype('float64')."   # [recalled]
NOT_CONVERGED = "Maximum number of iterations %d reached. Increase it to improve convergence."


def _is_int(v):
    return isinstance(v, numbers.Integral) and not isinstance(v, (bool, np.bool_))


def resolve(data):
    """The AnnData scOpen works on, as the reference resolves it."""
    from ._containers import is_anndata, is_mudata
    if is_anndata(data):
        return data
    if is_mudata(data) and "atac" in data.mod:
        return data.mod["atac"]
    raise TypeError("Expected AnnData or MuData object with 'atac' modality")


def check_params(n_components, max_iter, m, n):
    """The solver's parameter errors (ValueError), then the refusals (NotImplementedError) that need only the shape."""
    if not (_is_int(n_components) and n_components >= 1):
        raise ValueError("Number of components must be a positive integer; got (n_components=%r)" % (n_components,))
    if not (_is_int(max_iter) and max_iter >= 0):
        raise ValueError("Maximum number of iterations must be a positive integer; got (max_iter=%r)" % (max_iter,))
    if n_components > min(m, n):
        raise ValueError("init = 'nndsvd' can only be used when n_components <= min(n_samples, n_features)")
    if n_components > SCOPEN_MAX_COMPONENTS:
        raise NotImplementedError(f"scopen with {n_components} components: at most {SCOPEN_MAX_COMPONENTS} are "
                                  "supported on the GPU")
    if max(m, n) > MAX_DIM:
        raise NotImplementedError(f"scopen of {n} cells x {m} peaks: at most {MAX_DIM} of either are supported")


def scale_of(counts, min_rho, max_rho):
    """s_c = 1 / (1 - rho_c) from the open regions per cell, in float64 as the reference computes it; ValueError if
    a scale is not finite (a cell without open regions, all cells with equal counts, or rho == 1)."""
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.log10(np.asarray(counts, dtype=np.float64))
        rmax, rmin = np.max(r), np.min(r)
        rho = min_rho + (max_rho - min_rho) * (rmax - r) / (rmax - rmin)
        s = 1 / (1 - rho)
    if not np.all(np.isfinite(s)):
        raise ValueError(NOT_FINITE)
    return s


def host_pattern_source(X):
    """Host input as a CSR without duplicates (summed, as ``toarray`` sums them) and its positives per row."""
    import scipy.sparse as sp
    if sp.issparse(X):
        X = sp.csr_matrix(X, copy=True)
        X.sum_duplicates()
    else:
        X = sp.csr_matrix(np.asarray(X))
    if X.dtype not in (np.float32, np.float64):
        X = X.astype(np.float64)
    pos = np.concatenate([[0], np.cumsum(X.data > 0)])
    return X, np.diff(pos[X.indptr])


def nndsvd(U, S, V, eps=INIT_EPS):
    """sklearn's ``_initialize_nmf(init="nndsvd")`` from a given SVD X ~ U diag(S) V (U [m x k], V [k x n]), float64."""
    U, S, V = (np.asarray(a, dtype=np.float64) for a in (U, S, V))
    W = np.zeros_like(U)
    H = np.zeros_like(V)
    W[:, 0] = np.sqrt(S[0]) * np.abs(U[:, 0])
    H[0, :] = np.sqrt(S[0]) * np.abs(V[0, :])
    for j in range(1, U.shape[1]):
        x, y = U[:, j], V[j, :]
        x_p, y_p = np.maximum(x, 0), np.maximum(y, 0)
        x_n, y_n = np.abs(np.minimum(x, 0)), np.abs(np.minimum(y, 0))
        x_p_nrm, y_p_nrm = np.sqrt(np.dot(x_p, x_p)), np.sqrt(np.dot(y_p, y_p))
        x_n_nrm, y_n_nrm = np.sqrt(np.dot(x_n, x_n)), np.sqrt(np.dot(y_n, y_n))
        m_p, m_n = x_p_nrm * y_p_nrm, x_n_nrm * y_n_nrm
        if m_p > m_n:
            u, v, sigma = x_p / x_p_nrm, y_p / y_p_nrm, m_p
        else:
            u, v, sigma = x_n / x_n_nrm, y_n / y_n_nrm, m_n
        lbd = np.sqrt(S[j] * sigma)
        W[:, j] = lbd * u
        H[j, :] = lbd * v
    W[W < eps] = 0
    H[H < eps] = 0
    return W, H


def device_bytes(n, m, nnz, itemsize, k):
    """Device bytes of one fit: the uploaded input (none for a resident one: ``itemsize`` None), the pattern and its
    sorted transpose (with the sort's keys), the SVD's Krylov basis, the factors with their products, the workspace
    and one imputation block."""
    from ._device import pad_width
    from ._lib import load
    P = pad_width(k)
    upload = 0 if itemsize is None else 8 * (n + 1) + nnz * (4 + itemsize)
    pattern = 8 * (n + 1) + 8 * (m + 1) + 16 * nnz          # indices + fp32 data, both ways
    transpose = 24 * nnz + 8 * m                             # keys, sorted keys and sort order
    svd = 4 * (m + n) * P * 20
    factors = 16 * (m + n) * k
    ws = int(load().mub_scopen_workspace_bytes(max(m, n), k))
    block = min(IMPUTE_BLOCK_BYTES, 8 * m * n)
    return upload + pattern + max(transpose, svd + factors + ws + block) + 8 * (n + m) + (1 << 20)


def check_memory(n, m, nnz, itemsize, k):
    from ._snf import free_device_bytes
    need = device_bytes(n, m, nnz, itemsize, k)
    free = free_device_bytes()
    if need > free:
        raise NotImplementedError(f"scopen of {n} cells x {m} peaks ({nnz} stored entries) needs "
                                  f"{need / 2**30:.1f} GiB of device memory; {free / 2**30:.1f} GiB are free")


class SvdOperator:
    """The pattern with data s_c as a ``truncated_svd`` operator: A [cells x peaks] = X^T, so the SVD's U is X's V^T
    and its V is X's U.  Both products are row-warp SpMMs over sorted rows; nothing is summed over ranks."""

    def __init__(self, P, PT):
        from . import _device
        self._dev = _device
        self.P, self.PT = P, PT
        self.n_total, self.d = P.shape
        self.device = P.device

    def av(self, V):
        return self._dev.spmm(self.P, V, dynamic=False)

    def aty(self, Y):
        return self._dev.spmm(self.PT, Y, dynamic=True)

    def gram(self, Y, l):
        return self._dev.gram(Y, l, reduce=False)

    gram_local = gram


class Fit:
    """The device side of one scOpen fit: the pattern, its transpose, the factors and the calls on them.

    ``X`` is the cells x peaks input (a ``DeviceCSR``, or a duplicate-free scipy CSR from ``host_pattern_source``)."""

    def __init__(self, X, k):
        import torch

        from . import _device
        _device.require_cuda()
        self.k = int(k)
        self.A = X if isinstance(X, _device.DeviceCSR) else _device.DeviceCSR.from_scipy(X)
        self.n, self.m = self.A.shape
        self.dev = self.A.device
        self.sfx = "f64" if self.A.data.dtype == torch.float64 else "f32"
        self.counts_dev = None

    def _call(self, name, *args):
        from ._lib import call, stream_ptr
        call(name, *args, stream_ptr())

    def positives(self):
        """Entries > 0 per cell (int64, host)."""
        import torch

        from ._lib import ptr
        self.counts_dev = torch.empty(self.n, dtype=torch.int64, device=self.dev)
        self._call(f"mub_scopen_pattern_count_{self.sfx}", ptr(self.A.indptr), ptr(self.A.data), self.n,
                   ptr(self.counts_dev))
        return self.counts_dev.cpu().numpy()

    def build(self, s):
        """The pattern (fp32 data s_c), its transpose with every row in cell order, and the float64 scales."""
        import torch

        from . import _device
        from ._lib import ptr
        if self.counts_dev is None:
            self.positives()
        indptr = torch.zeros(self.n + 1, dtype=torch.int64, device=self.dev)
        torch.cumsum(self.counts_dev, 0, out=indptr[1:])
        nnz = int(indptr[-1])
        self.s = torch.from_numpy(np.ascontiguousarray(s, dtype=np.float64)).to(self.dev)
        s32 = self.s.to(torch.float32)
        indices = torch.empty(max(nnz, 1), dtype=torch.int32, device=self.dev)
        data = torch.empty(max(nnz, 1), dtype=torch.float32, device=self.dev)
        self._call(f"mub_scopen_pattern_fill_{self.sfx}", ptr(self.A.indptr), ptr(self.A.indices), ptr(self.A.data),
                   self.n, ptr(indptr), ptr(s32), ptr(indices), ptr(data))
        self.P = _device.DeviceCSR(indptr, indices[:nnz], data[:nnz], (self.n, self.m), n_total=self.n,
                                   sorted_indices=self.A.sorted_indices)
        del self.A, self.counts_dev
        T = _device.csr_transpose(self.P)
        rows = torch.repeat_interleave(torch.arange(self.m, device=self.dev), T.indptr[1:] - T.indptr[:-1])
        keys = torch.sort(rows * self.n + T.indices.to(torch.int64)).values
        t_indptr = T.indptr
        del rows, T
        t_indices = (keys % self.n).to(torch.int32)
        del keys
        self.PT = _device.DeviceCSR(t_indptr, t_indices, s32[t_indices.to(torch.int64)], (self.m, self.n),
                                    n_total=self.m, sorted_indices=True)
        self.nnz = nnz

    def svd(self):
        """(U [m x k], S [k], V [k x n]) of X, float64 on the host."""
        from . import _device
        from ._lsi import truncated_svd
        k = self.k
        U, S, V, _ = truncated_svd(SvdOperator(self.P, self.PT), k, pad_to=_device.pad_width(k), tol=SVD_TOL,
                                   seed=SVD_SEED)
        return (V[:, :k].cpu().numpy().astype(np.float64), S[:k].cpu().numpy().astype(np.float64),
                U[:, :k].cpu().numpy().astype(np.float64).T)

    def set_factors(self, W, H):
        import torch

        from ._lib import load
        f64 = dict(dtype=torch.float64, device=self.dev)
        self.W = torch.from_numpy(np.ascontiguousarray(W, dtype=np.float64)).to(self.dev)
        self.Ht = torch.from_numpy(np.ascontiguousarray(np.asarray(H, dtype=np.float64).T)).to(self.dev)
        self.XHt = torch.empty((self.m, self.k), **f64)
        self.XtW = torch.empty((self.n, self.k), **f64)
        self.G = torch.empty((self.k, self.k), **f64)
        self.viol = torch.empty(2, **f64)
        ws = int(load().mub_scopen_workspace_bytes(max(self.m, self.n), self.k))
        self.ws = torch.empty(max(ws, 8), dtype=torch.uint8, device=self.dev)

    def products(self, which):
        """XHt = X Ht (``which`` = "W") or XtW = X^T W ("H"), and the Gram of the other factor."""
        from ._lib import ptr
        if which == "W":
            self._call("mub_scopen_gram_f64", ptr(self.Ht), self.n, self.k, ptr(self.ws), ptr(self.G))
            self._call("mub_scopen_spmm_f64", ptr(self.PT.indptr), ptr(self.PT.indices), self.m, None, ptr(self.s),
                       ptr(self.Ht), self.k, ptr(self.XHt))
        else:
            self._call("mub_scopen_gram_f64", ptr(self.W), self.m, self.k, ptr(self.ws), ptr(self.G))
            self._call("mub_scopen_spmm_f64", ptr(self.P.indptr), ptr(self.P.indices), self.n, ptr(self.s), None,
                       ptr(self.W), self.k, ptr(self.XtW))

    def sweep(self, which, alpha, upper):
        from ._lib import ptr
        if which == "W":
            self._call("mub_scopen_cd_f64", ptr(self.W), self.m, self.k, ptr(self.G), float(alpha), ptr(self.XHt),
                       float(upper), ptr(self.ws), ptr(self.viol))
        else:
            self._call("mub_scopen_cd_f64", ptr(self.Ht), self.n, self.k, ptr(self.G), float(alpha), ptr(self.XtW),
                       float(upper), ptr(self.ws), ptr(self.viol) + 8)

    def iterate(self, alpha, upper):
        """One iteration, W then H; returns the two sweeps' violations."""
        self.products("W")
        self.sweep("W", alpha, upper)
        self.products("H")
        self.sweep("H", alpha, upper)
        v = self.viol.cpu().numpy()
        return float(v[0]), float(v[1])

    def factors(self):
        """(W [m x k], H [k x n]) float64 on the host."""
        return self.W.cpu().numpy(), self.Ht.cpu().numpy().T.copy()

    def impute(self, out):
        """out[:] = clip(W H, 0, 1), m x n float64 C-ordered host array, block by block of peak rows."""
        import torch

        from . import _device
        from ._lib import ptr
        rows = max(1, min(self.m, IMPUTE_BLOCK_BYTES // max(8 * self.n, 1), 65535 * 16))
        buf = torch.empty(rows * self.n, dtype=torch.float64, device=self.dev)
        for p0 in range(0, self.m, rows):
            p1 = min(self.m, p0 + rows)
            self._call("mub_scopen_impute_f64", ptr(self.W), p0, p1, ptr(self.Ht), self.n, self.k, ptr(buf))
            _device.to_host(buf[:(p1 - p0) * self.n], out=out[p0:p1].reshape(-1))
        return out


def solve(fit, max_iter, alpha, upper=UPPER, tol=TOL, verbose=False):
    """sklearn's ``_fit_coordinate_descent`` loop over ``fit.iterate``; returns n_iter."""
    n_iter = 0
    violation_init = None
    for n_iter in range(1, max_iter + 1):
        vw, vh = fit.iterate(alpha, upper)
        violation = 0.0
        violation += vw
        violation += vh
        if n_iter == 1:
            violation_init = violation
        if violation_init == 0:
            break
        if verbose:
            print("violation:", violation / violation_init)
        if violation / violation_init <= tol:
            if verbose:
                print("Converged at iteration", n_iter + 1)
            break
    return n_iter


def _input(adata):
    """(source for ``Fit``, n cells, m peaks, stored entries, bytes per value to upload (None: resident), host
    positives per cell (None: counted on the device))."""
    from ._device import DeviceCSR
    X = adata.X
    if isinstance(X, DeviceCSR):
        return X, X.shape[0], X.shape[1], X.nnz, None, None
    src, counts = host_pattern_source(X)
    return src, src.shape[0], src.shape[1], src.nnz, src.dtype.itemsize, counts


def scopen(data, n_components=30, max_iter=500, min_rho=0.0, max_rho=0.5, alpha=1, verbose=False):
    """Impute ATAC accessibility with scOpen -- ``muon.atac.pp.scopen`` (muon/_atac/preproc.py:155-236).

    ``data`` is an AnnData, or a MuData with an "atac" modality (else TypeError).  Its ``X`` (cells x peaks: any
    scipy sparse format, a dense array, or a :class:`muon_b200.DeviceCSR` without duplicate entries) counts as open
    where an entry is > 0.  Writes the reference's slots: ``obsm["X_scopen"]`` = H^T (cells x k),
    ``varm["scopen"]`` = W (peaks x k) and ``X`` = M^T, M = clip(W H, 0, 1) a peaks x cells float64 C-ordered array,
    so ``X`` is the same F-ordered view the reference stores.  Prints the reference's lines, and with ``verbose``
    sklearn's per-iteration violations; reaching ``max_iter`` warns with ConvergenceWarning.

    The fit runs on the GPU in float64 and never forms the dense matrix there; two calls return the same bits.  The
    host output (8 bytes per cell and peak) is allocated before any device work.  More than 64 components, more than
    2^31 - 1 cells or peaks, and a fit that does not fit in free device memory raise NotImplementedError."""
    adata = resolve(data)
    start = time.time()
    src, n, m, nnz, itemsize, counts = _input(adata)
    check_params(n_components, max_iter, m, n)
    k = int(n_components)
    M = np.empty((m, n), dtype=np.float64)
    check_memory(n, m, nnz, itemsize, k)

    fit = None
    if counts is None:
        fit = Fit(src, k)
        counts = fit.positives()
    print(f"Number of peaks: {m}\nNumber of cells: {n}")
    print(f"Number of non-zeros before imputation: {int(np.sum(counts))}")
    s = scale_of(counts, min_rho, max_rho)
    if fit is None:
        fit = Fit(src, k)
    fit.build(s)
    W0, H0 = nndsvd(*fit.svd())
    fit.set_factors(W0, H0)
    n_iter = solve(fit, int(max_iter), float(alpha), verbose=verbose)
    if n_iter == max_iter and TOL > 0:
        warnings.warn(NOT_CONVERGED % max_iter, ConvergenceWarning)
    W, H = fit.factors()
    fit.impute(M)
    del fit

    adata.obsm["X_scopen"] = H.T
    adata.varm["scopen"] = W
    adata.X = M.T

    secs = time.time() - start
    mi, sec = divmod(secs, 60)
    h, mi = divmod(mi, 60)
    print("[total time: ", "%dh %dm %ds" % (h, mi, sec), "]")
