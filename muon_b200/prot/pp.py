"""``mu.prot.pp`` -- protein (CITE-seq) preprocessing.  ``dsb`` runs its per-cell mixture fits on the GPU."""
from __future__ import annotations

import numbers
from typing import Iterable, Literal, Optional, Tuple, Union
from warnings import warn

import numpy as np

from .._containers import is_anndata, is_mudata

# host draws of the initial responsibilities staged per chunk (float64 values)
_DRAW_CHUNK = 1 << 23


class ConvergenceWarning(UserWarning):
    """Some of the per-cell mixture fits stopped at the iteration limit."""


def _check_random_state(seed):
    """What sklearn's ``check_random_state`` accepts: None, an int or a RandomState."""
    if seed is None or isinstance(seed, np.random.RandomState):
        return
    if isinstance(seed, numbers.Integral) and not isinstance(seed, (bool, np.bool_)):
        return
    raise ValueError(f"{seed!r} cannot be used to seed a numpy.random.RandomState instance")


def _scaled_dtype(dtype, pseudocount):
    """dtype of ``np.log(X + pseudocount)``: float32 counts stay float32, integer counts become float64."""
    return np.log(np.zeros(1, dtype=dtype) + pseudocount).dtype


def _upload(X, dt, dev):
    """(indptr, indices, data) device tensors of a CSR matrix, or (None, None, data) of a dense one, with the
    values in ``dt``.  Duplicate CSR entries are summed first, as ``toarray()`` does."""
    import scipy.sparse as sp
    import torch
    if sp.issparse(X):
        X = sp.csr_matrix(X)
        if not X.has_canonical_format:
            X = X.copy()
            X.sum_duplicates()
        return (torch.from_numpy(X.indptr.astype(np.int64)).to(dev),
                torch.from_numpy(X.indices.astype(np.int32, copy=False)).to(dev),
                torch.from_numpy(np.ascontiguousarray(X.data, dtype=dt)).to(dev))
    return None, None, torch.from_numpy(np.ascontiguousarray(np.asarray(X), dtype=dt)).to(dev)


def _quantiles_linear(n, qs, value_at, dtype):
    """``np.quantile(a, qs)`` (method "linear") of an array of ``n`` values of ``dtype`` from two of its order
    statistics each: ``value_at(k)`` is the k-th smallest value.  Same index and interpolation arithmetic as
    numpy (virtual index ``(n - 1) q``, lerp from the nearer end)."""
    out = []
    for q in np.asarray(qs, dtype=np.float64):
        v = (n - 1) * q
        lo = np.floor(v)
        hi = lo + 1
        if v >= n - 1:
            lo = hi = n - 1
        elif v < 0:
            lo = hi = 0
        gamma = np.asarray([v - np.floor(v)])
        a = np.asarray([value_at(int(lo))], dtype=dtype)
        b = np.asarray([value_at(int(hi))], dtype=dtype)
        diff = b - a
        r = a + diff * gamma
        if gamma[0] >= 0.5:
            r = b - diff * (1 - gamma)
        out.append(r[0])
    return np.asarray(out)


def dsb(
    data,
    data_raw=None,
    pseudocount: numbers.Integral = 10,
    denoise_counts: bool = True,
    isotype_controls: Optional[Iterable[str]] = None,
    empty_counts_range: Optional[Tuple[numbers.Real, numbers.Real]] = None,
    cell_counts_range: Optional[Tuple[numbers.Real, numbers.Real]] = None,
    scale_factor: Literal["standardize", "mean_subtract"] = "standardize",
    quantile_clipping: bool = False,
    quantile_clip: Tuple[float, float] = (0.001, 0.9995),
    add_layer: bool = False,
    random_state: Optional[Union[int, np.random.RandomState]] = None,
    *,
    return_info: bool = False,
):
    """Normalise protein counts with DSB (Denoised and Scaled by Background; Mulè et al. 2022) -- drop-in for
    ``muon.prot.pp.dsb`` (reference muon/_prot/preproc.py:17-224; same arguments, branches, errors, warnings
    and slots).

    Counts are log-transformed with ``pseudocount``, centred (and with ``scale_factor="standardize"`` scaled) by
    the empty droplets, and -- with ``denoise_counts`` -- each cell's background level ``bgmean`` is estimated
    from two 2-component Gaussian mixtures over its protein values (shared and separate variances, the one
    with the smaller BIC wins).  The regression of every protein on ``bgmean`` (or on the first principal
    component of ``bgmean`` and the isotype controls) is then subtracted.  The result is written to
    ``X`` (or ``layers["dsb"]``) of ``data`` or ``data.mod["prot"]`` as a dense array.

    ``data_raw=None``: ``data`` is the unfiltered MuData with ``rna`` and ``prot``; cells and empty droplets are
    chosen by their log10 RNA counts and the filtered MuData is returned.  Otherwise ``None`` is returned.

    The work runs on the GPU (``csrc/dsb.cu``): one pass over the empty droplets (stored entries only, never
    densified), one fused kernel that scales each cell's row and fits both mixtures in float64 (one warp per
    cell, at most 1024 proteins), and one reduction plus one apply kernel for the regression and the clip.
    Counts may be dense arrays or scipy sparse matrices of float32 (computed in float32 like the reference),
    float64, integer or bool dtype (both computed in float64).

    ``random_state`` is used as the reference uses it: an int gives every fit the same initial draw, while a
    RandomState (or None: numpy's global generator) is consumed cell by cell, 4 * n_proteins values per cell,
    leaving the generator in the state the reference leaves it.  Those draws are made on the host, chunk by
    chunk, while the GPU fits the previous chunk; they cost about 9 ns each (about 7 s for 1M cells x 200
    proteins), so an int seed is much faster on large data.

    Divergences: where the reference warns once per mixture fit that hits the iteration limit, one
    ``ConvergenceWarning`` per call gives the count; float32 counts are fitted in float64, so float32 input can
    differ from the reference (which fits in float32) in the last digits of ``bgmean``.

    ``return_info=True`` returns ``(result, info)``; ``info`` holds the per-cell ``bgmean`` (output dtype),
    ``model`` (0 shared variance, 1 separate variances), ``n_iter`` (cells x 2: shared, separate) and
    ``converged`` (cells x 2), or is empty when ``denoise_counts=False``.
    """
    toreturn = None
    if data_raw is None:
        if empty_counts_range is None or cell_counts_range is None:
            raise ValueError(
                "data_raw is None, assuming data is the unfiltered object, but no count ranges provided")
        if max(*empty_counts_range) > min(*cell_counts_range):
            raise ValueError("overlapping count ranges")
        if not is_mudata(data) or "prot" not in data.mod or "rna" not in data.mod:
            raise TypeError(
                "No data_raw given, assuming data is the unfiltered object, but data is not MuData"
                " or does not contain 'prot' and 'rna' modalities")
        if data.mod["rna"].n_obs != data.mod["prot"].n_obs:
            raise ValueError("different numbers of cells in 'rna' and 'prot' modalities.")
        log10umi = np.log10(np.asarray(data.mod["rna"].X.sum(axis=1)).squeeze() + 1)
        empty_idx = np.where((log10umi >= min(*empty_counts_range)) & (log10umi < max(*empty_counts_range)))[0]
        cell_idx = np.where((log10umi >= min(*cell_counts_range)) & (log10umi < max(*cell_counts_range)))[0]
        cellidx = data.mod["prot"].obs_names[cell_idx]
        empty = data.mod["prot"][empty_idx, :]
        data = data[cellidx, :].copy()
        cells = data.mod["prot"]
        toreturn = data
    elif is_anndata(data_raw):
        empty = data_raw
    elif is_mudata(data_raw) and "prot" in data_raw.mod:
        empty = data_raw.mod["prot"]
    else:
        raise TypeError("data_raw must be an AnnData or a MuData object with 'prot' modality")

    if is_anndata(data):
        cells = data
    elif is_mudata(data) and "prot" in data.mod:
        cells = data.mod["prot"]
    else:
        raise TypeError("data must be an AnnData or a MuData object with 'prot' modality")

    if pseudocount < 0:
        raise ValueError("pseudocount cannot be negative")
    if quantile_clipping:
        if len(quantile_clip) != 2:
            raise ValueError("quantile_clip must have exactly 2 values")
        quantile_clip = np.asarray(quantile_clip)
        if np.any((quantile_clip < 0) | (quantile_clip > 1)):
            raise ValueError("quantile_clip must be between 0 and 1")
    if cells.shape[1] != empty.shape[1]:
        raise ValueError("data and data_raw have different numbers of proteins")

    if empty_counts_range is None:
        warn("empty_counts_range values are not provided, treating all the non-cells as empty droplets")
        empty = empty[~empty.obs_names.isin(cells.obs_names)]
    else:
        warn("empty_counts_range will be deprecated in the future versions", DeprecationWarning, stacklevel=2)
        if data_raw is not None:
            if not is_mudata(data_raw) or "rna" not in data_raw.mod:
                warn("data_raw must be a MuData object with 'rna' modality, ignoring empty_counts_range and "
                     "treating all the non-cells as empty droplets")
                empty = empty[~empty.obs_names.isin(cells.obs_names)]
            else:
                rna = data_raw.mod["rna"]
                log10umi = np.log10(np.asarray(rna.X.sum(axis=1)).squeeze() + 1)
                inrange = (log10umi >= min(*empty_counts_range)) & (log10umi < max(*empty_counts_range))
                droplets = np.asarray(rna.obs_names)[inrange]
                keep = ~np.isin(droplets, np.asarray(cells.obs_names))
                if not keep.all():
                    warn(f"Dropping {int((~keep).sum())} empty droplets as they are already defined as cells")
                empty = empty[droplets[keep]].copy()
    if data_raw is not None and cell_counts_range is not None:
        warn("cell_counts_range values are ignored since cells are provided in data")

    n, P = cells.shape
    if P > 1024:
        raise NotImplementedError(f"dsb supports at most 1024 proteins, got {P}")
    out_dt = _scaled_dtype(cells.X.dtype, pseudocount)
    emp_dt = _scaled_dtype(empty.X.dtype, pseudocount)
    for dt in (out_dt, emp_dt):
        if dt not in (np.float32, np.float64):
            raise NotImplementedError(f"dsb computes in float32 or float64, not {dt}")
    ctrl_idx = np.zeros(0, dtype=np.int32)
    if denoise_counts:
        if P < 2:
            raise ValueError(f"Found array with {P} sample(s) (shape=({P}, 1)) while a minimum of 2 is "
                             "required by GaussianMixture.")
        if n == 0:
            raise ValueError("Found array with 0 sample(s) (shape=(0, 1)) while a minimum of 1 is required "
                             "by LinearRegression.")
        _check_random_state(random_state)
        if isotype_controls is not None:
            isotype_controls = list(isotype_controls)
            ctrl_idx = np.where(np.asarray(cells.var_names.isin(set(isotype_controls))))[0].astype(np.int32)
            if len(ctrl_idx) < len(isotype_controls):
                warn("Some isotype controls are not present in the data.")
            if len(ctrl_idx) > 14:
                raise NotImplementedError(f"dsb supports at most 14 isotype controls, got {len(ctrl_idx)}")

    y, info = _dsb_device(cells.X, empty.X, out_dt, emp_dt, pseudocount, denoise_counts, ctrl_idx,
                          scale_factor == "standardize", quantile_clip if quantile_clipping else None,
                          random_state)
    if add_layer:
        cells.layers["dsb"] = y
    else:
        cells.X = y
    return (toreturn, info) if return_info else toreturn


def _dsb_device(X, E, out_dt, emp_dt, pseudocount, denoise, ctrl_idx, standardize, quantile_clip, random_state):
    import torch

    from .. import _lib
    from .._lib import call, phase, ptr, stream_ptr

    dev = torch.device("cuda", torch.cuda.current_device())
    sfx = "f32" if out_dt == np.float32 else "f64"
    n, P = X.shape
    pc = float(pseudocount)

    with phase("dsb_moments"):
        eptr, eidx, edat = _upload(E, emp_dt, dev)
        n_empty = E.shape[0]
        ws = torch.empty(max(1, _lib.load().mub_dsb_moments_workspace_bytes(n_empty, P)), dtype=torch.uint8,
                         device=dev)
        mean = torch.empty(P, dtype=torch.float64, device=dev)
        std = torch.empty(P, dtype=torch.float64, device=dev)
        call("mub_dsb_moments_" + ("f32" if emp_dt == np.float32 else "f64"), ptr(eptr), ptr(eidx), ptr(edat),
             n_empty, P, pc, ptr(ws), ptr(mean), ptr(std), stream_ptr())
        del eptr, eidx, edat, ws

    tdt = torch.float32 if out_dt == np.float32 else torch.float64
    with phase("dsb_fit"):
        cptr, cidx, cdat = _upload(X, out_dt, dev)
        y = torch.empty((n, P), dtype=tdt, device=dev)
        flags = _lib.DSB_STANDARDIZE if standardize else 0
        info = {}
        if denoise:
            flags |= _lib.DSB_FIT
            bg = torch.empty(n, dtype=torch.float64, device=dev)
            model = torch.empty(n, dtype=torch.int8, device=dev)
            n_iter = torch.empty((n, 2), dtype=torch.int32, device=dev)
            conv = torch.empty((n, 2), dtype=torch.int8, device=dev)
            status = torch.zeros(1, dtype=torch.int32, device=dev)
            outs = (bg, model, n_iter, conv, status)
        else:
            outs = (None,) * 5

        def launch(c0, c1, draws, cell_stride, model_stride):
            rows = (cptr[c0:], cidx, cdat) if cptr is not None else (None, None, cdat[c0:])
            call("mub_dsb_fit_" + sfx, ptr(rows[0]), ptr(rows[1]), ptr(rows[2]), c1 - c0, P, pc, ptr(mean),
                 ptr(std), flags, ptr(draws), cell_stride, model_stride, ptr(y[c0:]),
                 *(None if t is None else ptr(t[c0:]) for t in outs[:4]), ptr(outs[4]), stream_ptr())

        if not denoise or isinstance(random_state, numbers.Integral):
            draws = None
            if denoise:
                draws = torch.from_numpy(np.random.RandomState(random_state).uniform(size=(P, 2))).to(dev)
            launch(0, n, draws, 0, 0)
        else:
            rs = np.random.mtrand._rand if random_state is None else random_state
            chunk = max(1, _DRAW_CHUNK // (4 * P))
            host = [torch.empty(chunk * 4 * P, dtype=torch.float64, pin_memory=True) for _ in range(2)]
            devb = [torch.empty(chunk * 4 * P, dtype=torch.float64, device=dev) for _ in range(2)]
            copied = [None, None]
            stream = torch.cuda.current_stream()
            for k, c0 in enumerate(range(0, n, chunk)):
                c1 = min(n, c0 + chunk)
                b = k % 2
                if copied[b] is not None:
                    copied[b].synchronize()          # the pinned buffer's previous copy has been read
                u = rs.uniform(size=(c1 - c0, 2, P, 2))
                host[b][:u.size].numpy()[:] = u.reshape(-1)
                devb[b][:u.size].copy_(host[b][:u.size], non_blocking=True)
                copied[b] = torch.cuda.Event()
                copied[b].record(stream)
                launch(c0, c1, devb[b], 4 * P, 2 * P)
        del cptr, cidx, cdat
        if denoise:
            if int(status.item()) & 1:
                raise ValueError("Input X contains NaN or infinity: the scaled counts of some cells are not "
                                 "finite (an empty-droplet column with zero standard deviation?).")
            info = {"bgmean": bg.cpu().numpy().astype(out_dt), "model": model.cpu().numpy(),
                    "n_iter": n_iter.cpu().numpy(), "converged": conv.cpu().numpy().astype(bool)}
            n_bad = int((~info["converged"]).sum())
            if n_bad:
                warn(f"{n_bad} of {2 * n} per-cell mixture fits did not converge within 100 iterations; "
                     "consider checking the input", ConvergenceWarning)

    if denoise:
        with phase("dsb_denoise"):
            m = len(ctrl_idx)
            q = m + 1
            ctrl = torch.from_numpy(ctrl_idx).to(dev) if m else None
            ws = torch.empty(max(1, _lib.load().mub_dsb_cross_workspace_bytes(n, P, m)), dtype=torch.uint8,
                             device=dev)
            S = q + q * q + P + q * P
            sums = torch.empty(S, dtype=torch.float64, device=dev)
            call("mub_dsb_cross_" + sfx, ptr(y), n, P, ptr(bg), ptr(ctrl), m, ptr(ws), ptr(sums), stream_ptr())
            s = sums.cpu().numpy()
            sz, szz = s[:q], s[q:q + q * q].reshape(q, q)
            sy, szy = s[q + q * q:q + q * q + P], s[q + q * q + P:].reshape(q, P)
            zbar = sz / n
            C = szz - n * np.outer(zbar, zbar)
            w = np.ones(1) if q == 1 else np.linalg.eigh(C)[1][:, -1]
            b = float(zbar @ w)
            beta = (w @ szy - b * sy) / (w @ C @ w)
            w_d = torch.from_numpy(np.ascontiguousarray(w)).to(dev)
            beta_d = torch.from_numpy(beta).to(dev)
            call("mub_dsb_apply_" + sfx, ptr(y), n, P, ptr(bg), ptr(ctrl), m, ptr(w_d), b, ptr(beta_d), 0.0, 0.0,
                 0, stream_ptr())

    if quantile_clip is not None:
        with phase("dsb_clip"):
            srt = torch.sort(y.reshape(-1)).values
            N = srt.numel()
            if N and torch.isnan(srt[-1]).item():
                y.fill_(float("nan"))
            else:
                qv = _quantiles_linear(N, quantile_clip, lambda k: srt[k].item(), out_dt)
                del srt
                call("mub_dsb_apply_" + sfx, ptr(y), n, P, None, None, 0, None, 0.0, None,
                     float(qv.min()), float(qv.max()), _lib.DSB_CLIP, stream_ptr())
    with phase("dsb_download"):
        y = y.cpu().numpy()
    return y, info
