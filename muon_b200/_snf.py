"""``mu.tl.snf`` -- similarity network fusion (Wang et al. 2014) of the per-modality neighbour graphs on the GPU.

The reference (muon/_core/tools.py:716-920) turns each modality's distances into an affinity matrix, normalises it,
keeps the top ``n_neighbors`` of each column ("dominate set" S_j) and then diffuses: every iteration replaces each
modality's W_j by the normalised S_j P_j S_j^T, P_j the mean of the other modalities' W, as two dense float64
``np.dot``s of N x N matrices.  The fused graph is the normalised mean of the W_j; its rows give the two outputs.

Here every N x N state lives on the device in float64 (csrc/snf.cu).  S_j has ``n_neighbors`` entries per column, so
each product is a sparse x dense product of O(N^2 k) work: R^T = (S_j P_j)^T, then the upper triangle of S_j R^T,
mirrored so that the new state is bit-symmetric.  The normalisation is never a pass of its own: a state is its raw
product plus its row sums, and every reader applies the normalisation on load.  No float atomics: two calls give
the same bits.

Semantics (DESIGN.md section 8):
  * Dense ``ndarray`` distances follow the reference's arithmetic step by step: (D + D^T) / 2 with a zero diagonal,
    the finite mean of sorted positions 1..k per row, the normal pdf as scipy writes it (exp(-y^2/2) / sqrt(2 pi) /
    scale), ``_normalize``, ``_dominateset`` with its broadcasting quirk (entry [i, j] is divided by row sum j), the
    diffusion with S_j fixed across iterations, the mean, the final ``_normalize`` and the two row selections over
    the non-zero entries.
  * Sparse distances (what ``sc.pp.neighbors`` stores) cannot run in the reference (``todense`` gives an
    ``np.matrix`` that current numpy refuses).  Here they are symmetrised and cleaned as scipy does ((D + D^T) / 2,
    ``setdiag(0)``, ``eliminate_zeros()``: an edge stored one way becomes d / 2); every unstored off-diagonal entry
    is then +inf, with affinity 0.
  * Kept quirks: ``connectivities`` holds the ``n_neighbors`` *smallest* non-zero fused affinities of each row, and
    ``distances`` the smallest non-zero 0.5 - w; ``n_neighbors >= n_obs`` raises ValueError.
  * Divergences: a ``neighbor_keys`` dict uses only the modalities it names; fewer than two modalities, or
    modalities with different ``n_obs``, raise ValueError; every top-k selection breaks ties by ascending column.
  * Refused with NotImplementedError before any device work: ``n_neighbors`` above 255, more than 16 modalities,
    and a state that does not fit in free device memory ((2M + 1) N^2 doubles, one more for M > 2).
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._containers import is_mudata
from ._lib import (SNF_DIFFUSE_SYMMETRIC, SNF_DIFFUSE_TRANSPOSED, SNF_MAX_CELLS, SNF_MAX_MODALITIES,
                   SNF_MAX_NEIGHBORS, SNF_SELECT_CONN, SNF_SELECT_DIST, SNF_SELECT_LARGEST, SNF_SELECT_SMALLEST)


def state_bytes(n: int, n_mod: int, n_neighbors: int) -> int:
    """Device bytes of one fusion: M current and M next states, the intermediate product, P when M > 2, and the
    O(N k) selections and row sums."""
    dense = (2 * n_mod + 1 + (1 if n_mod > 2 else 0)) * n * n * 8
    return dense + n * (n_neighbors + 1) * 12 * (n_mod + 2) + 16 * n * (2 * n_mod + 4)


def free_device_bytes() -> int:
    """Free device memory plus what torch's allocator holds unused."""
    import torch
    free, _ = torch.cuda.mem_get_info()
    return int(free + torch.cuda.memory_reserved() - torch.cuda.memory_allocated())


def check_limits(n: int, n_mod: int, n_neighbors: int) -> None:
    """Every refusal that does not need the device's answer, then the memory refusal; all before device work."""
    if n_mod < 2:
        raise ValueError(f"SNF fuses at least two modalities, got {n_mod}")
    if n_mod > SNF_MAX_MODALITIES:
        raise NotImplementedError(f"SNF of {n_mod} modalities: at most {SNF_MAX_MODALITIES} are supported")
    if n_neighbors < 1:
        raise ValueError("'n_neighbors' must be at least 1")
    if n_neighbors >= n:
        raise ValueError("'n_neighbors' seems to be too high.")
    if n_neighbors > SNF_MAX_NEIGHBORS:
        raise NotImplementedError(f"n_neighbors = {n_neighbors} > {SNF_MAX_NEIGHBORS} is not supported by the CUDA "
                                  "row selection")
    if n > SNF_MAX_CELLS:
        raise NotImplementedError(f"SNF of {n} cells: at most {SNF_MAX_CELLS} are supported")
    need = state_bytes(n, n_mod, n_neighbors)
    free = free_device_bytes()
    if need > free:
        raise NotImplementedError(f"SNF of {n} cells and {n_mod} modalities needs {need / 2**30:.1f} GiB of device "
                                  f"memory for its dense float64 state; {free / 2**30:.1f} GiB are free")


def _upload_distances(dist, out) -> None:
    """Write the symmetrised distance matrix (diagonal 0; unstored sparse entries +inf) into the device buffer out."""
    import scipy.sparse as sp
    import torch

    from ._lib import call, ptr, stream_ptr
    n = out.shape[0]
    if sp.issparse(dist):
        D = sp.csr_matrix(dist, dtype=np.float64)
        D = sp.csr_matrix((D + D.T) / 2)
        D.setdiag(0)
        D.eliminate_zeros()
        D.sum_duplicates()
        D.sort_indices()
        dev = out.device
        indptr = torch.from_numpy(D.indptr.astype(np.int64)).to(dev)
        indices = torch.from_numpy(D.indices.astype(np.int32)).to(dev)
        data = torch.from_numpy(D.data.astype(np.float64)).to(dev)
        call("mub_snf_densify_f64", ptr(indptr), ptr(indices), ptr(data), n, ptr(out), stream_ptr())
    else:
        out.copy_(torch.from_numpy(np.ascontiguousarray(np.asarray(dist), dtype=np.float64)))
        call("mub_snf_symmetrise_f64", ptr(out), n, stream_ptr())


def _average(xs, rs, div, out) -> None:
    from ._lib import call, ptr, stream_ptr
    m = len(xs)
    xa = (C.c_void_p * m)(*[ptr(x) for x in xs])
    ra = (C.c_void_p * m)(*[ptr(r) for r in rs])
    call("mub_snf_average_f64", xa, ra, m, float(div), out.shape[0], ptr(out), stream_ptr())


def _select(X, r, k, mode, count=False):
    import torch

    from ._lib import call, ptr, stream_ptr
    n = X.shape[0]
    idx = torch.empty((n, k), dtype=torch.int32, device=X.device)
    val = torch.empty((n, k), dtype=torch.float64, device=X.device)
    cnt = torch.empty(n, dtype=torch.int32, device=X.device) if count else None
    call("mub_snf_select_f64", ptr(X), ptr(r), n, k, mode, ptr(idx), ptr(val), ptr(cnt), stream_ptr())
    return idx, val, cnt


def _rowsum(X, r) -> None:
    from ._lib import call, ptr, stream_ptr
    call("mub_snf_rowsum_f64", ptr(X), X.shape[0], ptr(r), stream_ptr())


def _dominate_set(W, r, k):
    """S of ``_dominateset(nv(W), k)`` as a CSR (ptr, col, val) on the device.  nv(W) is bit-symmetric, so the top
    k of column c is the top k of row c: T = per-row top k, S[i, c] = T[c, i] / (sum over row i of T^T)[c]."""
    import torch

    from ._lib import call, ptr, stream_ptr
    n = W.shape[0]
    tidx, tval, _ = _select(W, r, k, SNF_SELECT_LARGEST)
    rows = tidx.reshape(-1).to(torch.int64)                         # i: T[c, i] is stored in row c
    cols = torch.arange(n, device=W.device, dtype=torch.int64).repeat_interleave(k)
    order = torch.sort(rows * n + cols).indices                     # unique keys: the order is fixed
    sptr = torch.zeros(n + 1, dtype=torch.int64, device=W.device)
    sptr[1:] = torch.cumsum(torch.bincount(rows, minlength=n), 0)
    scol = cols[order].to(torch.int32).contiguous()
    tv = tval.reshape(-1)[order].contiguous()
    cs = torch.empty(n, dtype=torch.float64, device=W.device)
    sval = torch.empty_like(tv)
    call("mub_snf_dominate_f64", ptr(sptr), ptr(scol), ptr(tv), n, ptr(cs), ptr(sval), stream_ptr())
    return sptr, scol, sval


def _diffuse(S, B, rB, out, mode) -> None:
    from ._lib import call, ptr, stream_ptr
    call("mub_snf_diffuse_f64", ptr(S[0]), ptr(S[1]), ptr(S[2]), B.shape[0], ptr(B), ptr(rB), ptr(out), mode,
         stream_ptr())


def fuse(distances, n_neighbors=20, n_iterations=20, sigma=0.5, eps=np.finfo(np.float64).eps, *,
         return_dense=False, return_modalities=False, timings=None):
    """SNF of the per-modality distance matrices (dense ndarrays or scipy sparse, all N x N).

    Returns a dict with ``distances`` and ``connectivities`` (scipy ``csr_array``, ``n_neighbors`` entries per row in
    ascending value order), and, when asked, ``w`` (the normalised fused matrix) and ``modalities`` (the normalised
    W_j after the last iteration) as float64 device tensors.  ``timings``, a list, receives one (start, end) CUDA event pair
    per diffusion iteration."""
    import scipy.sparse as sp
    import torch

    from . import _device
    from ._lib import call, ptr, stream_ptr
    n_mod = len(distances)
    n = int(distances[0].shape[0])
    for d in distances:
        if tuple(d.shape) != (n, n):
            raise ValueError(f"every modality must hold an {n} x {n} distance matrix, got {tuple(d.shape)}")
    k = int(n_neighbors)
    check_limits(n, n_mod, k)
    _device.require_cuda()
    dev = torch.device("cuda", torch.cuda.current_device())
    cur = [torch.empty((n, n), dtype=torch.float64, device=dev) for _ in range(n_mod)]
    nxt = [torch.empty((n, n), dtype=torch.float64, device=dev) for _ in range(n_mod)]
    R = torch.empty((n, n), dtype=torch.float64, device=dev)
    P = torch.empty((n, n), dtype=torch.float64, device=dev) if n_mod > 2 else None
    r_cur = [torch.empty(n, dtype=torch.float64, device=dev) for _ in range(n_mod)]
    r_nxt = [torch.empty(n, dtype=torch.float64, device=dev) for _ in range(n_mod)]
    means = torch.empty(n, dtype=torch.float64, device=dev)

    # affinity matrices, normalised (as raw state + row sums)
    for m, dist in enumerate(distances):
        _upload_distances(dist, cur[m])
        _, sel, _ = _select(cur[m], None, k + 1, SNF_SELECT_SMALLEST)
        call("mub_snf_affinity_f64", ptr(cur[m]), n, ptr(sel), k, float(sigma), float(eps), ptr(means), stream_ptr())
        del sel
        _rowsum(cur[m], r_cur[m])
    S = [_dominate_set(cur[m], r_cur[m], k) for m in range(n_mod)]

    for _ in range(int(n_iterations)):
        if timings is not None:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
        for j in range(n_mod):
            others = [q for q in range(n_mod) if q != j]
            if n_mod == 2:
                B, rB = cur[others[0]], r_cur[others[0]]
            else:
                _average([cur[q] for q in others], [r_cur[q] for q in others], n_mod - 1, P)
                B, rB = P, None
            _diffuse(S[j], B, rB, R, SNF_DIFFUSE_TRANSPOSED)
            _diffuse(S[j], R, None, nxt[j], SNF_DIFFUSE_SYMMETRIC)
            _rowsum(nxt[j], r_nxt[j])
        cur, nxt = nxt, cur
        r_cur, r_nxt = r_nxt, r_cur
        if timings is not None:
            e1.record()
            timings.append((e0, e1))

    # fused matrix: the mean of the normalised states, normalised again
    w, rw = nxt[0], r_nxt[0]
    _average(cur, r_cur, n_mod, w)
    _rowsum(w, rw)
    didx, dval, dcnt = _select(w, rw, k, SNF_SELECT_DIST, count=True)
    cidx, cval, ccnt = _select(w, rw, k, SNF_SELECT_CONN, count=True)
    short = int(torch.minimum(dcnt.min(), ccnt.min()).item())
    if short < k:
        raise ValueError(f"a row of the fused matrix has only {short} non-zero entries, fewer than "
                         f"n_neighbors = {k}")
    indptr = np.arange(0, n * k + 1, k, dtype=np.int64)

    def csr(idx, val):
        return sp.csr_array((val.reshape(-1).cpu().numpy(), idx.reshape(-1).cpu().numpy(), indptr), shape=(n, n))

    out = {"distances": csr(didx, dval), "connectivities": csr(cidx, cval)}
    if return_dense:
        _average([w], [rw], 1, w)
        out["w"] = w
    if return_modalities:
        mods = []
        for m in range(n_mod):
            _average([cur[m]], [r_cur[m]], 1, cur[m])
            mods.append(cur[m])
        out["modalities"] = mods
    return out


def _modality_keys(mdata, neighbor_keys):
    """(modalities, neighbor_keys dict) as the reference resolves them, except that a dict selects its modalities
    for every later step too."""
    if neighbor_keys is None:
        return list(mdata.mod.keys()), {}
    if isinstance(neighbor_keys, str):
        mods = list(mdata.mod.keys())
        return mods, {m: neighbor_keys for m in mods}
    mods = list(neighbor_keys.keys())
    for m in mods:
        if m not in mdata.mod:
            raise ValueError(f"neighbor_keys names modality {m!r}, which the MuData does not hold")
    return mods, dict(neighbor_keys)


def snf(
    mdata,
    n_neighbors: int = 20,
    neighbor_keys=None,
    key_added=None,
    n_iterations: int = 20,
    sigma: float = 0.5,
    eps: float = np.finfo(np.float64).eps,
    copy: bool = False,
):
    """Similarity network fusion (Wang et al. 2014) of the modalities' neighbour graphs -- ``muon.tl.snf``
    (muon/_core/tools.py:716-920), the same arguments and slots: ``obsp[conns_key]``, ``obsp[dists_key]`` (float64
    ``csr_array``, ``n_neighbors`` entries per row in ascending value order) and ``uns[key_added]``.

    Each modality's distances are ``mod.obsp[mod.uns[key]["distances_key"]]``, ``key`` from ``neighbor_keys``
    ("neighbors" by default).  Dense distances follow the reference's arithmetic; sparse ones count every unstored
    pair as infinitely far (affinity 0).  ``connectivities`` are the ``n_neighbors`` smallest non-zero fused
    affinities of each row, as in the reference.  A ``neighbor_keys`` dict fuses only the modalities it names; fewer
    than two modalities or different ``n_obs`` raise ValueError; ties in every top-k selection go to the lower
    column.  ``n_neighbors`` above 255, more than 16 modalities and a dense state of (2M + 1) N^2 doubles (one more
    for M > 2) beyond free device memory raise NotImplementedError.  All arithmetic is float64 on the GPU, and two
    calls return the same bits.
    """
    if not is_mudata(mdata):
        raise TypeError("Expected a MuData object")
    modalities, nkeys = _modality_keys(mdata, neighbor_keys)
    mod_reps, mod_n_pcs, dists = {}, {}, []
    for mod in modalities:
        nkey = nkeys.get(mod, "neighbors")
        try:
            nparams = mdata.mod[mod].uns[nkey]
        except KeyError:
            raise ValueError(
                f'Did not find .uns["{nkey}"] for modality "{mod}". Run `sc.pp.neighbors` on all modalities first.')
        use_rep = nparams["params"].get("use_rep", None)
        n_pcs = nparams["params"].get("n_pcs", None)
        mod_reps[mod] = use_rep if use_rep is not None else -1
        mod_n_pcs[mod] = n_pcs if n_pcs is not None else -1
        dists.append(mdata.mod[mod].obsp[nparams["distances_key"]])
    if len(modalities) < 2:
        raise ValueError(f"SNF fuses at least two modalities, got {len(modalities)}")
    n_obs = {mod: mdata.mod[mod].n_obs for mod in modalities}
    if len(set(n_obs.values())) != 1:
        raise ValueError(f"SNF needs modalities with the same observations, got n_obs {n_obs}")
    res = fuse(dists, n_neighbors=n_neighbors, n_iterations=n_iterations, sigma=sigma, eps=eps)

    mdata = mdata.copy() if copy else mdata
    if key_added is None:
        key_added = "neighbors"
        conns_key = "connectivities"
        dists_key = "distances"
    else:
        conns_key = key_added + "_connectivities"
        dists_key = key_added + "_distances"
    neighbors_dict = {"connectivities_key": conns_key, "distances_key": dists_key}
    neighbors_dict["params"] = {
        "n_neighbors": n_neighbors,
        "eps": eps,
        "use_rep": mod_reps,
        "n_pcs": mod_n_pcs,
        "method": "snf",
    }
    mdata.obsp[conns_key] = res["connectivities"]
    mdata.obsp[dists_key] = res["distances"]
    mdata.uns[key_added] = neighbors_dict
    return mdata if copy else None
