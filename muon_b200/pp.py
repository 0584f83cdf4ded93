"""``mu.pp`` -- multimodal preprocessing.  ``neighbors`` (WNN) is the first "next" row of the coverage contract
(SURVEY section 8f-f1, BASELINE configs[4]); status: first correct GPU path, exact instead of approximate search.
"""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np

from ._containers import is_mudata


def _choose_representation(adata, use_rep=None, n_pcs=None):
    """scanpy.tools._utils._choose_representation for what muon passes (preproc.py:378)."""
    if use_rep is None or use_rep == "X":
        if use_rep is None and adata.n_vars > 50:
            if "X_pca" in adata.obsm:
                X = adata.obsm["X_pca"]
                return X[:, :n_pcs] if n_pcs else X
            # scanpy would compute a PCA here (n_vars > 50 and no X_pca); silently searching in the raw X instead
            # would give a different graph, so ask for the representation explicitly
            raise ValueError("use_rep is None, the modality has more than 50 variables and no .obsm['X_pca']: scanpy would "
                             "compute a PCA at this point; run it first or set use_rep in the modality's neighbors call")
        return adata.X
    if use_rep in adata.obsm:
        X = adata.obsm[use_rep]
        return X[:, :n_pcs] if n_pcs else X
    raise ValueError(f"Did not find {use_rep} in `.obsm.keys()`.")


def _umap_connectivities(knn_idx, knn_dist, n_obs):
    """UMAP fuzzy simplicial set on a precomputed kNN table (what scanpy's ``umap`` connectivities wrapper
    returns to preproc.py:607-614): smooth-kNN bandwidths by bisection (64 steps, local_connectivity=1),
    membership strengths exp(-(d - rho)/sigma), fuzzy union A + A^T - A.A^T.  Vectorised over cells on the device."""
    import scipy.sparse as sp
    import torch
    d = knn_dist.to(torch.float32)
    n, k = d.shape
    target = float(np.log2(k))
    big = torch.finfo(torch.float32).max
    pos = torch.where(d > 0, d, torch.full_like(d, big))
    rho = pos.min(dim=1).values
    rho = torch.where(rho == big, torch.zeros_like(rho), rho)          # no positive distance: rho = 0
    lo = torch.zeros(n, dtype=torch.float64, device=d.device)
    hi = torch.full((n,), float("inf"), dtype=torch.float64, device=d.device)
    mid = torch.ones(n, dtype=torch.float64, device=d.device)
    done = torch.zeros(n, dtype=torch.bool, device=d.device)
    dd = (d[:, 1:] - rho[:, None]).to(torch.float64)                   # the first column is skipped (umap: j from 1)
    for _ in range(64):
        psum = torch.where(dd > 0, torch.exp(-dd / mid[:, None]), torch.ones_like(dd)).sum(1)
        done |= (psum - target).abs() < 1e-5
        gt = psum > target
        new_hi = torch.where(gt, mid, hi)
        new_lo = torch.where(gt, lo, mid)
        new_mid = torch.where(gt, (lo + mid) / 2.0,
                              torch.where(torch.isinf(hi), mid * 2.0, (mid + hi) / 2.0))
        hi = torch.where(done, hi, new_hi)
        lo = torch.where(done, lo, new_lo)
        mid = torch.where(done, mid, new_mid)
    sigma = mid.to(torch.float32)
    mean_row = d.mean(dim=1)
    mean_all = d.mean()
    floor = torch.where(rho > 0, 1e-3 * mean_row, 1e-3 * mean_all.expand_as(mean_row))
    sigma = torch.maximum(sigma, floor)
    rows = torch.arange(n, device=d.device)[:, None].expand(n, k)
    val = torch.where((d - rho[:, None] <= 0) | (sigma[:, None] == 0), torch.ones_like(d),
                      torch.exp(-(d - rho[:, None]) / sigma[:, None]))
    val = torch.where(knn_idx == rows, torch.zeros_like(val), val)
    val = torch.where(knn_idx < 0, torch.zeros_like(val), val)
    # fuzzy union A + A^T - A.A^T on the device: the entries of A and of A^T keyed by (row, column), sorted; a key
    # occurs once (one-sided edge: value a) or twice (mutual edge: a + b - a*b, the same float32 operations in the
    # same order as scipy's (A + A.T) - A.multiply(A.T))
    r = rows.reshape(-1).to(torch.int64)
    c = knn_idx.clamp_min(0).reshape(-1).to(torch.int64)
    v = val.reshape(-1)
    keep = v != 0
    r, c, v = r[keep], c[keep], v[keep]
    keys = torch.cat([r * n_obs + c, c * n_obs + r])
    vals = torch.cat([v, v])
    keys, order = torch.sort(keys, stable=True)
    vals = vals[order]
    first = torch.ones(keys.numel(), dtype=torch.bool, device=keys.device)
    first[1:] = keys[1:] != keys[:-1]
    second = ~first
    pos = torch.nonzero(first).reshape(-1)
    a = vals[pos]
    out_val = a.clone()
    has_pair = torch.zeros(pos.numel(), dtype=torch.bool, device=keys.device)
    seg_of_second = torch.cumsum(first.to(torch.int64), 0)[second] - 1
    has_pair[seg_of_second] = True
    b = torch.zeros_like(a)
    b[seg_of_second] = vals[second]
    out_val = torch.where(has_pair, (a + b) - a * b, a)
    out_key = keys[pos]
    nz = out_val != 0
    out_key, out_val = out_key[nz], out_val[nz]
    out_rows = torch.div(out_key, n_obs, rounding_mode="floor")
    out_cols = (out_key - out_rows * n_obs).to(torch.int32)
    indptr = torch.zeros(n_obs + 1, dtype=torch.int64, device=keys.device)
    indptr[1:] = torch.cumsum(torch.bincount(out_rows, minlength=n_obs), 0)
    out = sp.csr_matrix((n_obs, n_obs), dtype=np.float32)
    idt = np.int32 if int(indptr[-1]) < 2**31 - 1 else np.int64
    out.data, out.indices, out.indptr = out_val.cpu().numpy(), out_cols.cpu().numpy().astype(idt, copy=False), \
        indptr.cpu().numpy().astype(idt, copy=False)
    out.has_sorted_indices = True
    return out


def neighbors(
    mdata,
    n_neighbors: Optional[int] = None,
    n_bandwidth_neighbors: int = 20,
    n_multineighbors: int = 200,
    neighbor_keys: Optional[Dict[str, Optional[str]]] = None,
    metric: str = "euclidean",
    low_memory: Optional[bool] = None,
    key_added: Optional[str] = None,
    weight_key: Optional[str] = "mod_weight",
    add_weights_to_modalities: bool = False,
    eps: float = 1e-4,
    copy: bool = False,
    random_state=42,
):
    """Multimodal (weighted) nearest-neighbour search -- ``muon.pp.neighbors`` (reference
    muon/_core/preproc.py:264-640), same arguments and slots: ``obsp[distances/connectivities]``,
    ``uns[key]``, per-modality cell weights in ``obs["<mod>:mod_weight"]``.

    Differences, all deliberate: every nearest-neighbour search is **exact** (brute force on the GPU) where the
    reference runs NN-descent, so ``random_state`` has no effect and ``low_memory`` only bounds the search workspace
    (queries run in blocks of 131 072 cells); only the Euclidean metric is supported; sparse representations are
    densified (same distances); all modalities must hold the same observations in the same order.
    """
    import scipy.sparse as sp
    import torch

    from . import _device
    from ._lib import call, ptr, stream_ptr

    if not is_mudata(mdata):
        raise TypeError("Expected a MuData object")
    mdata = mdata.copy() if copy else mdata
    if neighbor_keys is None:
        modalities = list(mdata.mod.keys())
        neighbor_keys = {}
    else:
        modalities = list(neighbor_keys.keys())
    if metric != "euclidean":
        raise NotImplementedError("only metric='euclidean' is supported by the CUDA path yet")

    params, reps, mod_reps, mod_n_pcs, mod_k = {}, {}, {}, {}, []
    for mod in modalities:
        nkey = neighbor_keys.get(mod, "neighbors")
        try:
            nparams = mdata.mod[mod].uns[nkey]
        except KeyError:
            raise ValueError(f'Did not find .uns["{nkey}"] for modality "{mod}". Run `sc.pp.neighbors` on all '
                             "modalities first.")
        use_rep = nparams["params"].get("use_rep", None)
        n_pcs = nparams["params"].get("n_pcs", None)
        mod_k.append(nparams["params"].get("n_neighbors", 0))
        if nparams["params"].get("metric", "euclidean") != "euclidean" or nparams.get("metric", "euclidean") != "euclidean":
            raise NotImplementedError("only Euclidean per-modality neighbour graphs are supported yet")
        params[mod] = nparams
        R = _choose_representation(mdata.mod[mod], use_rep, n_pcs)
        if sp.issparse(R):
            # sparse representation (reference: _jaccard_sparse_euclidean_metric / _sparse_csr_ptp, preproc.py:79-159,
            # 425-447): Euclidean distances between sparse rows equal those between the densified rows, and the
            # exact search needs the rows dense anyway -- densify if it fits, say so if it does not
            if R.shape[0] * R.shape[1] * 4 > (8 << 30):
                raise NotImplementedError(f"modality '{mod}': a sparse representation of shape {R.shape} does not fit the dense "
                                          "exact search (8 GiB limit); reduce it first (PCA / LSI) and set use_rep")
            R = R.toarray()
        reps[mod] = np.ascontiguousarray(np.asarray(R), dtype=np.float32)
        mod_reps[mod] = use_rep if use_rep is not None else -1
        mod_n_pcs[mod] = n_pcs if n_pcs is not None else -1
    if n_neighbors is None:
        ks = np.asarray([k for k in mod_k if k > 0])
        n_neighbors = int(round(float(np.mean(ks)), 0))

    obs = np.asarray(mdata.obs_names).astype(str)
    for mod in modalities:
        if not np.array_equal(np.asarray(mdata.mod[mod].obs_names).astype(str), obs):
            raise NotImplementedError("modalities with different observations are not supported by the CUDA path yet")
    N, M = len(obs), len(modalities)
    if M > 4:
        raise NotImplementedError("more than 4 modalities")
    # limits of the per-cell candidate tables (csrc/wnn.cu kWnnMaxCand) and of the exact kNN kernels, checked up
    # front instead of failing data-dependently in the middle of the call
    if M * n_multineighbors > 1536:
        raise NotImplementedError(f"n_multineighbors * modalities = {M * n_multineighbors} > 1536 candidates per cell is not "
                                  "supported by the CUDA path yet")
    if n_multineighbors + 1 > 320:
        raise NotImplementedError("n_multineighbors > 319 is not supported by the CUDA path yet (exact kNN kernels: k <= 320)")

    _device.require_cuda()
    dev = torch.device("cuda", torch.cuda.current_device())
    st = stream_ptr()
    Xd, Gd, nnd, sig = {}, {}, {}, {}
    for mod in modalities:
        G = sp.csr_matrix(mdata.mod[mod].obsp[params[mod]["distances_key"]])
        deg = np.diff(G.indptr)
        if np.any(deg == 0):
            i = int(np.where(deg == 0)[0][0])
            raise ValueError(f"Cell {i} in modality {mod} does not have any neighbors. This could be due to subsetting "
                             "after nearest neighbors calculation. Make sure to subset before calculating nearest neighbors.")
        nnd[mod] = torch.from_numpy(np.minimum.reduceat(G.data.astype(np.float64), G.indptr[:-1])).to(dev)
        Gd[mod] = _device.DeviceCSR.from_scipy(G, dtype=np.float32)
        Xd[mod] = torch.from_numpy(reps[mod]).to(dev)

    # ---- kernel bandwidths sigma (preproc.py:408-470) ----------------------------------------------------------
    for mod in modalities:
        X = Xd[mod]
        bbox = float(np.linalg.norm(np.ptp(reps[mod].astype(np.float64), axis=0), ord=2))
        Gt = _device.csr_transpose(Gd[mod])
        s = torch.empty(N, dtype=torch.float64, device=dev)
        status = torch.zeros(1, dtype=torch.int32, device=dev)
        call("mub_wnn_bandwidth_f32", ptr(Gd[mod].indptr), ptr(Gd[mod].indices), ptr(Gt.indptr), ptr(Gt.indices),
             ptr(X), N, X.shape[1], X.shape[1], n_bandwidth_neighbors, bbox, ptr(s), ptr(status), None, 0, None, 0, 0, st)
        if int(status[0]) & 1:
            # hub cells (sharing neighbours with > 1536 cells): redo them with big hash tables in global memory
            from ._lib import load
            hubs = torch.nonzero(s < 0).reshape(-1).contiguous()
            slots, tables = 1 << 18, 64
            ws = torch.empty(int(load().mub_wnn_bandwidth_workspace_bytes(slots, tables)), dtype=torch.uint8, device=dev)
            status.zero_()
            call("mub_wnn_bandwidth_f32", ptr(Gd[mod].indptr), ptr(Gd[mod].indices), ptr(Gt.indptr), ptr(Gt.indices),
                 ptr(X), N, X.shape[1], X.shape[1], n_bandwidth_neighbors, bbox, ptr(s), ptr(status), ptr(hubs),
                 hubs.numel(), ptr(ws), slots, tables, st)
            if int(status[0]) & 2:
                raise RuntimeError("neighbors: a cell shares kNN neighbours with more than 131072 cells")
        sig[mod] = s

    # ---- modality weights (preproc.py:472-508) -----------------------------------------------------------------
    ratios = torch.full((N, M), float("-inf"), dtype=torch.float64, device=dev)
    for i1, m1 in enumerate(modalities):
        X = Xd[m1]
        d = X.shape[1]
        P = _device.pad_width(d)
        Xp = torch.zeros((N, P), dtype=torch.float32, device=dev)
        Xp[:, :d] = X
        cur, others = None, []
        for i2, m2 in enumerate(modalities):
            G2 = Gd[m2]
            # mean over the stored neighbours with a NON-ZERO distance (the reference takes graph.nonzero(),
            # preproc.py:480-483, which skips explicitly stored zeros such as duplicate cells)
            lens = G2.indptr[1:] - G2.indptr[:-1]
            nz = (G2.data != 0).to(torch.float32)
            rowid = torch.repeat_interleave(torch.arange(N, device=dev), lens)
            deg = torch.zeros(N, dtype=torch.float32, device=dev).index_add_(0, rowid, nz)
            mean_graph = G2.with_data(nz / deg.clamp_min(1.0)[rowid])
            r = _device.spmm(mean_graph, Xp, dynamic=False)[:, :d]       # mean of X over the cell's neighbours in m2
            dist = (X.to(torch.float64) - r.to(torch.float64)).norm(dim=1)
            theta = torch.exp(-torch.clamp(dist - nnd[m1], min=0) / (sig[m1] - nnd[m1]))
            if i1 == i2:
                cur = theta
            else:
                others.append(theta)
        best_other = torch.stack(others, 1).max(dim=1).values if others else torch.full_like(cur, float("-inf"))
        ratios[:, i1] = cur / (best_other + eps)
    weights = torch.softmax(ratios, dim=1).contiguous()

    # ---- candidates: n_multineighbors exact neighbours per modality (preproc.py:509-567) ----------------------
    # low_memory (reference: NN-descent's memory mode, default on above 50 000 cells, preproc.py:356-359,517): here it
    # bounds the per-query workspace of the exact search by running the queries in blocks
    lmem = low_memory if low_memory is not None else N > 50000
    cands = []
    for mod in modalities:
        idx, _ = _device.knn_l2(Xd[mod], min(n_multineighbors + 1, N), query_chunk=131072 if lmem else None)
        cands.append(idx[:, 1:].contiguous())                            # drop the cell itself (preproc.py:531)
    n_cand = cands[0].shape[1]

    # ---- weighted affinities over the union of candidates, top n_neighbors+1 (preproc.py:569-604) --------------
    import ctypes as C
    n_out = n_neighbors + 1
    out_idx = torch.empty((N, n_out), dtype=torch.int32, device=dev)
    out_dist = torch.empty((N, n_out), dtype=torch.float64, device=dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    arr_p = (C.c_void_p * M)
    reps_p = arr_p(*[Xd[m].data_ptr() for m in modalities])
    cands_p = arr_p(*[c.data_ptr() for c in cands])
    sig_p = arr_p(*[sig[m].data_ptr() for m in modalities])
    dims_p = (C.c_int32 * M)(*[Xd[m].shape[1] for m in modalities])
    call("mub_wnn_affinity_topk_f32", M, reps_p, dims_p, dims_p, cands_p, sig_p, ptr(weights), N, n_cand, n_out,
         ptr(out_idx), ptr(out_dist), ptr(status), st)
    if int(status[0]) != 0:
        raise RuntimeError("neighbors: candidate union overflow")
    if bool((out_idx < 0).any()):
        raise ValueError("neighbors: fewer candidates than n_neighbors + 1; increase n_multineighbors")

    indptr = np.arange(0, (N + 1) * n_out, n_out)
    distances = sp.csr_matrix((out_dist.cpu().numpy().ravel(), out_idx.cpu().numpy().ravel().astype(np.int64), indptr),
                              shape=(N, N))
    connectivities = _umap_connectivities(out_idx.to(torch.int64), out_dist, N)

    if key_added is None:
        key_added, conns_key, dists_key = "neighbors", "connectivities", "distances"
    else:
        conns_key, dists_key = f"{key_added}_connectivities", f"{key_added}_distances"
    W = weights.cpu().numpy()
    for i, m in enumerate(modalities):
        if weight_key:
            if add_weights_to_modalities:
                mdata.mod[m].obs[weight_key] = W[:, i]
            else:
                mdata.obs[":".join([m, weight_key])] = W[:, i]
    mdata.obsp[dists_key] = distances
    mdata.obsp[conns_key] = connectivities
    mdata.uns[key_added] = {
        "connectivities_key": conns_key, "distances_key": dists_key,
        "params": {"n_neighbors": n_neighbors, "n_multineighbors": n_multineighbors, "metric": metric, "eps": eps,
                   "random_state": random_state, "use_rep": mod_reps, "n_pcs": mod_n_pcs, "method": "umap"},
    }
    mdata.update_obs()
    return mdata if copy else None
