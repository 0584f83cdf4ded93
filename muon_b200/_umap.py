"""``mu.tl.umap`` -- UMAP layout of the (multimodal) neighbour graph on the GPU.

The reference (muon/_core/tools.py:1209-1362) hands the graph to ``sc.tl.umap``, which runs umap-learn's
``simplicial_set_embedding``: a sequential (seeded) or numba-hogwild SGD of roughly n_epochs x stored edges x
(1 + negative_sample_rate) gradient steps.  Here the host prepares what umap-learn prepares -- curve parameters,
epoch count, pruning, per-entry sampling rates, initial positions, the sampler's seed -- and the epochs run as one
CUDA launch each (csrc/umap.cu): a Jacobi update in which every vertex sums its own terms in a fixed order.

Departures from umap-learn, all deliberate:
  * Jacobi, not sequential: every vertex moves from the positions of the previous epoch.  The result is
    bit-identical from run to run for a given ``random_state`` (no hogwild), but it is not umap-learn's layout
    for the same seed; the two agree in quality (trustworthiness, neighbourhood preservation).
  * The sampling schedule is evaluated in closed form from eps_e = w_max / w_e (exact arithmetic, see umap.cu),
    where umap-learn accumulates fp64 counters; the negative samples come from a counter-based Philox4x32-10
    keyed by the three ints umap-learn draws for its own sampler.
  * Spectral init: the eigenvectors of the normalised adjacency come from the project's block Krylov solver on
    the device (``_lsi.truncated_svd``), not ARPACK.  Graphs with more than 2 * n_components connected
    components would need umap-learn's data-centroid meta layout and are refused.
  * Nothing is imputed into a representation matrix: it only serves that many-component meta layout.
"""
from __future__ import annotations

import numbers

import numpy as np

from ._containers import is_anndata, is_mudata
from ._lib import UMAP_MAX_COMPONENTS

INT32_MIN = np.iinfo(np.int32).min + 1
INT32_MAX = np.iinfo(np.int32).max - 1
SPECTRAL_TOL = 1e-5        # relative residual of the Krylov eigenpairs


# ---- host-side preparation (umap-learn 0.5 simplicial_set_embedding as scanpy calls it) ---------------------
def find_ab_params(spread, min_dist):
    """Fit 1 / (1 + a x^(2b)) to 1 below ``min_dist`` and exp(-(x - min_dist) / spread) above, on [0, 3 spread]."""
    from scipy.optimize import curve_fit

    def curve(x, a, b):
        return 1.0 / (1.0 + a * x ** (2 * b))

    xv = np.linspace(0, spread * 3, 300)
    yv = np.zeros(xv.shape)
    yv[xv < min_dist] = 1.0
    yv[xv >= min_dist] = np.exp(-(xv[xv >= min_dist] - min_dist) / spread)
    params, _ = curve_fit(curve, xv, yv)
    return params[0], params[1]


def check_random_state(seed):
    """sklearn.utils.check_random_state: None -> numpy's global RandomState, int -> a new one, or the instance."""
    if seed is None or seed is np.random:
        return np.random.mtrand._rand
    if isinstance(seed, numbers.Integral):
        return np.random.RandomState(seed)
    if isinstance(seed, np.random.RandomState):
        return seed
    raise ValueError(f"{seed!r} cannot be used to seed a numpy.random.RandomState instance")


def default_epochs(n: int) -> int:
    return 500 if n <= 10000 else 200


def prune(graph, n_epochs: int):
    """The graph as float32 CSR with duplicates summed and the weights below w_max / n_epochs dropped (w_max / the
    default epoch count when n_epochs <= 10), and the number of epochs to run (``n_epochs``, or the default for
    None / 0)."""
    import scipy.sparse as sp
    G = sp.csr_matrix(graph, dtype=np.float32, copy=True)
    G.sum_duplicates()          # canonical CSR: umap's sorted COO entries in the same order
    default = default_epochs(G.shape[0])
    n_epochs = default if not n_epochs else int(n_epochs)
    if G.nnz:
        G.data[G.data < G.data.max() / float(n_epochs if n_epochs > 10 else default)] = 0.0
    G.eliminate_zeros()
    return G, n_epochs


def epochs_per_sample(w: np.ndarray) -> np.ndarray:
    """eps_e = w_max / w_e >= 1 as float32: entry e is sampled once every eps_e epochs."""
    if w.size == 0:
        return np.zeros(0, np.float32)
    return (float(w.max()) / w.astype(np.float64)).astype(np.float32)


def components(G):
    from scipy.sparse.csgraph import connected_components
    return connected_components(G)


def meta_positions(n_comp: int, dim: int) -> np.ndarray:
    """umap's multi_component_layout for n_comp <= 2 dim: +-e_1, +-e_2, ..."""
    k = int(np.ceil(n_comp / 2.0))
    base = np.hstack([np.eye(k), np.zeros((k, dim - k))])
    return np.vstack([base, -base])[:n_comp]


def spectral_layout(G, dim: int, random_state, eigvecs) -> np.ndarray:
    """umap's spectral_layout: the ``dim`` non-trivial eigenvectors of the normalised Laplacian per connected
    component (``eigvecs(W, dim)``), placed around meta positions +-e_i when there are several components.
    Components too small for the eigenproblem get uniform positions from ``random_state``."""
    n_comp, labels = components(G)
    if n_comp == 1:
        return eigvecs(G, dim)
    if n_comp > 2 * dim:
        raise NotImplementedError(
            f"spectral init of a graph with {n_comp} connected components (> 2 * n_components = {2 * dim}) needs "
            "umap-learn's data-centroid meta layout, which is not supported; pass init_pos='random' or an array")
    meta = meta_positions(n_comp, dim)
    out = np.zeros((G.shape[0], dim), dtype=np.float64)
    G = G.tocsr()
    for label in range(n_comp):
        mask = labels == label
        sub = G[mask][:, mask]
        dist = np.linalg.norm(meta - meta[label], axis=1)
        data_range = dist[dist > 0.0].min() / 2.0
        size = sub.shape[0]
        if size < 2 * dim or size <= dim + 1:
            out[mask] = random_state.uniform(low=-data_range, high=data_range, size=(size, dim)) + meta[label]
            continue
        emb = eigvecs(sub, dim)
        out[mask] = emb * (data_range / np.max(np.abs(emb))) + meta[label]
    return out


def initial_positions(G, dim: int, init, random_state, eigvecs) -> np.ndarray:
    """Initial float32 positions, rescaled to [0, 10] per axis, as umap's simplicial_set_embedding builds them."""
    n = G.shape[0]
    if isinstance(init, str) and init == "random":
        Y = random_state.uniform(low=-10.0, high=10.0, size=(n, dim)).astype(np.float32)
    elif isinstance(init, str) and init == "spectral":
        Y = spectral_layout(G, dim, random_state, eigvecs)
        Y = (Y * (10.0 / np.abs(Y).max())).astype(np.float32) + \
            random_state.normal(scale=0.0001, size=[n, dim]).astype(np.float32)
    else:
        Y = np.array(init, dtype=np.float32)
    lo, hi = Y.min(0), Y.max(0)
    return (10.0 * (Y - lo) / (hi - lo)).astype(np.float32, order="C")


def sampler_key(random_state) -> tuple:
    """The three ints umap draws for its sampler, as uint32 words (s0, s1, s2) of the Philox key and counter."""
    s = random_state.randint(INT32_MIN, INT32_MAX, 3).astype(np.int64)
    return tuple(int(v) & 0xFFFFFFFF for v in s)


# ---- device ----------------------------------------------------------------------------------------------
class NormalisedAdjacency:
    """M = I + D^-1/2 W D^-1/2 (symmetric W) as a ``truncated_svd`` operator.  M is PSD with spectrum in [0, 2], so its
    largest singular triplets are its largest eigenpairs, i.e. the smallest eigenpairs of the normalised Laplacian
    I - D^-1/2 W D^-1/2 (eigenvalue 2 - sigma).  M = M^T, so ``aty`` is ``av``."""

    def __init__(self, W):
        import torch

        from . import _device
        self._dev = _device
        deg = np.asarray(W.sum(axis=0), dtype=np.float64).ravel()
        A = _device.DeviceCSR.from_scipy(W.tocsr(), dtype=np.float32)
        dinv = torch.from_numpy(1.0 / np.sqrt(deg)).to(A.device)
        rows = torch.repeat_interleave(torch.arange(A.shape[0], device=A.device), A.indptr[1:] - A.indptr[:-1])
        self.N = A.with_data((A.data.to(torch.float64) * dinv[rows] * dinv[A.indices.to(torch.int64)])
                             .to(torch.float32))
        self.d = self.n_total = A.shape[0]
        self.device = A.device

    def av(self, V):
        return self._dev.spmm(self.N, V, dynamic=False) + V

    aty = av

    def gram(self, Y, l):
        return self._dev.gram(Y, l, reduce=False)


def spectral_eigs(W, k: int):
    """The k smallest eigenvalues (ascending, fp64) and eigenvectors [n x k] of the normalised Laplacian of the
    symmetric graph W, on the device."""
    from . import _device
    from ._lsi import truncated_svd
    _device.require_cuda()
    op = NormalisedAdjacency(W)
    _, s, V, _ = truncated_svd(op, k, pad_to=_device.pad_width(k), tol=SPECTRAL_TOL)
    return 2.0 - s.cpu().numpy(), V.cpu().numpy().astype(np.float64)


def spectral_vectors(W, dim: int) -> np.ndarray:
    return spectral_eigs(W, dim + 1)[1][:, 1:dim + 1]


class Layout:
    """The pruned graph on the device as head entries (CSR rows) and tail entries (its transpose, each row in
    ascending column order so the tail sums run in a fixed order), both carrying eps_e."""

    def __init__(self, G, eps: np.ndarray):
        import scipy.sparse as sp
        import torch

        from . import _device
        _device.require_cuda()
        n = G.shape[0]
        H = sp.csr_matrix((eps, G.indices, G.indptr), shape=G.shape)
        H.has_sorted_indices = True
        self.H = _device.DeviceCSR.from_scipy(H, dtype=np.float32)
        T = _device.csr_transpose(self.H)
        rows = torch.repeat_interleave(torch.arange(n, device=T.device), T.indptr[1:] - T.indptr[:-1])
        order = torch.sort(rows * n + T.indices.to(torch.int64)).indices
        self.T = _device.DeviceCSR(T.indptr, T.indices[order].contiguous(), T.data[order].contiguous(), T.shape)
        self.n = n

    def run(self, Y0, epochs, n_epochs, *, a, b, gamma, alpha, negative_sample_rate, key):
        """Epochs ``epochs`` (a range) of the ``n_epochs``-epoch schedule from positions Y0 [n x dim] float32
        (numpy or device tensor); returns the device tensor of the final positions."""
        import torch

        from ._lib import call, ptr, stream_ptr
        dev = self.H.device
        Y = torch.as_tensor(np.ascontiguousarray(Y0, dtype=np.float32) if isinstance(Y0, np.ndarray) else Y0,
                            dtype=torch.float32, device=dev).contiguous()
        Y, Z = Y.clone(), torch.empty_like(Y)
        dim = Y.shape[1]
        H, T = self.H, self.T
        st = stream_ptr()
        for ep in epochs:
            alpha_n = alpha * (1.0 - float(ep) / float(n_epochs))
            call("mub_umap_epoch_f32", ptr(H.indptr), ptr(H.indices), ptr(H.data), ptr(T.indptr), ptr(T.indices),
                 ptr(T.data), self.n, dim, ptr(Y), ptr(Z), float(a), float(b), float(gamma), alpha_n, int(ep),
                 int(negative_sample_rate), *key, st)
            Y, Z = Z, Y
        return Y


def philox4x32_10(ctr: np.ndarray, k0: int, k1: int) -> np.ndarray:
    """Philox4x32-10 of the uint32 counters ctr [n x 4] under key (k0, k1), on the device (the epoch's generator)."""
    import torch

    from ._lib import call, ptr, stream_ptr
    c = torch.from_numpy(np.ascontiguousarray(ctr, dtype=np.uint32).view(np.int32)).cuda()
    out = torch.empty_like(c)
    call("mub_philox4x32_10", ptr(c), c.shape[0], int(k0), int(k1), ptr(out), stream_ptr())
    return out.cpu().numpy().view(np.uint32)


def embed(graph, *, n_components=2, maxiter=None, alpha=1.0, gamma=1.0, negative_sample_rate=5,
          init_pos="spectral", random_state=42, a=1.0, b=1.0):
    """umap's simplicial_set_embedding of the connectivities ``graph`` -> float32 [n x n_components]."""
    G, n_epochs = prune(graph, 0 if maxiter is None else maxiter)
    rs = check_random_state(random_state)
    Y0 = initial_positions(G, n_components, init_pos, rs, spectral_vectors)
    key = sampler_key(rs)
    lay = Layout(G, epochs_per_sample(G.data))
    Y = lay.run(Y0, range(n_epochs), n_epochs, a=a, b=b, gamma=gamma, alpha=alpha,
                negative_sample_rate=negative_sample_rate, key=key)
    return Y.cpu().numpy()


# ---- public entry point ------------------------------------------------------------------------------------
def umap(
    mdata,
    min_dist: float = 0.5,
    spread: float = 1.0,
    n_components: int = 2,
    maxiter=None,
    alpha: float = 1.0,
    gamma: float = 1.0,
    negative_sample_rate: int = 5,
    init_pos="spectral",
    random_state=42,
    a=None,
    b=None,
    copy: bool = False,
    method: str = "umap",
    neighbors_key=None,
):
    """Embed the (multimodal) neighbour graph with UMAP -- ``muon.tl.umap`` (muon/_core/tools.py:1209-1362), the same
    arguments and slots: ``obsm["X_umap"]`` (n x n_components, float32) and ``uns["umap"]["params"]``.

    MuData and AnnData take the same path: the graph is ``obsp[uns[neighbors_key]["connectivities_key"]]``
    (``neighbors_key`` defaults to "neighbors").  ``method="rapids"`` is accepted and runs this same CUDA layout.
    ``init_pos`` is "spectral", "random", an array of initial positions, or the name of an ``obsm`` entry (scanpy).
    The layout is bit-identical from run to run for a given int ``random_state``; the module docstring lists where
    it departs from umap-learn's.
    """
    import scipy.sparse as sp
    data = mdata
    if not (is_mudata(data) or is_anndata(data)):
        raise TypeError("Expected a MuData or AnnData object")
    if method not in ("umap", "rapids"):
        raise ValueError(f"method must be 'umap' or 'rapids', not {method!r}")
    if neighbors_key is None:
        neighbors_key = "neighbors"
    try:
        neighbors = data.uns[neighbors_key]
    except KeyError:
        raise ValueError(f'Did not find .uns["{neighbors_key}"]. Run `muon.pp.neighbors` first.')
    n_components = int(n_components)
    if n_components < 1:
        raise ValueError("n_components must be at least 1")
    if n_components > UMAP_MAX_COMPONENTS:
        raise NotImplementedError(f"n_components = {n_components} > {UMAP_MAX_COMPONENTS} is not supported by the "
                                  "CUDA layout")
    graph = data.obsp[neighbors.get("connectivities_key", "connectivities")]
    n = graph.shape[0]
    if isinstance(init_pos, str) and init_pos in data.obsm:
        init_pos = np.asarray(data.obsm[init_pos])
    if isinstance(init_pos, str):
        if init_pos == "paga":
            raise NotImplementedError("init_pos='paga' is not supported")
        if init_pos not in ("spectral", "random"):
            raise ValueError(f"init_pos must be 'spectral', 'random', an array or an .obsm key, not {init_pos!r}")
    else:
        init_pos = np.asarray(init_pos, dtype=np.float32)
        if init_pos.shape != (n, n_components):
            raise ValueError(f"init_pos has shape {init_pos.shape}, expected {(n, n_components)}")
    if not sp.issparse(graph):
        graph = sp.csr_matrix(graph)
    if a is None or b is None:
        a, b = find_ab_params(spread, min_dist)
    Y = embed(graph, n_components=n_components, maxiter=maxiter, alpha=alpha, gamma=gamma,
              negative_sample_rate=negative_sample_rate, init_pos=init_pos, random_state=random_state, a=a, b=b)
    out = data.copy() if copy else data
    out.obsm["X_umap"] = Y
    params = {"a": a, "b": b}
    if random_state != 0:
        params["random_state"] = random_state
    out.uns["umap"] = {"params": params}
    return out if copy else None
