"""Float64 numpy oracle for ``mu.tl.leiden`` / ``mu.tl.louvain``, stand-ins for the third-party packages the
reference's ``_cluster`` imports, and the loader that runs the unmodified reference driver with them.

What is restated from memory, because leidenalg, louvain-igraph, igraph, scanpy and natsort are not installed where
this was written [recalled]:
  * the RB-configuration quality of one layer, Q = sum_ij (A_ij - g k_i^out k_j^in / m) [s_i == s_j] with
    m = sum_ij A_ij, and of the multiplex, sum_l w_l Q_l;
  * scanpy's ``get_igraph_from_adjacency`` adds one edge per stored entry, so an undirected graph built from a
    symmetric matrix holds every edge twice and its quality is twice the directed one;
  * leidenalg's optimiser: queue-based local moving in random order over the neighbour communities plus an empty
    one, a refinement that merges singletons inside each community (restated greedy, without leidenalg's
    randomness and well-connectedness test), aggregation on the refined partition starting from the unrefined
    membership, levels while the aggregate shrinks, ``n_iterations`` rounds (< 0: until one changes nothing), and
    the membership renumbered by decreasing community size; louvain-igraph is the same without refinement, run until
    nothing changes;
  * ``optimise_partition_multiplex`` returns sum_l w_l (Q_l(after) - Q_l(before)) (its ``n_iterations`` default 2);
  * scanpy's ``_choose_graph`` raises ``KeyError('No "<key>" in .uns')`` for a missing neighbours key.

Also here: the device's local-moving sweep and refinement round restated in numpy with the same fixed-point
arithmetic and hash (the tight reference of csrc/leiden.cu), brute-force move gains, node optimality and a
per-community connectivity check.  Nothing in the package imports this module.
"""
from __future__ import annotations

import os
import sys
import types
from collections import deque

import numpy as np
import scipy.sparse as sp

MASK = np.uint64(0xFFFFFFFFFFFFFFFF)


# ---- quality --------------------------------------------------------------------------------------------------
def layer_quality(labels, A, gamma):
    A = sp.csr_matrix(A, dtype=np.float64)
    labels = np.asarray(labels)
    m = A.sum()
    coo = A.tocoo()
    E = coo.data[labels[coo.row] == labels[coo.col]].sum()
    _, inv = np.unique(labels, return_inverse=True)
    Kout = np.bincount(inv, np.asarray(A.sum(1)).ravel())
    Kin = np.bincount(inv, np.asarray(A.sum(0)).ravel())
    return float(E - gamma * (Kout * Kin).sum() / m)


def quality(labels, layers, weights, gammas, directed=True):
    """sum_l w_l Q_l (RB configuration); twice that for igraph's undirected graphs (every edge stored twice)."""
    q = sum(w * layer_quality(labels, A, g) for A, w, g in zip(layers, weights, gammas))
    return q if directed else 2.0 * q


# ---- the collapsed problem in float64 ------------------------------------------------------------------------------
class Collapsed:
    """sum_l w_l A^l as one CSR (float64), degrees k [n x L], c_l = w_l g_l / m_l."""

    def __init__(self, layers, weights, gammas):
        layers = [sp.csr_matrix(A, dtype=np.float64) for A in layers]
        S = sum(w * A for A, w in zip(layers, weights)).tocsr()
        S.sum_duplicates()
        S.eliminate_zeros()
        S.sort_indices()
        self.A = S
        self.n = S.shape[0]
        self.k = np.stack([np.asarray(A.sum(1)).ravel() for A in layers], 1)
        self.c = np.array([w * g / A.sum() for A, w, g in zip(layers, weights, gammas)])

    def quality(self, labels):
        coo = self.A.tocoo()
        _, inv = np.unique(labels, return_inverse=True)
        E = coo.data[labels[coo.row] == labels[coo.col]].sum()
        K = np.stack([np.bincount(inv, self.k[:, l]) for l in range(self.k.shape[1])], 1)
        return float(E - (self.c * (K * K)).sum())


def move_gain(C: Collapsed, labels, v, b):
    """Closed-form gain of moving v from its community to b (any label, or a label no vertex has: empty)."""
    labels = np.asarray(labels)
    a = labels[v]
    if b == a:
        return 0.0
    row = slice(C.A.indptr[v], C.A.indptr[v + 1])
    nb, w = C.A.indices[row], C.A.data[row]
    off = nb != v
    e_b = w[off & (labels[nb] == b)].sum()
    e_a = w[off & (labels[nb] == a)].sum()
    Ka = C.k[labels == a].sum(0)
    Kb = C.k[labels == b].sum(0)
    kv = C.k[v]
    return float(2 * (e_b - e_a) - 2 * (C.c * kv * (Kb - Ka + kv)).sum())


def best_moves(C: Collapsed, labels):
    """For every vertex the largest gain of a move to a neighbour community or to an empty one (brute force,
    vectorised over the stored entries)."""
    labels = np.asarray(labels, dtype=np.int64)
    n = C.n
    _, inv = np.unique(labels, return_inverse=True)
    nc = inv.max() + 1
    K = np.stack([np.bincount(inv, C.k[:, l], minlength=nc) for l in range(C.k.shape[1])], 1)
    size = np.bincount(inv, minlength=nc)
    coo = C.A.tocoo()
    keep = coo.row != coo.col
    r, cc, w = coo.row[keep], inv[coo.col[keep]], coo.data[keep]
    E = sp.csr_matrix((w, (r, cc)), shape=(n, nc))
    E.sum_duplicates()
    e_own = np.asarray(E[np.arange(n), inv]).ravel()
    Ka = K[inv]
    kv = C.k
    best = np.full(n, -np.inf)
    Ec = E.tocoo()
    g = 2 * (Ec.data - e_own[Ec.row]) - 2 * (C.c * kv[Ec.row] * (K[Ec.col] - Ka[Ec.row] + kv[Ec.row])).sum(1)
    g[Ec.col == inv[Ec.row]] = -np.inf
    np.maximum.at(best, Ec.row, g)
    g_empty = -2 * e_own - 2 * (C.c * kv * (-Ka + kv)).sum(1)
    g_empty[size[inv] == 1] = -np.inf
    return np.maximum(best, g_empty)


def node_optimality_violations(C: Collapsed, labels, tol):
    """Vertices with a move (to a neighbour community or an empty one) that gains more than tol."""
    return int((best_moves(C, labels) > tol).sum())


def disconnected_communities(A, labels):
    """Communities whose induced subgraph of A is not connected."""
    from scipy.sparse.csgraph import connected_components
    coo = sp.coo_matrix(A)
    keep = labels[coo.row] == labels[coo.col]
    G = sp.csr_matrix((np.ones(keep.sum()), (coo.row[keep], coo.col[keep])), shape=A.shape)
    n_comp, comp = connected_components(G, directed=False)
    return int(n_comp - np.unique(labels).size)


# ---- the device steps, restated --------------------------------------------------------------------------------
def _splitmix64(x):
    x = (x + np.uint64(0x9E3779B97F4A7C15)) & MASK
    x = ((x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)) & MASK
    x = ((x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)) & MASK
    return x ^ (x >> np.uint64(31))


def vertex_hash(key, v):
    with np.errstate(over="ignore"):
        return _splitmix64(np.uint64(key) ^ (np.asarray(v, dtype=np.uint64) * np.uint64(0xD1B54A32D192ED03)))


def priority(key, v):
    h = vertex_hash(key, v)
    return (np.uint64(1 << 63) | ((h >> np.uint64(33)) << np.uint64(32))
            | np.asarray(v, dtype=np.uint64) & np.uint64(0xFFFFFFFF))


def coin(key, v):
    return (vertex_hash(key, v) >> np.uint64(63)) != 0


def _score(ev, kv, Kc, ce, cl):
    acc = np.zeros(len(ev))
    for l in range(len(cl)):
        acc = acc + (cl[l] * kv[:, l].astype(np.float64)) * Kc[:, l].astype(np.float64)
    return ev.astype(np.float64) * ce + (-acc)


def _pairs(indptr, indices, wq, memb, keep=None):
    """(vertex, community, e) for every vertex and every community among its neighbours u != v (int64 sums)."""
    n = len(indptr) - 1
    rows = np.repeat(np.arange(n), np.diff(indptr))
    ok = indices != rows
    if keep is not None:
        ok &= keep(rows, indices)
    r, c, w = rows[ok], memb[indices[ok]].astype(np.int64), wq[ok]
    key = r * (n + 1) + c
    uk, inv = np.unique(key, return_inverse=True)
    e = np.zeros(uk.size, dtype=np.int64)
    np.add.at(e, inv, w)
    return uk // (n + 1), uk % (n + 1), e


def _totals(memb, kq, cap):
    K = np.zeros((cap, kq.shape[1]), dtype=np.int64)
    np.add.at(K, memb, kq)
    return K, np.bincount(memb, minlength=cap)


def _argbest(v, c, s, n):
    """Per vertex: the index of the largest s, ties to the smaller c (-1 where v has none)."""
    out = np.full(n, -1, dtype=np.int64)
    if v.size:
        order = np.lexsort((c, -s, v))
        first = np.ones(order.size, dtype=bool)
        first[1:] = v[order][1:] != v[order][:-1]
        out[v[order][first]] = order[first]
    return out


def _pick(arr, ib, fill):
    """arr[ib] where ib >= 0, else fill."""
    out = np.full(ib.shape, fill, dtype=np.result_type(arr, type(fill)))
    out[ib >= 0] = arr[ib[ib >= 0]]
    return out


def compact(memb):
    _, inv = np.unique(memb, return_inverse=True)
    return inv.astype(np.int64)


MARGIN = 2.0 ** -40


def sweep_ref(P, comm, key):
    """One local-moving sweep of csrc/leiden.cu on the fixed-point problem P (``_leiden.Problem`` fields) from the
    compact membership comm -> (new compact membership, moves, target [n], gain [n])."""
    n = P.n
    comm = np.asarray(comm, dtype=np.int64)
    K, size = _totals(comm, P.kq, n)
    v, c, e = _pairs(P.indptr, P.indices, P.wq, comm)
    own = c == comm[v]
    e_own = np.zeros(n, dtype=np.int64)
    e_own[v[own]] = e[own]
    v, c, e = v[~own], c[~own], e[~own]
    s = _score(e, P.kq[v], K[c], P.ce, P.cl)
    ib = _argbest(v, c, s, n)
    has = ib >= 0
    best, bc, eb = _pick(s, ib, -np.inf), _pick(c, ib, -1), _pick(e, ib, 0)
    to_empty = (size[comm] > 1) & (~has | (best < 0.0))
    go = has | to_empty
    de = np.where(to_empty, 0, eb) - e_own
    Kb = np.where(to_empty[:, None], 0, K[np.maximum(bc, 0)])
    acc = np.zeros(n)
    mag = np.zeros(n)
    for l in range(P.L):
        dK = Kb[:, l] - K[comm, l] + P.kq[:, l]
        t = (P.cl[l] * P.kq[:, l].astype(np.float64)) * dK.astype(np.float64)
        acc = acc + t
        mag = mag + np.abs(t)
    ex = de.astype(np.float64) * P.ce
    g = 2.0 * (ex + (-acc))
    scale = 2.0 * (np.abs(ex) + mag)
    take = go & (g > MARGIN * scale)
    target = np.where(take, np.where(to_empty, n + np.arange(n), bc), -1)
    gain = np.where(take, g, 0.0)
    # all proposals at once; while the exact change of quality is not positive, the higher-priority half of them
    movers = np.nonzero(target >= 0)[0]
    if movers.size == 0:
        return comm, 0, target, gain
    p = priority(key, movers)
    movers, p = movers[np.argsort(p)[::-1]], np.sort(p)[::-1]
    e0 = _internal(P, comm)
    Kp = np.zeros((2 * n, P.L), dtype=np.int64)
    Kp[:n] = K
    keep = movers.size
    while True:
        new = comm.copy()
        new[movers[:keep]] = target[movers[:keep]]
        K1, _ = _totals(new, P.kq, 2 * n)
        dK = ((K1 - Kp).astype(np.float64) * (K1 + Kp).astype(np.float64) * P.cl).sum()
        dQ = float(_internal(P, new) - e0) * P.ce - dK
        if dQ > 0.0:
            break
        if keep <= 1:
            return comm, 0, target, gain
        keep = (keep + 1) // 2
    if (new >= n).any():
        new = compact(new)
    return new, int(keep), target, gain


def _internal(P, memb):
    rows = np.repeat(np.arange(P.n), np.diff(P.indptr))
    return int(P.wq[memb[rows] == memb[P.indices]].sum())


def refine_round_ref(P, refined, comm, key):
    """One refinement round of csrc/leiden.cu -> (new refined membership, moves, pending, target, gain)."""
    n = P.n
    refined = np.asarray(refined, dtype=np.int64)
    comm = np.asarray(comm, dtype=np.int64)
    K, size = _totals(refined, P.kq, n)
    single = size[refined] == 1
    v, c, e = _pairs(P.indptr, P.indices, P.wq, refined, keep=lambda r, u: comm[r] == comm[u])
    sel = single[v]
    v, c, e = v[sel], c[sel], e[sel]
    s = _score(e, P.kq[v], K[c], P.ce, P.cl)
    pending_v = np.zeros(n, dtype=bool)
    np.logical_or.at(pending_v, v, s >= 0.0)
    allowed = ~((size[c] == 1) & coin(key, c))
    ib = _argbest(v[allowed], c[allowed], s[allowed], n)
    has = ib >= 0
    best = _pick(s[allowed], ib, -np.inf)
    mover = coin(key, np.arange(n))
    take = single & mover & has & (best >= 0.0)
    target = np.where(take, _pick(c[allowed], ib, -1), -1)
    gain = np.where(take, 2.0 * best, 0.0)
    pending = bool((pending_v & single & ~take).any())
    new = refined.copy()
    new[take] = target[take]
    return new, int(take.sum()), pending, target, gain


# ---- leidenalg's optimiser, restated sequentially (quality reference and stand-in) -------------------------------
def _move_nodes(A, k, c, comm, rng):
    n = A.shape[0]
    K = np.zeros((n, k.shape[1]))
    np.add.at(K, comm, k)
    size = np.bincount(comm, minlength=n)
    empty = [i for i in range(n) if size[i] == 0]
    queue = deque(rng.permutation(n).tolist())
    inq = np.ones(n, dtype=bool)
    indptr, indices, data = A.indptr, A.indices, A.data
    while queue:
        v = queue.popleft()
        inq[v] = False
        a = comm[v]
        e = {}
        for j in range(indptr[v], indptr[v + 1]):
            u = indices[j]
            if u != v:
                e[comm[u]] = e.get(comm[u], 0.0) + data[j]
        K[a] -= k[v]
        size[a] -= 1
        if size[a] == 0:
            empty.append(a)
        kc = c * k[v]
        best, best_s = a, e.get(a, 0.0) - float(kc @ K[a])
        for cc, ev in e.items():
            if cc == a:
                continue
            s = ev - float(kc @ K[cc])
            if s > best_s:
                best, best_s = cc, s
        if size[a] > 0 and empty and 0.0 > best_s:
            best = empty[-1]
        if size[best] == 0:
            empty.remove(best)
        K[best] += k[v]
        size[best] += 1
        comm[v] = best
        if best != a:
            for j in range(indptr[v], indptr[v + 1]):
                u = indices[j]
                if comm[u] != best and not inq[u]:
                    queue.append(u)
                    inq[u] = True
    return compact(comm)


def _merge_constrained(A, k, c, comm, rng):
    n = A.shape[0]
    refined = np.arange(n)
    Kr = k.astype(np.float64).copy()
    size = np.ones(n, dtype=np.int64)
    indptr, indices, data = A.indptr, A.indices, A.data
    for v in rng.permutation(n):
        if size[refined[v]] != 1:
            continue
        e = {}
        for j in range(indptr[v], indptr[v + 1]):
            u = indices[j]
            if u != v and comm[u] == comm[v]:
                e[refined[u]] = e.get(refined[u], 0.0) + data[j]
        kc = c * k[v]
        best, best_s = None, 0.0
        for cc in sorted(e):
            s = e[cc] - float(kc @ Kr[cc])
            if s >= best_s and (best is None or s > best_s):
                best, best_s = cc, s
        if best is not None:
            Kr[refined[v]] -= k[v]
            size[refined[v]] -= 1
            refined[v] = best
            Kr[best] += k[v]
            size[best] += 1
    return compact(refined)


def renumber_by_size(labels):
    uniq, first, inv = np.unique(labels, return_index=True, return_inverse=True)
    size = np.bincount(inv)
    order = np.lexsort((first, -size))
    rank = np.empty_like(order)
    rank[order] = np.arange(order.size)
    return rank[inv]


def sequential(C: Collapsed, *, refine=True, n_iterations=2, seed=0, initial=None):
    """leidenalg's optimise_partition (refine) / louvain-igraph's (not) on the collapsed problem -> labels by size."""
    rng = np.random.RandomState(seed)
    memb = np.arange(C.n) if initial is None else compact(initial)
    it = 0
    while n_iterations < 0 or it < n_iterations:
        A, k = C.A, C.k
        comm = memb.copy()
        to_top = np.arange(C.n)
        while True:
            comm = _move_nodes(A, k, C.c, comm, rng)
            if refine:
                rid = _merge_constrained(A, k, C.c, comm, rng)
                agg = np.zeros(rid.max() + 1, dtype=np.int64)
                agg[rid] = comm
                agg = compact(agg)
            else:
                rid = comm
                agg = np.arange(rid.max() + 1)
            n_agg = rid.max() + 1
            if n_agg == A.shape[0]:
                break
            Pm = sp.csr_matrix((np.ones(A.shape[0]), (np.arange(A.shape[0]), rid)), shape=(A.shape[0], n_agg))
            A = (Pm.T @ A @ Pm).tocsr()
            A.sort_indices()
            k = Pm.T @ k
            to_top = rid[to_top]
            comm = agg
        new = compact(comm[to_top])
        it += 1
        changed = not np.array_equal(renumber_by_size(new), renumber_by_size(memb))
        memb = new
        if not changed:
            break
    return renumber_by_size(memb)


# ---- planted graphs -------------------------------------------------------------------------------------------------
def random_graph(labels, p_in, p_out, seed, weighted=True):
    """Symmetric graph: pairs with the same label are linked with probability p_in, others p_out; weights in
    (0.5, 1] (or 1)."""
    rng = np.random.default_rng(seed)
    n = len(labels)
    iu, ju = np.triu_indices(n, 1)
    same = labels[iu] == labels[ju]
    keep = rng.random(iu.size) < np.where(same, p_in, p_out)
    r, c = iu[keep], ju[keep]
    w = 0.5 + 0.5 * rng.random(r.size) if weighted else np.ones(r.size)
    A = sp.coo_matrix((np.r_[w, w], (np.r_[r, c], np.r_[c, r])), shape=(n, n)).tocsr()
    A.sort_indices()
    return A.astype(np.float32)


def small_case():
    """Two modalities over the same 4 planted clusters of distinct sizes (the fixture's graphs)."""
    labels = np.repeat(np.arange(4), [80, 60, 45, 30])
    return labels, random_graph(labels, 0.3, 0.01, 1), random_graph(labels, 0.25, 0.012, 2)


# the reference calls recorded in tests/golden/leiden_small.npz
REFERENCE_CALLS = {
    "default": {},
    "resolution_dict": {"resolution": {"rna": 0.8, "atac": 1.2}},
    "mod_weights_list": {"mod_weights": [1.0, 0.5]},
    "weighted": {"partition_kwargs": {"weights": "weight"}},
}


def multiplex_case(s=60, seed=0):
    """8 planted clusters; modality a links clusters 2i and 2i+1 alike, modality b links i and i + 4 alike, so each
    alone sees 4 groups and only both together separate the 8."""
    labels = np.repeat(np.arange(8), s)
    A = random_graph(labels // 2, 0.3, 0.005, seed + 1)
    B = random_graph(labels % 4, 0.3, 0.005, seed + 2)
    return labels, A, B


# ---- stand-ins for the reference driver's third-party imports ----------------------------------------------------
class Graph:
    """igraph.Graph as scanpy's get_igraph_from_adjacency builds it: one edge per stored entry, es['weight']."""

    def __init__(self, adjacency, directed):
        self.adjacency = sp.csr_matrix(adjacency)
        self.directed = bool(directed)
        self.es = {"weight": self.adjacency.data}

    def vcount(self):
        return self.adjacency.shape[0]


def get_igraph_from_adjacency(adjacency, directed=None):
    return Graph(adjacency, directed)


def choose_graph(adata, obsp, neighbors_key):
    if obsp is not None and neighbors_key is not None:
        raise ValueError("You can't specify both obsp, neighbors_key. Please select only one.")
    if obsp is not None:
        return adata.obsp[obsp]
    key = "neighbors" if neighbors_key is None else neighbors_key
    if key not in adata.uns:
        raise KeyError(f'No "{key}" in .uns')
    return adata.obsp[adata.uns[key].get("connectivities_key", "connectivities")]


def natsorted(seq):
    import re
    return sorted(seq, key=lambda s: [int(t) if t.isdigit() else t for t in re.split(r"(\d+)", str(s))])


def _partition_module(name, refine):
    class RBConfigurationVertexPartition:
        def __init__(self, graph, weights=None, resolution_parameter=1.0, initial_membership=None):
            self.graph = graph
            self.weights = weights
            self.resolution_parameter = resolution_parameter
            self.membership = list(range(graph.vcount()))

        def layer(self):
            A = graph_matrix = self.graph.adjacency.astype(np.float64)
            if self.weights is None:
                A = graph_matrix.copy()
                A.data[:] = 1.0
            elif isinstance(self.weights, str):
                A = sp.csr_matrix((np.asarray(self.graph.es[self.weights], np.float64), graph_matrix.indices,
                                   graph_matrix.indptr), shape=graph_matrix.shape)
            return A

    class Optimiser:
        def __init__(self):
            self.seed = 0

        def set_rng_seed(self, seed):
            self.seed = int(seed)

        def optimise_partition_multiplex(self, partitions, layer_weights=None, n_iterations=2,
                                         is_membership_fixed=None):
            weights = [1.0] * len(partitions) if layer_weights is None else list(layer_weights)
            layers = [p.layer() for p in partitions]
            gammas = [p.resolution_parameter for p in partitions]
            directed = partitions[0].graph.directed
            before = quality(np.asarray(partitions[0].membership), layers, weights, gammas, directed)
            C = Collapsed(layers, weights, gammas)
            labels = sequential(C, refine=refine, n_iterations=n_iterations if refine else -1, seed=self.seed)
            for p in partitions:
                p.membership = labels.tolist()
            return quality(labels, layers, weights, gammas, directed) - before

    m = types.ModuleType(name)
    m.__dict__["__stub__"] = True
    m.RBConfigurationVertexPartition = RBConfigurationVertexPartition
    m.Optimiser = Optimiser
    return m


def load_reference_cluster():
    """The reference's own ``leiden`` and ``louvain`` (muon/_core/tools.py:1057, 1133), executed unmodified with the
    stand-ins above for leidenalg, louvain, igraph, natsort, h5py and the scanpy helpers."""
    from oracle import _refload
    if not _refload.reference_available():
        raise FileNotFoundError(_refload.REF_ROOT)
    _refload.load_reference_neighbors()          # stubs for anndata / mudata / scanpy, and preproc.py itself
    sys.modules.setdefault("h5py", types.ModuleType("h5py"))
    sys.modules.setdefault("natsort", types.ModuleType("natsort")).natsorted = natsorted
    sys.modules["scanpy.tools._utils"]._choose_graph = choose_graph
    sys.modules["scanpy._utils"].get_igraph_from_adjacency = get_igraph_from_adjacency
    sys.modules["leidenalg"] = _partition_module("leidenalg", refine=True)
    sys.modules["louvain"] = _partition_module("louvain", refine=False)
    if "_refmuon_core" not in sys.modules:
        pkg = types.ModuleType("_refmuon_core")
        pkg.__path__ = []
        sys.modules["_refmuon_core"] = pkg
    sys.modules["_refmuon_core.preproc"] = sys.modules["_refmuon_core_preproc"]
    m = sys.modules.get("_refmuon_core.tools")
    if m is None:
        import importlib.util
        spec = importlib.util.spec_from_file_location("_refmuon_core.tools",
                                                      os.path.join(_refload.REF_ROOT, "muon/_core/tools.py"))
        m = importlib.util.module_from_spec(spec)
        sys.modules["_refmuon_core.tools"] = m
        spec.loader.exec_module(m)
    return m.leiden, m.louvain
