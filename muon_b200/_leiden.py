"""``mu.tl.leiden`` / ``mu.tl.louvain`` -- multiplex community detection on the GPU.

The reference (muon/_core/tools.py:928-1206) builds one igraph graph per modality and hands them to leidenalg's (or
louvain-igraph's) ``optimise_partition_multiplex`` with RB-configuration partitions; an AnnData goes to
``sc.tl.leiden`` / ``sc.tl.louvain``, i.e. the same optimiser on one graph.  Here both branches build the same
problem and run it on the device (csrc/leiden.cu).

The multiplex objective  sum_l w_l sum_ij (A^l_ij - g_l k^l_i k^l_j / m_l) [s_i == s_j]  is linear in the adjacency,
so the host collapses it to one graph with weights sum_l w_l A^l_uv, the per-layer degrees k^l_v and the constants
c_l = w_l g_l / m_l (``prepare``).  Aggregating a partition keeps that form, so every level is the same problem.
Weights and degrees go to the device as int64 fixed point (every total below 2^53), which makes every sum exact:
the result does not depend on the order of atomics, and a given ``random_state`` gives bit-identical labels.

One level: local moving (sweeps until no vertex has a positive move; a sweep applies every proposal at once and is
kept only if the exact change of quality is positive, else the higher-priority half of its moves is tried), then -- Leiden only -- the refinement (singletons merge into sub-communities of their
community that they touch), then aggregation on the refined partition (Leiden, starting from the unrefined
membership) or on the moved partition (Louvain).  Levels repeat while the aggregate shrinks.  An outer iteration
restarts from the current membership on the original graph, ``n_iterations`` times (< 0: until one changes nothing).

Departures from leidenalg, all deliberate:
  * The moves are parallel sweeps, not a sequential queue, and ``random_state`` seeds a counter-based hash
    (splitmix64) that sets the sweep priorities and the refinement's coins, not leidenalg's generator: the labels are
    a local optimum of the same objective, not leidenalg's for the same seed.
  * The refinement is greedy (leidenalg draws among the positive merges with randomness 0.01) and has no
    well-connectedness test; every refined sub-community lies inside one community and is connected.
  * ``random_state=0`` (or None) is a seed like any other: the run is deterministic.
"""
from __future__ import annotations

import numbers
from collections.abc import Mapping, Sequence
from types import MappingProxyType

import numpy as np

from ._containers import is_anndata, is_mudata
from ._lib import LEIDEN_MAX_LAYERS

MASK64 = (1 << 64) - 1
MOVE, REFINE = 0, 1
REFINE_ROUND_CAP = 100_000      # far above the rounds the coins need (about 150 per level measured)


# ---- the problem: one graph, per-layer degrees, fixed point ------------------------------------------------------
class Problem:
    """The multiplex RB-configuration problem as one graph (host, numpy).

    ``indptr, indices`` the union pattern (symmetric, sorted rows), ``w`` [nnz] the combined weights sum_l w_l A^l_uv
    and ``k`` [n x L] the per-layer degrees in float64; ``wq`` / ``kq`` the same in int64 fixed point (scales 2^se /
    2^sk); ``c`` [L] = w_l g_l / m_l, ``ce`` = 2^-se and ``cl`` = c_l 2^-2sk the constants the kernels use."""

    def __init__(self, layers, layer_weights, gammas):
        import scipy.sparse as sp
        L = len(layers)
        n = layers[0].shape[0]
        self.n, self.L = n, L
        self.layer_weights = np.asarray(layer_weights, dtype=np.float64)
        self.gammas = np.asarray(gammas, dtype=np.float64)
        self.m = np.array([float(A.sum()) for A in layers])
        S = sp.csr_matrix((n, n), dtype=np.float64)
        for A, wl in zip(layers, self.layer_weights):
            S = S + wl * A
        S = sp.csr_matrix(S)
        S.sum_duplicates()
        S.eliminate_zeros()
        S.sort_indices()
        self.indptr = S.indptr.astype(np.int64)
        self.indices = S.indices.astype(np.int32)
        self.w = S.data.astype(np.float64)
        self.k = np.stack([np.asarray(A.sum(axis=1), dtype=np.float64).ravel() for A in layers], 1)
        self.c = self.layer_weights * self.gammas / self.m
        self.se = 52 - int(np.ceil(np.log2(max(float(self.w.sum()), 1.0))))
        self.sk = 52 - int(np.ceil(np.log2(max(float(self.m.max()), 1.0))))
        self.wq = np.rint(np.ldexp(self.w, self.se)).astype(np.int64)
        self.kq = np.ascontiguousarray(np.rint(np.ldexp(self.k, self.sk)).astype(np.int64))
        self.ce = float(np.ldexp(1.0, -self.se))
        self.cl = np.array([float(np.ldexp(c, -2 * self.sk)) for c in self.c])


def layer_matrix(adjacency, use_weights: bool):
    """A connectivities matrix as float64 CSR: its values (``use_weights``) or 1 on its pattern.  It must be square
    and symmetric in pattern and values, and non-negative."""
    import scipy.sparse as sp
    A = sp.csr_matrix(adjacency, dtype=np.float64, copy=True)
    A.sum_duplicates()
    A.eliminate_zeros()
    if A.shape[0] != A.shape[1]:
        raise ValueError(f"the adjacency must be square, not {A.shape}")
    if A.nnz and A.data.min() < 0:
        raise NotImplementedError("negative edge weights are not supported")
    if not use_weights:
        A.data[:] = 1.0
    if (A != A.T).nnz:
        raise NotImplementedError("the adjacency must be symmetric (pattern and values): directed graphs with "
                                  "asymmetric edges are not supported")
    A.sort_indices()
    return A


# ---- keys of the counter-based hash ----------------------------------------------------------------------------
def splitmix64(x: int) -> int:
    x = (x + 0x9E3779B97F4A7C15) & MASK64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & MASK64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & MASK64
    return x ^ (x >> 31)


def stream_key(seed: int, phase: int, iteration: int, level: int, step: int) -> int:
    """The key of one sweep (phase MOVE) or refinement round (phase REFINE)."""
    tag = (phase << 60) | ((iteration & 0xFFFFF) << 40) | ((level & 0xFFFF) << 24) | (step & 0xFFFFFF)
    return splitmix64(splitmix64(seed & MASK64) ^ tag)


# ---- device ------------------------------------------------------------------------------------------------------
def _compact(memb, cap):
    """Order-preserving renumbering of the ids in memb (device int32, values < cap) -> (new memb, count)."""
    import torch
    used = torch.zeros(cap, dtype=torch.int32, device=memb.device)
    used[memb.long()] = 1
    newid = torch.cumsum(used, 0, dtype=torch.int32) - 1
    return newid[memb.long()].contiguous(), int(used.sum())


class Level:
    """One level's graph on the device: CSR with fixed-point weights, fixed-point degrees [n x L], and the hub rows
    (longer than the shared-memory table takes) with their global-memory tables."""

    def __init__(self, indptr, indices, wq, kq, ce, cl):
        import torch

        from . import _lib
        from ._device import require_cuda
        require_cuda()
        dev = torch.device("cuda", torch.cuda.current_device())

        def t(a, dt):
            return a.to(dev, dt).contiguous() if isinstance(a, torch.Tensor) else \
                torch.from_numpy(np.ascontiguousarray(a)).to(dev, dt)

        self.indptr, self.indices, self.wq = t(indptr, torch.int64), t(indices, torch.int32), t(wq, torch.int64)
        self.kq = t(kq, torch.int64)
        self.n, self.L = self.kq.shape
        self.ce = float(ce)
        self.cl = torch.from_numpy(np.ascontiguousarray(cl, dtype=np.float64))    # host array, read at launch
        self.dev = dev
        deg = self.indptr[1:] - self.indptr[:-1]
        hubs = torch.nonzero(deg > _lib.load().mub_leiden_max_shared_degree()).ravel()
        self.n_hubs = int(hubs.numel())
        if self.n_hubs:
            d = deg[hubs]
            slots = torch.pow(2, torch.ceil(torch.log2((2 * d).double())).long()).to(torch.int64)
            self.hub_slots = slots.to(torch.int32)
            self.hub_off = (torch.cumsum(slots, 0) - slots).contiguous()
            total = int(slots.sum())
            self.hubs = hubs.to(torch.int32)
            self.hub_keys = torch.empty(total, dtype=torch.int32, device=dev)
            self.hub_vals = torch.empty(total, dtype=torch.int64, device=dev)
            self.hub_lists = torch.empty(total // 2, dtype=torch.int32, device=dev)
            self.hub_counts = torch.empty(self.n_hubs, dtype=torch.int32, device=dev)
        else:
            self.hubs = self.hub_off = self.hub_slots = self.hub_keys = None
            self.hub_vals = self.hub_lists = self.hub_counts = None
        self.flags = torch.zeros(1, dtype=torch.int32, device=dev)
        self.counts = torch.zeros(2, dtype=torch.int32, device=dev)
        self.prio = torch.empty(self.n, dtype=torch.int64, device=dev)
        self.cl_dev = self.cl.to(dev)

    @classmethod
    def from_problem(cls, P: Problem):
        return cls(P.indptr, P.indices, P.wq, P.kq, P.ce, P.cl)

    # -- single steps --
    def totals(self, memb, n_comm):
        import torch

        from ._lib import call, ptr, stream_ptr
        K = torch.empty((n_comm, self.L), dtype=torch.int64, device=self.dev)
        size = torch.empty(n_comm, dtype=torch.int32, device=self.dev)
        call("mub_leiden_totals", self.n, self.L, ptr(memb), ptr(self.kq), n_comm, ptr(K), ptr(size), stream_ptr())
        return K, size

    def scan(self, mode, memb, parent, K, size, key):
        """Every vertex's proposal: (target, gain) device tensors."""
        import torch

        from ._lib import call, ptr, stream_ptr
        target = torch.empty(self.n, dtype=torch.int32, device=self.dev)
        gain = torch.empty(self.n, dtype=torch.float64, device=self.dev)
        self.flags.zero_()
        call("mub_leiden_scan", mode, ptr(self.indptr), ptr(self.indices), ptr(self.wq), ptr(self.kq), self.n,
             self.L, self.ce, self.cl.data_ptr(), ptr(memb), ptr(parent), ptr(K), ptr(size), key, ptr(target),
             ptr(gain), ptr(self.flags), ptr(self.hubs), self.n_hubs, ptr(self.hub_off), ptr(self.hub_slots),
             ptr(self.hub_keys), ptr(self.hub_vals), ptr(self.hub_lists), ptr(self.hub_counts), stream_ptr())
        return target, gain

    def sweep(self, comm, key, stats=None):
        """One local-moving sweep from the membership ``comm`` (device int32, ids < n).  Every vertex with a positive
        move proposes it; all proposals are applied at once and kept if the exact change of quality is positive,
        otherwise the higher-priority half of them is tried, and so on.  Returns the new membership (compact when a
        vertex opened a community), the number of accepted moves (0: no vertex has a positive move, or only a single
        move whose gain is lost in rounding is left) and every vertex's proposal (target, gain)."""
        import torch

        from ._lib import call, ptr, stream_ptr
        n = self.n
        K, size = self.totals(comm, n)
        target, gain = self.scan(MOVE, comm, None, K, size, key)
        e0 = self.internal(comm)
        Kp = torch.zeros((2 * n, self.L), dtype=torch.int64, device=self.dev)
        Kp[:n] = K
        thr, movers = 0, None
        while True:
            new = comm.clone()
            call("mub_leiden_apply", MOVE, n, ptr(new), ptr(target), key, thr, ptr(self.prio), ptr(self.counts),
                 stream_ptr())
            moved, to_empty = (int(v) for v in self.counts.cpu())
            if not moved:
                return comm, 0, target, gain
            K1, _ = self.totals(new, 2 * n)
            dK = float(((K1 - Kp).double() * (K1 + Kp).double() * self.cl_dev).sum())
            dQ = float(self.internal(new) - e0) * self.ce - dK
            if dQ > 0.0:
                break
            if movers is None:          # the priorities have their top bit set: as int64 they sort like uint64
                movers = torch.sort(self.prio[self.prio != 0], descending=True).values
            if movers.numel() <= 1:
                return comm, 0, target, gain
            movers = movers[:(movers.numel() + 1) // 2]
            thr = int(movers[-1]) & MASK64
            if stats is not None:
                stats["retries"] = stats.get("retries", 0) + 1
        if to_empty:
            new, _ = _compact(new, 2 * n)
        return new, moved, target, gain

    def refine_round(self, refined, comm, key):
        """One refinement round: (new refined membership, moves, pending flag, target, gain).  Sub-community ids are
        vertex ids (a sub-community is named after the singleton it grew from)."""
        from ._lib import call, ptr, stream_ptr
        K, size = self.totals(refined, self.n)
        target, gain = self.scan(REFINE, refined, comm, K, size, key)
        new = refined.clone()
        call("mub_leiden_apply", REFINE, self.n, ptr(new), ptr(target), key, 0, None, ptr(self.counts),
             stream_ptr())
        moved = int(self.counts[0])
        pending = bool(int(self.flags[0]))
        return new, moved, pending, target, gain

    # -- phases --
    def local_moving(self, comm, seed, iteration, level, stats):
        sweep = 0
        while True:
            comm, moved, _, _ = self.sweep(comm, stream_key(seed, MOVE, iteration, level, sweep), stats)
            sweep += 1
            if not moved:
                break
        stats["sweeps"] += sweep
        return comm

    def refine(self, comm, seed, iteration, level, stats):
        import torch
        refined = torch.arange(self.n, dtype=torch.int32, device=self.dev)
        r = 0
        while True:
            refined, moved, pending, _, _ = self.refine_round(refined, comm, stream_key(seed, REFINE, iteration,
                                                                                        level, r))
            r += 1
            if not moved and not pending:
                break
            # Every round either moves a singleton (at most n moves in all) or has a singleton whose only targets are
            # moving singletons; the hashed coins change every round, so such a round repeats with probability <= 3/4.
            if r > REFINE_ROUND_CAP:
                raise RuntimeError(f"the refinement did not settle in {REFINE_ROUND_CAP} rounds")
        stats["refine_rounds"] += r
        return refined

    def aggregate(self, rid, n_agg):
        """The graph of the partition rid (compact, device): entry (rid[u], rid[v]) carries the sum of the weights,
        degrees are summed.  Keys are sorted (torch.sort), the reduces run in leiden.cu."""
        import torch

        from ._lib import call, ptr, stream_ptr
        rows = torch.repeat_interleave(torch.arange(self.n, device=self.dev, dtype=torch.int64),
                                       self.indptr[1:] - self.indptr[:-1])
        keys = rid.long()[rows] * n_agg + rid.long()[self.indices.long()]
        keys, order = torch.sort(keys)
        w = self.wq[order].contiguous()
        new_seg = torch.ones_like(keys, dtype=torch.bool)
        new_seg[1:] = keys[1:] != keys[:-1]
        seg = (torch.cumsum(new_seg.to(torch.int64), 0) - 1).contiguous()
        uk = keys[new_seg]
        nnz = int(uk.numel())
        wq = torch.empty(nnz, dtype=torch.int64, device=self.dev)
        call("mub_leiden_segment_sum", int(keys.numel()), ptr(seg), ptr(w), nnz, ptr(wq), stream_ptr())
        r, c = uk // n_agg, uk % n_agg
        indptr = torch.zeros(n_agg + 1, dtype=torch.int64, device=self.dev)
        indptr[1:] = torch.cumsum(torch.bincount(r, minlength=n_agg), 0)
        K, _ = self.totals(rid, n_agg)
        return Level(indptr, c.to(torch.int32), wq, K, self.ce, self.cl.numpy())

    def internal(self, memb) -> int:
        import torch

        from ._lib import call, ptr, stream_ptr
        out = torch.empty(1, dtype=torch.int64, device=self.dev)
        call("mub_leiden_internal", self.n, ptr(self.indptr), ptr(self.indices), ptr(self.wq), ptr(memb), ptr(out),
             stream_ptr())
        return int(out.item())

    def quality(self, memb) -> float:
        """sum_l w_l Q_l of the membership (directed form), from the fixed-point totals."""
        memb, n_comm = _compact(memb, self.n)
        K, _ = self.totals(memb, n_comm)
        Kd = K.cpu().numpy().astype(np.float64)
        return float(self.internal(memb)) * self.ce - float(((Kd * Kd) * self.cl.numpy()).sum())


def optimise(P: Problem, *, refine: bool, n_iterations: int, seed: int, stats=None):
    """Run the optimiser from singletons.  Returns (labels [n] int64 on the host, renumbered by decreasing size with
    ties to the smallest vertex, improvement sum_l w_l (Q_l(final) - Q_l(singletons)) in the directed form)."""
    import torch
    stats = stats if stats is not None else {}
    for s in ("levels", "sweeps", "retries", "refine_rounds", "iterations"):
        stats.setdefault(s, 0)
    base = Level.from_problem(P)
    memb = torch.arange(P.n, dtype=torch.int32, device=base.dev)
    q0 = base.quality(memb)
    it = 0
    while n_iterations < 0 or it < n_iterations:
        new = _one_iteration(base, memb, refine, seed, it, stats)
        it += 1
        changed = not torch.equal(new, memb)
        memb = new
        if not changed:
            break
    stats["iterations"] = it
    q1 = base.quality(memb)
    return renumber_by_size(memb.cpu().numpy()), q1 - q0


def _one_iteration(base, memb, refine, seed, iteration, stats):
    import torch
    level, lvl = base, 0
    comm, _ = _compact(memb, base.n)
    to_top = torch.arange(base.n, dtype=torch.int64, device=base.dev)
    while True:
        comm = level.local_moving(comm, seed, iteration, lvl, stats)
        stats["levels"] += 1
        if refine:
            rid, n_agg = _compact(level.refine(comm, seed, iteration, lvl, stats), level.n)
            agg = torch.empty(n_agg, dtype=torch.int32, device=base.dev)
            agg[rid.long()] = comm
            agg, _ = _compact(agg, level.n)
        else:
            rid, n_agg = _compact(comm, level.n)
            agg = torch.arange(n_agg, dtype=torch.int32, device=base.dev)
        if n_agg == level.n:
            break
        level = level.aggregate(rid, n_agg)
        to_top = rid.long()[to_top]
        comm, lvl = agg, lvl + 1
    # canonical ids: order of first occurrence on the original vertices
    out = comm[to_top]
    first = torch.full((base.n,), base.n, dtype=torch.int64, device=base.dev)
    first.scatter_reduce_(0, out.long(), torch.arange(base.n, device=base.dev), reduce="amin")
    rank = torch.empty_like(first)
    rank[torch.argsort(first)] = torch.arange(base.n, device=base.dev)
    return rank[out.long()].to(torch.int32)


def renumber_by_size(labels: np.ndarray) -> np.ndarray:
    """Labels 0..K-1 by decreasing community size, ties to the community holding the smallest vertex."""
    labels = np.asarray(labels)
    uniq, first, inv = np.unique(labels, return_index=True, return_inverse=True)
    size = np.bincount(inv)
    order = np.lexsort((first, -size))
    rank = np.empty_like(order)
    rank[order] = np.arange(order.size)
    return rank[inv].astype(np.int64)


# ---- public entry points -----------------------------------------------------------------------------------------
def _choose_graph(adata, neighbors_key):
    """scanpy.tools._utils._choose_graph(adata, None, neighbors_key): obsp[uns[key]["connectivities_key"]]."""
    key = "neighbors" if neighbors_key is None else neighbors_key
    if key not in adata.uns:
        raise KeyError(f'No "{key}" in .uns')
    return adata.obsp[adata.uns[key].get("connectivities_key", "connectivities")]


def _seed(random_state) -> int:
    if random_state is None:
        return 0
    if isinstance(random_state, numbers.Integral):
        return int(random_state)
    raise NotImplementedError("random_state must be an int (or None)")


def _categorical(labels):
    import pandas as pd
    k = int(labels.max()) + 1 if labels.size else 0
    return pd.Categorical(values=labels.astype("U"), categories=[str(i) for i in range(k)])


def _check_partition_type(partition_type):
    if partition_type is not None and getattr(partition_type, "__name__", None) != "RBConfigurationVertexPartition":
        raise NotImplementedError(f"partition_type {partition_type!r} is not supported: only "
                                  "RBConfigurationVertexPartition runs on the GPU")


def _anndata(adata, resolution, random_state, key_added, neighbors_key, algorithm, kwargs):
    """sc.tl.leiden / sc.tl.louvain on obsp[uns[neighbors_key]["connectivities_key"]]."""
    kwargs = dict(kwargs)
    for bad in ("restrict_to", "adjacency", "obsp", "flavor", "partition_type"):
        if bad in kwargs:
            raise NotImplementedError(f"{bad} is not supported")
    use_weights = bool(kwargs.pop("use_weights", algorithm == "leiden"))
    kwargs.pop("directed", None)            # a symmetric graph: directed or not gives the same partition
    copy = bool(kwargs.pop("copy", False))
    n_iterations = int(kwargs.pop("n_iterations", -1)) if algorithm == "leiden" else -1
    if kwargs:
        raise TypeError(f"unexpected keyword arguments: {sorted(kwargs)}")
    if resolution is not None and not isinstance(resolution, numbers.Real):
        raise TypeError("resolution must be a number for an AnnData object")
    A = layer_matrix(_choose_graph(adata, neighbors_key), use_weights)
    if A.nnz == 0:
        raise ValueError("the graph has no edges")
    gamma = 1.0 if resolution is None else float(resolution)
    labels, _ = optimise(Problem([A], [1.0], [gamma]), refine=algorithm == "leiden", n_iterations=n_iterations,
                         seed=_seed(random_state))
    out = adata.copy() if copy else adata
    out.obs[key_added] = _categorical(labels)
    params = dict(resolution=resolution, random_state=random_state)
    if algorithm == "leiden":
        params["n_iterations"] = n_iterations
    out.uns[key_added] = {"params": params}
    return out if copy else None


def _per_layer(value, mods, what):
    """The reference's Mapping / Sequence / scalar expansion of resolution and mod_weights."""
    if isinstance(value, Mapping):
        return value
    if isinstance(value, Sequence) and not isinstance(value, str):
        assert len(value) == len(mods), \
            f"Length of {what} ({len(value)}) does not match the number of modalities ({len(mods)})"
        return list(value)
    return [value for _ in mods]


def cluster(data, resolution=None, mod_weights=None, random_state=0, key_added="louvain", neighbors_key=None,
            directed=True, partition_type=None, partition_kwargs=MappingProxyType({}), algorithm="leiden",
            **kwargs):
    if algorithm not in ("leiden", "louvain"):
        raise ValueError(f"Algorithms should be either 'louvain' or 'leiden', not '{algorithm}'")
    if is_anndata(data) and not is_mudata(data):
        return _anndata(data, resolution, random_state, key_added, neighbors_key, algorithm, kwargs)
    if not is_mudata(data):
        raise TypeError("Expected a MuData object")
    mdata = data
    partition_kwargs = dict(partition_kwargs)
    mods = list(mdata.mod)
    graphs = [_choose_graph(mdata.mod[m], neighbors_key) for m in mods]

    if mod_weights:
        if isinstance(mod_weights, Mapping):
            layer_weights = [mod_weights.get(m, 1) for m in mods]
        else:
            layer_weights = _per_layer(mod_weights, mods, "layers_weights")
    else:
        layer_weights = [1.0] * len(mods)
    _check_partition_type(partition_type)
    unknown = set(partition_kwargs) - {"weights", "resolution_parameter"}
    if unknown:
        raise NotImplementedError(f"partition_kwargs {sorted(unknown)} are not supported")
    weights = partition_kwargs.get("weights")
    if weights is not None and not (isinstance(weights, str) and weights == "weight"):
        raise NotImplementedError("partition_kwargs['weights'] must be None or 'weight'")
    kwargs = dict(kwargs)
    if "is_membership_fixed" in kwargs:
        raise NotImplementedError("is_membership_fixed is not supported")
    n_iterations = int(kwargs.pop("n_iterations", 2)) if algorithm == "leiden" else -1
    if kwargs:
        raise TypeError(f"optimise_partition_multiplex() got unexpected keyword arguments {sorted(kwargs)}")

    if resolution:
        if "resolution_parameter" in partition_kwargs:
            raise TypeError("got multiple values for keyword argument 'resolution_parameter'")
        res = _per_layer(resolution, mods, "resolution")
        gammas = [res[m] for m in mods] if isinstance(res, Mapping) else res
    else:
        gammas = [partition_kwargs.get("resolution_parameter", 1.0)] * len(mods)

    if len(mods) > LEIDEN_MAX_LAYERS:
        raise NotImplementedError(f"{len(mods)} modalities: at most {LEIDEN_MAX_LAYERS} layers are supported")
    names = [list(map(str, mdata.mod[m].obs_names)) for m in mods]
    if any(nm != names[0] for nm in names[1:]) or list(map(str, mdata.obs_names)) != names[0]:
        raise NotImplementedError("every modality must hold the same observations in the same order")
    if any(float(x) < 0 for x in layer_weights):
        raise NotImplementedError("negative modality weights are not supported")
    layers = [layer_matrix(g, weights is not None) for g in graphs]
    for m, A in zip(mods, layers):
        if A.nnz == 0:
            raise ValueError(f"the graph of modality {m!r} has no edges")
    P = Problem(layers, [float(x) for x in layer_weights], [float(g) for g in gammas])
    labels, improvement = optimise(P, refine=algorithm == "leiden", n_iterations=n_iterations,
                                   seed=_seed(random_state) if random_state else 0)
    if not directed:
        improvement *= 2.0      # igraph's undirected graph from both triangles holds every edge twice
    mdata.obs[key_added] = _categorical(labels)
    mdata.uns[algorithm] = {"params": dict(resolution=resolution, random_state=random_state,
                                           partition_improvement=improvement)}
    return None


def leiden(data, resolution=None, mod_weights=None, random_state: int = 0, key_added: str = "leiden",
           neighbors_key: str = None, directed: bool = True, partition_type=None,
           partition_kwargs=MappingProxyType({}), **kwargs):
    """Cluster cells with multiplex Leiden on the GPU -- ``muon.tl.leiden`` (muon/_core/tools.py:1057), the same
    arguments and slots: ``obs[key_added]`` (categorical labels "0".."K-1" by decreasing size) and
    ``uns["leiden"]["params"]`` (MuData) or ``uns[key_added]["params"]`` (AnnData, as scanpy).  See the module
    docstring for what is supported and where the optimiser departs from leidenalg's."""
    return cluster(data, resolution=resolution, mod_weights=mod_weights, random_state=random_state,
                   key_added=key_added, neighbors_key=neighbors_key, directed=directed,
                   partition_type=partition_type, partition_kwargs=partition_kwargs, algorithm="leiden", **kwargs)


def louvain(data, resolution=None, mod_weights=None, random_state: int = 0, key_added: str = "louvain",
            neighbors_key: str = None, directed: bool = True, partition_type=None,
            partition_kwargs=MappingProxyType({}), **kwargs):
    """Cluster cells with multiplex Louvain on the GPU -- ``muon.tl.louvain`` (muon/_core/tools.py:1133): Leiden's
    local moving and aggregation without the refinement, run until an iteration changes nothing."""
    return cluster(data, resolution=resolution, mod_weights=mod_weights, random_state=random_state,
                   key_added=key_added, neighbors_key=neighbors_key, directed=directed,
                   partition_type=partition_type, partition_kwargs=partition_kwargs, algorithm="louvain", **kwargs)
