"""TEST INFRASTRUCTURE ONLY -- numpy restatement of the UMAP layout behind ``mu.tl.umap``.

umap-learn and scanpy are not installed here, so every umap-learn step below is RECALLED from umap-learn 0.5
(``simplicial_set_embedding``, ``spectral_layout``, ``multi_component_layout``, ``optimize_layout_euclidean`` with
parallel=False, ``tau_rand_int``) and scanpy's ``tl.umap`` wrapper, not copied or pinned against the package -- the
same standing as the recalled mofapy2 steps in SURVEY.md.

  * ``find_ab``, ``prune``, ``epochs_per_sample``, ``init_ref`` (ARPACK eigsh on the normalised Laplacian),
    ``sampler_key``: the host-side preparation.
  * ``layout_ref``: umap-learn's sequential SGD (stateful fp64 counters, Tausworthe sampler, in-place updates).
    It is the QUALITY reference: the product's Jacobi layout is a different trajectory.
  * ``epoch_ref``: the product's Jacobi epoch (csrc/umap.cu), vectorised, with a numpy Philox4x32-10.  It is the
    TIGHT reference of the kernel.  ``epoch_loop`` states the same epoch vertex by vertex.
  * ``trustworthiness``, ``knn_label_agreement``: layout quality scores.
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp

M32 = 0xFFFFFFFF
INT32_MIN = np.iinfo(np.int32).min + 1
INT32_MAX = np.iinfo(np.int32).max - 1

try:                                   # numba only speeds up layout_ref; the restatement is plain Python
    from numba import njit
except Exception:                      # pragma: no cover
    def njit(*a, **k):
        return (lambda f: f) if not (len(a) == 1 and callable(a[0])) else a[0]


# ---- host-side preparation (recalled) ------------------------------------------------------------------
def find_ab(spread, min_dist):
    from scipy.optimize import curve_fit
    x = np.linspace(0, spread * 3, 300)
    y = np.where(x < min_dist, 1.0, np.exp(-(x - min_dist) / spread))
    (a, b), _ = curve_fit(lambda x, a, b: 1.0 / (1.0 + a * x ** (2 * b)), x, y)
    return a, b


def n_epochs_for(n, maxiter):
    return (500 if n <= 10000 else 200) if not maxiter else int(maxiter)


def prune(graph, n_epochs):
    G = sp.coo_matrix(graph, dtype=np.float32)
    G.sum_duplicates()
    ne = n_epochs if n_epochs > 10 else (500 if G.shape[0] <= 10000 else 200)
    G.data[G.data < G.data.max() / float(ne)] = 0.0
    G.eliminate_zeros()
    return G.tocsr()


def epochs_per_sample(w):
    return (float(w.max()) / w.astype(np.float64)).astype(np.float32)


def _laplacian_eigs(W, k):
    from scipy.sparse.linalg import eigsh
    deg = np.asarray(W.sum(axis=0)).ravel()
    D = sp.diags(1.0 / np.sqrt(deg))
    L = sp.identity(W.shape[0]) - D @ W @ D
    ncv = max(2 * k + 1, int(np.sqrt(W.shape[0])))
    vals, vecs = eigsh(L, k, which="SM", ncv=ncv, tol=1e-8, v0=np.ones(W.shape[0]), maxiter=W.shape[0] * 5)
    order = np.argsort(vals)
    return vals[order], vecs[:, order]


def laplacian_eigs(W, k):
    """The k smallest eigenpairs (ascending) of I - D^-1/2 W D^-1/2 by ARPACK, as umap's spectral_layout asks."""
    return _laplacian_eigs(sp.csr_matrix(W, dtype=np.float64), k)


def init_ref(G, dim, init, rs):
    """umap's initial positions, rescaled to [0, 10] per axis (spectral: per component, meta positions +-e_i)."""
    from scipy.sparse.csgraph import connected_components
    n = G.shape[0]
    if isinstance(init, str) and init == "random":
        Y = rs.uniform(low=-10.0, high=10.0, size=(n, dim)).astype(np.float32)
    elif isinstance(init, str) and init == "spectral":
        nc, labels = connected_components(G)
        if nc == 1:
            Y = laplacian_eigs(G, dim + 1)[1][:, 1:]
        else:
            assert nc <= 2 * dim
            k = int(np.ceil(nc / 2.0))
            base = np.hstack([np.eye(k), np.zeros((k, dim - k))])
            meta = np.vstack([base, -base])[:nc]
            Y = np.zeros((n, dim))
            for lab in range(nc):
                mask = labels == lab
                sub = G.tocsr()[mask][:, mask]
                dist = np.linalg.norm(meta - meta[lab], axis=1)
                rng = dist[dist > 0].min() / 2.0
                if sub.shape[0] < 2 * dim or sub.shape[0] <= dim + 1:
                    Y[mask] = rs.uniform(low=-rng, high=rng, size=(sub.shape[0], dim)) + meta[lab]
                    continue
                e = laplacian_eigs(sub, dim + 1)[1][:, 1:]
                Y[mask] = e * (rng / np.abs(e).max()) + meta[lab]
        Y = (Y * (10.0 / np.abs(Y).max())).astype(np.float32) + \
            rs.normal(scale=0.0001, size=[n, dim]).astype(np.float32)
    else:
        Y = np.array(init, dtype=np.float32)
    return (10.0 * (Y - Y.min(0)) / (Y.max(0) - Y.min(0))).astype(np.float32)


def sampler_key(rs):
    return tuple(int(v) & M32 for v in rs.randint(INT32_MIN, INT32_MAX, 3).astype(np.int64))


# ---- Philox4x32-10 and the closed-form schedule ----------------------------------------------------------
def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Vectorised Philox4x32-10 over uint32 arrays; key (k0, k1) ints."""
    c = [np.asarray(v, dtype=np.uint64) & M32 for v in (c0, c1, c2, c3)]
    k0, k1 = int(k0) & M32, int(k1) & M32
    for r in range(10):
        if r:
            k0, k1 = (k0 + 0x9E3779B9) & M32, (k1 + 0xBB67AE85) & M32
        p0 = c[0] * np.uint64(0xD2511F53)
        p1 = c[2] * np.uint64(0xCD9E8D57)
        hi0, lo0, hi1, lo1 = p0 >> np.uint64(32), p0 & np.uint64(M32), p1 >> np.uint64(32), p1 & np.uint64(M32)
        c = [hi1 ^ c[1] ^ np.uint64(k0), lo1, hi0 ^ c[3] ^ np.uint64(k1), lo0]
    return [v.astype(np.uint32) for v in c]


def schedule(epoch, eps, rate):
    """(sampled, n_neg) per entry at ``epoch`` from eps (float32): csrc/umap.cu's closed form, in fp64."""
    e = np.asarray(eps, dtype=np.float32).astype(np.float64)
    m = np.floor(epoch / e)
    hit = (epoch >= 1) & (m > np.floor((epoch - 1) / e))
    if rate <= 0:
        return hit, np.zeros(e.shape, np.int64)
    c_now = np.floor(epoch * float(rate) / e) - 1
    n_prev = np.ceil((m - 1) * e)
    c_prev = np.where(m >= 2, np.floor(n_prev * float(rate) / e) - 1, 0)
    return hit, np.where(hit, np.maximum(c_now - c_prev, 0), 0).astype(np.int64)


def negative_vertices(entries, epoch, n_neg, key, n):
    """Vertex of every negative draw of ``entries`` (int64) with counts ``n_neg``: (owner entry per draw, vertex)."""
    s0, s1, s2 = key
    own = np.repeat(entries, n_neg)
    starts = np.repeat(np.cumsum(n_neg) - n_neg, n_neg)
    q = np.arange(own.size) - starts
    x = philox4x32_10(own & M32, ((own >> 32) & M32) ^ s2, np.full(own.size, epoch), q, s0, s1)[0]
    return own, (x.astype(np.int64) % n)


def _terms(diff, d2, a, b):
    p = np.power(d2, b, dtype=np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        gc = np.where(d2 > 0, -2.0 * a * b * (p / d2) / (a * p + 1.0), 0.0).astype(np.float32)
    return np.clip(gc[:, None] * diff, -4.0, 4.0)


def epoch_ref(G, eps, Y, epoch, n_epochs, a, b, gamma, alpha, rate, key):
    """One Jacobi epoch (csrc/umap.cu), vectorised.  G: pruned CSR (entries in row-major order), eps per entry."""
    n, dim = Y.shape
    Y = np.asarray(Y, dtype=np.float32)
    a, b, gamma = np.float32(a), np.float32(b), np.float32(gamma)
    rows = np.repeat(np.arange(n), np.diff(G.indptr))
    hit, n_neg = schedule(epoch, eps, rate)
    E = np.nonzero(hit)[0]
    h, t = rows[E], G.indices[E].astype(np.int64)
    acc = np.zeros((n, dim), dtype=np.float64)
    diff = Y[h] - Y[t]
    g = _terms(diff, (diff * diff).sum(1, dtype=np.float32), a, b)
    np.add.at(acc, h, g)
    np.add.at(acc, t, -g)
    own, k = negative_vertices(E.astype(np.int64), epoch, n_neg[E], key, n)
    hv = rows[own]
    keep = k != hv
    hv, k = hv[keep], k[keep]
    diff = Y[hv] - Y[k]
    d2 = (diff * diff).sum(1, dtype=np.float32)
    with np.errstate(divide="ignore"):
        gc = (2.0 * gamma * b / ((np.float32(0.001) + d2) * (a * np.power(d2, b, dtype=np.float32) + 1.0)))
    rep = np.where(d2[:, None] > 0, np.clip(gc[:, None] * diff, -4.0, 4.0), 4.0)
    np.add.at(acc, hv, rep)
    alpha_n = alpha * (1.0 - float(epoch) / float(n_epochs))
    return (Y + alpha_n * acc).astype(np.float32)


def epoch_loop(G, eps, Y, epoch, n_epochs, a, b, gamma, alpha, rate, key):
    """``epoch_ref`` stated vertex by vertex: each vertex sums its head entries (attraction + negatives), then its
    tail entries (attraction from the other end), from the positions of the previous epoch."""
    n, dim = Y.shape
    T = sp.csr_matrix((np.arange(G.nnz, dtype=np.float64) + 1, G.indices, G.indptr), shape=G.shape).T.tocsr()
    hit, n_neg = schedule(epoch, eps, rate)
    alpha_n = alpha * (1.0 - float(epoch) / float(n_epochs))
    out = np.empty_like(Y)

    def attract(yi, yj):
        d = yi.astype(np.float64) - yj
        d2 = float(d @ d)
        gc = -2.0 * a * b * d2 ** (b - 1.0) / (a * d2 ** b + 1.0) if d2 > 0 else 0.0
        return np.clip(gc * d, -4.0, 4.0)

    for i in range(n):
        acc = np.zeros(dim)
        for e in range(G.indptr[i], G.indptr[i + 1]):
            if not hit[e]:
                continue
            acc += attract(Y[i], Y[G.indices[e]])
            for q in range(int(n_neg[e])):
                x = philox4x32_10([e & M32], [(e >> 32) ^ key[2]], [epoch], [q], key[0], key[1])[0][0]
                k = int(x) % n
                if k == i:
                    continue
                d = Y[i].astype(np.float64) - Y[k]
                d2 = float(d @ d)
                if d2 > 0:
                    acc += np.clip(2.0 * gamma * b / ((0.001 + d2) * (a * d2 ** b + 1.0)) * d, -4.0, 4.0)
                else:
                    acc += 4.0
        for p in range(T.indptr[i], T.indptr[i + 1]):
            e = int(T.data[p]) - 1
            if hit[e]:
                acc += attract(Y[i], Y[T.indices[p]])
        out[i] = Y[i] + alpha_n * acc
    return out


# ---- umap-learn's sequential SGD (recalled) --------------------------------------------------------------
@njit(cache=False)
def _tau_rand_int(state):
    state[0] = (((state[0] & 4294967294) << 12) & 0xFFFFFFFF) ^ ((((state[0] << 13) & 0xFFFFFFFF) ^ state[0]) >> 19)
    state[1] = (((state[1] & 4294967288) << 4) & 0xFFFFFFFF) ^ ((((state[1] << 2) & 0xFFFFFFFF) ^ state[1]) >> 25)
    state[2] = (((state[2] & 4294967280) << 17) & 0xFFFFFFFF) ^ ((((state[2] << 3) & 0xFFFFFFFF) ^ state[2]) >> 11)
    return state[0] ^ state[1] ^ state[2]


@njit(cache=False)
def _clip(v):
    return 4.0 if v > 4.0 else (-4.0 if v < -4.0 else v)


@njit(cache=False)
def _optimize(Y, head, tail, n, eps, a, b, rng_state, gamma, initial_alpha, rate, n_epochs):
    dim = Y.shape[1]
    next_sample = eps.copy()
    eps_neg = eps / rate
    next_neg = eps_neg.copy()
    alpha = initial_alpha
    for ep in range(n_epochs):
        for i in range(eps.shape[0]):
            if next_sample[i] <= ep:
                j = head[i]
                k = tail[i]
                d2 = 0.0
                for d in range(dim):
                    d2 += (Y[j, d] - Y[k, d]) ** 2
                gc = 0.0
                if d2 > 0.0:
                    gc = -2.0 * a * b * d2 ** (b - 1.0) / (a * d2 ** b + 1.0)
                for d in range(dim):
                    g = _clip(gc * (Y[j, d] - Y[k, d]))
                    Y[j, d] += g * alpha
                    Y[k, d] += -g * alpha
                next_sample[i] += eps[i]
                n_neg = int((ep - next_neg[i]) / eps_neg[i])
                for p in range(n_neg):
                    k = _tau_rand_int(rng_state) % n
                    d2 = 0.0
                    for d in range(dim):
                        d2 += (Y[j, d] - Y[k, d]) ** 2
                    if d2 > 0.0:
                        gc = 2.0 * gamma * b / ((0.001 + d2) * (a * d2 ** b + 1.0))
                    elif j == k:
                        continue
                    else:
                        gc = 0.0
                    for d in range(dim):
                        g = _clip(gc * (Y[j, d] - Y[k, d])) if gc > 0.0 else 4.0
                        Y[j, d] += g * alpha
                next_neg[i] += n_neg * eps_neg[i]
        alpha = initial_alpha * (1.0 - float(ep) / float(n_epochs))
    return Y


def layout_ref(graph, *, n_components=2, maxiter=None, alpha=1.0, gamma=1.0, negative_sample_rate=5,
               init_pos="spectral", random_state=42, a=None, b=None, min_dist=0.5, spread=1.0):
    """umap-learn's layout of ``graph`` as scanpy runs it (sequential, seeded) -> float32 [n x n_components]."""
    if a is None or b is None:
        a, b = find_ab(spread, min_dist)
    n_epochs = n_epochs_for(graph.shape[0], maxiter)
    G = prune(graph, n_epochs)
    rs = np.random.RandomState(random_state)
    Y = init_ref(G, n_components, init_pos, rs)
    rng_state = rs.randint(INT32_MIN, INT32_MAX, 3).astype(np.int64)
    C = G.tocoo()
    w = C.data.astype(np.float64)
    eps = float(n_epochs) / (float(n_epochs) * (w / w.max()))        # umap's make_epochs_per_sample
    return _optimize(Y, C.row.astype(np.int64), C.col.astype(np.int64), G.shape[0], eps, float(a), float(b),
                     rng_state, float(gamma), float(alpha), float(negative_sample_rate), n_epochs)


# ---- quality scores -------------------------------------------------------------------------------------
def _sq_dists(X):
    X = np.asarray(X, dtype=np.float64)
    s = (X * X).sum(1)
    D = s[:, None] + s[None, :] - 2.0 * X @ X.T
    np.fill_diagonal(D, np.inf)
    return D


def trustworthiness(X, Y, k=15):
    """sklearn.manifold.trustworthiness (Venna & Kaski): penalises layout neighbours that are far in X."""
    n = X.shape[0]
    DX, DY = _sq_dists(X), _sq_dists(Y)
    order = np.argsort(DX, axis=1, kind="stable")
    rank = np.empty((n, n), dtype=np.int64)
    rank[np.arange(n)[:, None], order] = np.arange(1, n + 1)[None, :]
    nnY = np.argsort(DY, axis=1, kind="stable")[:, :k]
    r = rank[np.arange(n)[:, None], nnY] - k
    return 1.0 - 2.0 / (n * k * (2.0 * n - 3.0 * k - 1.0)) * float(np.maximum(r, 0).sum())


def knn_label_agreement(Y, labels, k=15):
    """Mean fraction of each point's k nearest layout neighbours that carry its label."""
    nn = np.argsort(_sq_dists(Y), axis=1, kind="stable")[:, :k]
    return float((labels[nn] == labels[:, None]).mean())


def planted_graph(n=1500, n_clusters=6, dim=10, k=15, spread=2.2, seed=0):
    """Gaussian clusters in ``dim`` dimensions -> (representation, labels, umap connectivities of the exact kNN)."""
    from oracle._third_party import nearest_neighbors, umap_connectivities
    rng = np.random.default_rng(seed)
    centers = rng.normal(size=(n_clusters, dim)) * spread
    labels = rng.integers(0, n_clusters, n)
    X = (centers[labels] + rng.normal(size=(n, dim))).astype(np.float32)
    idx, dist, _ = nearest_neighbors(X, k, "euclidean")
    return X, labels, umap_connectivities(idx, dist, n_obs=n, n_neighbors=k).astype(np.float32)
