"""Float64 numpy restatement of sklearn 1.9's ``FastICA.fit_transform``, the arithmetic behind ``muon.tl.ica``
(muon/_core/tools.py:1365-1386).

Every step follows sklearn's order: centring, whitening by the SVD of the centred data (or ``eigh`` of its Gram with
the small-value clamp), the sign fix ``u *= sign(u[0])``, X1 = sqrt(n) K Xc^T, the parallel iteration with symmetric
decorrelation or the deflation iteration with Gram-Schmidt, the sources and the unit-variance rescale.  Everything
runs in float64 whatever the input dtype.  ``lims`` records the stopping value of every iteration, so that a fixture
can tell whether its iteration count depends on rounding.
"""
from __future__ import annotations

import numpy as np
from scipy import linalg


def contrast(fun, alpha):
    """(g, per-row mean of g') of sklearn's named contrast functions, on a 2-D array of projections."""
    if fun == "logcosh":
        def g(x):
            gx = np.tanh(alpha * x)
            return gx, (alpha * (1 - gx ** 2)).mean(axis=-1)
    elif fun == "exp":
        def g(x):
            e = np.exp(-(x ** 2) / 2)
            return x * e, ((1 - x ** 2) * e).mean(axis=-1)
    elif fun == "cube":
        def g(x):
            return x ** 3, (3 * x ** 2).mean(axis=-1)
    else:
        raise ValueError(fun)
    return g


def sym_decorrelation(W):
    """(W W^T)^(-1/2) W."""
    s, u = linalg.eigh(W @ W.T)
    s = np.clip(s, a_min=np.finfo(W.dtype).tiny, a_max=None)
    return np.linalg.multi_dot([u * (1.0 / np.sqrt(s)), u.T, W])


def ica_par(X1, tol, g, max_iter, w_init):
    W = sym_decorrelation(w_init)
    n = float(X1.shape[1])
    lims = []
    converged = False
    for ii in range(max_iter):
        gwtx, g_wtx = g(W @ X1)
        W1 = sym_decorrelation(gwtx @ X1.T / n - g_wtx[:, None] * W)
        lim = max(abs(abs(np.einsum("ij,ij->i", W1, W)) - 1))
        lims.append(lim)
        W = W1
        if lim < tol:
            converged = True
            break
    return W, ii + 1, lims, converged


def ica_def(X1, tol, g, max_iter, w_init):
    k = w_init.shape[0]
    W = np.zeros((k, k))
    n_iter, lims = [], []
    for j in range(k):
        w = w_init[j, :].copy()
        w /= np.sqrt((w ** 2).sum())
        for i in range(max_iter):
            gwtx, g_wtx = g((w @ X1)[None, :])
            w1 = (X1 * gwtx[0]).mean(axis=1) - g_wtx[0] * w
            w1 -= np.linalg.multi_dot([w1, W[:j].T, W[:j]])
            w1 /= np.sqrt((w1 ** 2).sum())
            lim = np.abs(np.abs((w1 * w).sum()) - 1)
            lims.append(lim)
            w = w1
            if lim < tol:
                break
        n_iter.append(i + 1)
        W[j, :] = w
    return W, max(n_iter), lims, True


def whitening(Xc, k, solver, eps_dtype=np.float64):
    """(K [k x p], small-value flag) of the centred data Xc [n x p] as sklearn computes it."""
    small = False
    if solver == "eigh":
        d, u = linalg.eigh(Xc.T @ Xc)
        order = np.argsort(d)[::-1]
        eps = np.finfo(eps_dtype).eps * 10
        small = bool(np.any(d < eps))
        d[d < eps] = eps
        d = np.sqrt(d)
        d, u = d[order], u[:, order]
    else:
        u, d = linalg.svd(Xc.T, full_matrices=False, check_finite=False)[:2]
    u = u * np.sign(u[0])
    return (u / d).T[:k], small


def fastica_ref(X, n_components=None, *, algorithm="parallel", whiten="unit-variance", fun="logcosh", fun_args=None,
                max_iter=200, tol=1e-4, w_init=None, whiten_solver="svd", random_state=None):
    """The outputs of ``FastICA(...).fit_transform(X)`` in float64: a dict with ``sources``, ``n_iter``,
    ``components``, ``mixing``, ``mean``, ``whitening`` (None without whitening), ``unmixing``, ``lims`` and
    ``converged``.  ``random_state`` is None, an int or a RandomState, consumed as sklearn consumes it."""
    Xin = np.asarray(X)
    eps_dtype = Xin.dtype if Xin.dtype in (np.float32, np.float64) else np.float64
    X = np.asarray(Xin, dtype=np.float64)
    n, p = X.shape
    alpha = (fun_args or {}).get("alpha", 1.0)
    g = contrast(fun, alpha)
    if random_state is None:
        rs = np.random.mtrand._rand
    elif isinstance(random_state, np.random.RandomState):
        rs = random_state
    else:
        rs = np.random.RandomState(random_state)
    k = n_components
    if not whiten:
        k = None
    if k is None:
        k = min(n, p)
    k = min(k, min(n, p))
    K = mean = None
    if whiten:
        mean = X.mean(axis=0)
        Xc = X - mean
        K, _ = whitening(Xc, k, whiten_solver, eps_dtype)
        X1 = (K @ Xc.T) * np.sqrt(n)
    else:
        X1 = X.T
    if w_init is None:
        w_init = np.asarray(rs.normal(size=(k, k)), dtype=eps_dtype).astype(np.float64)
    else:
        w_init = np.asarray(w_init, dtype=np.float64)
    run = ica_par if algorithm == "parallel" else ica_def
    W, n_iter, lims, converged = run(X1, tol, g, max_iter, w_init)
    if whiten:
        S = np.linalg.multi_dot([W, K, Xc.T]).T
    else:
        S = (W @ X.T).T
    if whiten:
        if whiten == "unit-variance":
            S_std = np.std(S, axis=0, keepdims=True)
            S /= S_std
            W /= S_std.T
        components = W @ K
    else:
        components = W
    return {"sources": S, "n_iter": n_iter, "components": components, "mixing": linalg.pinv(components),
            "mean": mean, "whitening": K, "unmixing": W, "lims": lims, "converged": converged}


def match_sources(S, T):
    """The worst recovered planted source: min over the columns T_j of T [n x m] of max_i |corr(S_i, T_j)|."""
    S = (S - S.mean(0)) / S.std(0)
    T = (T - T.mean(0)) / T.std(0)
    C = np.abs(S.T @ T) / S.shape[0]
    return float(C.max(axis=0).min())
