"""Float64 numpy restatement of scOpen's imputation (muon.atac.pp.scopen, muon/_atac/preproc.py:155-236) in the
sparse-pattern form, and the reference run through a ``scopen.MF`` stand-in built on it.

The reference factorises X [peaks x cells], X[p, c] = s_c where count(c, p) > 0, with scOpen's fork of sklearn's
coordinate-descent NMF.  Here both products of an iteration are scipy-sparse products over the pattern, and the
coordinate-descent sweep is vectorised over rows (rows are independent; components run in order), with every
update projected onto [0, ``upper``]; ``upper`` = inf is sklearn's ``_fit_coordinate_descent`` with
l2_reg_W = l2_reg_H = alpha.  The init is NNDSVD (sklearn's ``_initialize_nmf``) from the exact SVD.

``load_reference_scopen`` returns the reference's own ``scopen``, executed unmodified from its source file, with
``scopen.MF.non_negative_factorization`` replaced by ``non_negative_factorization`` below (exact-SVD NNDSVD, bound
1, tol 1e-4).  Test infrastructure only: nothing on the product path imports this module.
"""
from __future__ import annotations

import ast
import os
import sys
import types
import warnings
from typing import Union

import numpy as np
import scipy.sparse as sp

TOL = 1e-4
EPS = 1e-6


def pattern_of(X):
    """The cells x peaks CSR of entries > 0 (duplicates summed first) with float64 ones, and the positives per cell."""
    X = sp.csr_matrix(X, dtype=np.float64, copy=True)
    X.sum_duplicates()
    X.data = (X.data > 0).astype(np.float64)
    X.eliminate_zeros()
    X.sort_indices()
    return X, np.asarray(X.sum(axis=1)).ravel()


def scale_of(counts, min_rho=0.0, max_rho=0.5):
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.log10(np.asarray(counts, dtype=np.float64))
        rho = min_rho + (max_rho - min_rho) * (r.max() - r) / (r.max() - r.min())
        return 1 / (1 - rho)


def dense_of(P, s):
    """X [peaks x cells] as the reference builds it."""
    return np.asarray(P.T.toarray() * s[None, :])


def exact_svd(X, k):
    """Top-k SVD of the dense X: (U [m x k], S [k], V [k x n])."""
    U, S, V = np.linalg.svd(np.asarray(X, dtype=np.float64), full_matrices=False)
    return U[:, :k], S[:k], V[:k]


def nndsvd(U, S, V, eps=EPS):
    """sklearn's ``_initialize_nmf(init="nndsvd")`` given the SVD."""
    W = np.zeros_like(U)
    H = np.zeros_like(V)
    W[:, 0] = np.sqrt(S[0]) * np.abs(U[:, 0])
    H[0, :] = np.sqrt(S[0]) * np.abs(V[0, :])
    for j in range(1, U.shape[1]):
        x, y = U[:, j], V[j, :]
        x_p, y_p = np.maximum(x, 0), np.maximum(y, 0)
        x_n, y_n = np.abs(np.minimum(x, 0)), np.abs(np.minimum(y, 0))
        x_p_nrm, y_p_nrm = np.linalg.norm(x_p), np.linalg.norm(y_p)
        x_n_nrm, y_n_nrm = np.linalg.norm(x_n), np.linalg.norm(y_n)
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


def cd_sweep(W, HHt, XHt, upper=np.inf):
    """sklearn's ``_update_cdnmf_fast`` (no shuffle) over all rows of W in place, each update projected onto
    [0, upper]; returns the violation."""
    k = W.shape[1]
    violation = 0.0
    for t in range(k):
        grad = W @ HHt[t] - XHt[:, t]
        w = W[:, t]
        pg = np.where(w == 0, np.minimum(0.0, grad), grad)
        violation += np.abs(pg).sum()
        hess = HHt[t, t]
        if hess != 0:
            W[:, t] = np.minimum(np.maximum(w - grad / hess, 0.0), upper)
    return violation


class PatternMatrix:
    """X [peaks x cells] = P^T diag(s) as the two products the fit needs."""

    def __init__(self, P, s):
        self.P = sp.csr_matrix(P)
        self.PT = self.P.T.tocsr()
        self.s = np.asarray(s, dtype=np.float64)

    def x_ht(self, Ht):                 # X Ht  [m x k]
        return self.PT @ (self.s[:, None] * Ht)

    def xt_w(self, W):                  # X^T W [n x k]
        return self.s[:, None] * (self.P @ W)


def w_step(X, W, Ht, alpha, upper):
    HHt = Ht.T @ Ht + alpha * np.eye(W.shape[1])
    return cd_sweep(W, HHt, X.x_ht(Ht), upper)


def h_step(X, W, Ht, alpha, upper):
    WtW = W.T @ W + alpha * np.eye(W.shape[1])
    return cd_sweep(Ht, WtW, X.xt_w(W), upper)


def fit(X, W0, H0, alpha=1.0, max_iter=500, tol=TOL, upper=np.inf, verbose=False):
    """The coordinate-descent loop of sklearn's ``_fit_coordinate_descent`` on ``PatternMatrix`` X.  Returns
    (W, H, n_iter, ratios): ``ratios`` the violation / violation_init of every iteration."""
    W = np.array(W0, dtype=np.float64, order="C")
    Ht = np.array(np.asarray(H0, dtype=np.float64).T, order="C")
    ratios = []
    n_iter = 0
    for n_iter in range(1, max_iter + 1):
        violation = 0.0
        violation += w_step(X, W, Ht, alpha, upper)
        violation += h_step(X, W, Ht, alpha, upper)
        if n_iter == 1:
            violation_init = violation
        if violation_init == 0:
            break
        ratios.append(violation / violation_init)
        if verbose:
            print("violation:", violation / violation_init)
        if violation / violation_init <= tol:
            if verbose:
                print("Converged at iteration", n_iter + 1)
            break
    return W, Ht.T.copy(), n_iter, ratios


def objective(X, W, H, alpha):
    """0.5 ||X - W H||_F^2 + 0.5 alpha (||W||^2 + ||H||^2), with the dense X."""
    R = X - W @ H
    return 0.5 * np.sum(R * R) + 0.5 * alpha * (np.sum(W * W) + np.sum(H * H))


def scopen_ref(counts, n_components=30, max_iter=500, min_rho=0.0, max_rho=0.5, alpha=1.0, upper=1.0, init=None):
    """The whole computation on a cells x peaks input: dict with the pattern, scale, init, W, H, n_iter, ratios, M."""
    P, c = pattern_of(counts)
    s = scale_of(c, min_rho, max_rho)
    X = PatternMatrix(P, s)
    if init is None:
        init = nndsvd(*exact_svd(dense_of(P, s), n_components))
    W, H, n_iter, ratios = fit(X, init[0], init[1], alpha, max_iter, TOL, upper)
    M = np.clip(W @ H, 0, 1)
    return {"P": P, "s": s, "W0": init[0], "H0": init[1], "W": W, "H": H, "n_iter": n_iter, "ratios": ratios, "M": M}


# ---- the reference with a scopen.MF stand-in --------------------------------------------------------------------
def non_negative_factorization(X, W=None, H=None, n_components=None, init="nndsvd", update_H=True, solver="cd",
                               beta_loss="frobenius", tol=TOL, max_iter=200, alpha=0.0, l1_ratio=0.0,
                               regularization="both", random_state=None, verbose=0, shuffle=False):
    """scOpen's ``non_negative_factorization`` as this project states it: exact-SVD NNDSVD, coordinate descent with
    every update projected onto [0, 1], l2_reg_W = l2_reg_H = alpha.  X is the reference's dense peaks x cells
    matrix; its pattern and per-cell scale are read back from it."""
    from sklearn.exceptions import ConvergenceWarning
    X = np.asarray(X, dtype=np.float64)
    if not np.all(np.isfinite(X)):
        raise ValueError("Input contains NaN, infinity or a value too large for dtype('float64').")
    P = sp.csr_matrix(X.T != 0, dtype=np.float64)
    s = X.max(axis=0)
    W0, H0 = nndsvd(*exact_svd(X, n_components))
    W, H, n_iter, _ = fit(PatternMatrix(P, s), W0, H0, alpha, max_iter, tol, 1.0, verbose=bool(verbose))
    if n_iter == max_iter and tol > 0:
        warnings.warn("Maximum number of iterations %d reached. Increase it to improve convergence." % max_iter,
                      ConvergenceWarning)
    return W, H, n_iter


def _reference_function(name):
    from oracle._refload import REF_ROOT
    path = os.path.join(REF_ROOT, "muon", "_atac", "preproc.py")
    tree = ast.parse(open(path).read())
    (fn,) = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == name]
    return fn, path


def load_reference_scopen():
    """The reference's own ``scopen``; its ``from scopen.MF import non_negative_factorization`` imports the stand-in
    above."""
    from muon_b200 import SimpleAnnData, SimpleMuData
    if "scopen.MF" not in sys.modules:
        pkg = types.ModuleType("scopen")
        pkg.__path__ = []
        mf = types.ModuleType("scopen.MF")
        mf.non_negative_factorization = non_negative_factorization
        pkg.MF = mf
        sys.modules["scopen"], sys.modules["scopen.MF"] = pkg, mf
    fn, path = _reference_function("scopen")
    g = {"np": np, "Union": Union, "AnnData": SimpleAnnData, "MuData": SimpleMuData,
         "issparse": sp.issparse}
    exec(compile(ast.Module([fn], []), path, "exec"), g)
    return g["scopen"]


def reference_signature():
    fn, _ = _reference_function("scopen")
    a = fn.args
    return {"params": [x.arg for x in a.args], "defaults": [ast.unparse(d) for d in a.defaults]}
