"""Numpy-only restatement of DSB (reference muon/_prot/preproc.py:161-218) for the tests and the benchmark.

Steps 2-5 of the reference -- scaling by the empty droplets, the two per-cell two-component Gaussian mixtures
(``tied`` and ``full`` covariance, sklearn's ``GaussianMixture`` protocol with ``init_params="random"``), the
regression on the background covariate and the quantile clip -- written out in float64 numpy, vectorised over
cells.  Unlike the reference it also returns what the per-cell fits found: ``bgmean``, the chosen model and the
iteration counts.  It needs neither sklearn nor the reference, so it runs wherever the tests run.

The mixture arithmetic follows sklearn 1.9 (``sklearn/mixture/_base.py::fit``, ``_gaussian_mixture.py``):

- responsibilities start as ``U / U.sum(1)`` with ``U = random_state.uniform(size=(P, 2))``, one draw per fit;
- M-step: ``nk = sum r + 10 eps``, ``mu = sum r x / nk``, tied ``var = (x.x - sum nk mu^2) / sum nk + reg``,
  full ``var_k = sum r_k (x - mu_k)^2 / nk + reg``; weights ``nk / P`` after the first M-step and
  ``nk / sum nk`` after the others;
- E-step: ``log N(x | mu_k, var_k) + log w_k`` with the precision ``1 / sqrt(var)``, then sklearn's
  ``_logsumexp`` (the largest term factored out, ``log1p`` of the rest);
- up to ``max_iter`` rounds of E-step, M-step, ``lower bound = mean(logsumexp)``, stopping when the change is
  below ``tol``; ``bic = -2 P mean(logsumexp) + p log P`` with p = 4 (tied) or 5 (full).
"""
from __future__ import annotations

import numpy as np

REG_COVAR = 1e-6
TOL = 1e-3
MAX_ITER = 100
EPS10 = 10 * np.finfo(np.float64).eps
LOG_2PI = np.log(2 * np.pi)
LOG_2 = np.log(2.0)
MODEL_TIED, MODEL_FULL = 0, 1


def scaled_dtype(dtype, pseudocount):
    """dtype of ``np.log(X + pseudocount)`` for counts of ``dtype`` (reference preproc.py:161-170)."""
    return np.log(np.zeros(1, dtype=dtype) + pseudocount).dtype


def _dense(X):
    import scipy.sparse as sp
    return X.toarray() if sp.issparse(X) else np.asarray(X)


def scale(cells, empty, pseudocount=10, scale_factor="standardize"):
    """Step 2 (preproc.py:161-177): log, centre (and standardise) by the empty droplets, back to the input dtype."""
    empty_scaled = np.log(_dense(empty) + pseudocount)
    cells_scaled = np.log(_dense(cells) + pseudocount)
    dt = cells_scaled.dtype
    cells_scaled = cells_scaled - empty_scaled.mean(axis=0, dtype=np.float64)
    if scale_factor == "standardize":
        cells_scaled /= empty_scaled.std(axis=0, ddof=1, dtype=np.float64)
    if dt.kind == "f":
        cells_scaled = cells_scaled.astype(dt, copy=False)
    return cells_scaled


def _lse2(a, b):
    hi = np.maximum(a, b)
    lo = np.minimum(a, b)
    with np.errstate(under="ignore"):
        one = np.log1p(np.exp(lo - hi)) + 0.0 + hi
    return np.where(a == b, (0.0 + LOG_2) + hi, one)


def _m_step(X, R, tied, first):
    P = X.shape[1]
    nk = R.sum(axis=1) + EPS10                                  # (n, 2)
    mu = np.einsum("npk,np->nk", R, X) / nk
    if tied:
        var = ((X * X).sum(axis=1) - (nk * mu * mu).sum(axis=1)) / nk.sum(axis=1) + REG_COVAR
        var = np.repeat(var[:, None], 2, axis=1)
    else:
        d = X[:, :, None] - mu[:, None, :]
        var = (R * d * d).sum(axis=1) / nk + REG_COVAR
    w = nk / P if first else nk / nk.sum(axis=1, keepdims=True)
    return w, mu, var


def _e_step(X, w, mu, var):
    pc = 1.0 / np.sqrt(var)
    y = X[:, :, None] * pc[:, None, :] - (mu * pc)[:, None, :]
    wlp = (-0.5 * (LOG_2PI + y * y) + np.log(pc)[:, None, :]) + np.log(w)[:, None, :]
    lse = _lse2(wlp[..., 0], wlp[..., 1])
    with np.errstate(under="ignore"):
        R = np.exp(wlp - lse[..., None])
    return lse.mean(axis=1), R


def fit_mixtures(X, U, tied):
    """One two-component mixture per row of ``X`` (n x P, float64) from the initial draws ``U`` (n x P x 2).
    Returns (means (n, 2), bic (n,), n_iter (n,), converged (n,))."""
    X = np.asarray(X, dtype=np.float64)
    n, P = X.shape
    R = U / U.sum(axis=2, keepdims=True)
    w, mu, var = _m_step(X, R, tied, first=True)
    lb = np.full(n, -np.inf)
    n_iter = np.zeros(n, dtype=np.int32)
    conv = np.zeros(n, dtype=bool)
    act = np.arange(n)
    for it in range(1, MAX_ITER + 1):
        if act.size == 0:
            break
        Xa = X[act]
        lpn, R = _e_step(Xa, w[act], mu[act], var[act])
        wa, ma, va = _m_step(Xa, R, tied, first=False)
        w[act], mu[act], var[act] = wa, ma, va
        prev = lb[act]
        lb[act] = lpn
        n_iter[act] = it
        done = np.abs(lpn - prev) < TOL
        conv[act[done]] = True
        act = act[~done]
    lpn, _ = _e_step(X, w, mu, var)
    p = 4 if tied else 5
    bic = -2 * lpn * P + p * np.log(P)
    return mu, bic, n_iter, conv


def initial_draws(n, P, random_state):
    """The uniform draws the reference's fits consume, shaped (n, 2, P, 2): [cell, model (tied, full)].
    An int seeds every fit with the same draw; a RandomState (or None: numpy's global generator) is consumed
    in the order cell 0 tied, cell 0 full, cell 1 tied, ... (``check_random_state`` in every ``fit``)."""
    import numbers
    if isinstance(random_state, numbers.Integral) and not isinstance(random_state, bool):
        U = np.random.RandomState(random_state).uniform(size=(P, 2))
        return np.broadcast_to(U, (n, 2, P, 2))
    rs = np.random.mtrand._rand if random_state is None else random_state
    return rs.uniform(size=(n, 2, P, 2))


def background_means(cells_scaled, random_state=None):
    """Step 3 (preproc.py:179-198): per-cell ``bgmean`` in the dtype of ``cells_scaled`` and what the fits did."""
    n, P = cells_scaled.shape
    X = cells_scaled.astype(np.float64)
    U = initial_draws(n, P, random_state)
    mt, bt, it_t, cv_t = fit_mixtures(X, np.asarray(U[:, 0]), tied=True)
    mf, bf, it_f, cv_f = fit_mixtures(X, np.asarray(U[:, 1]), tied=False)
    model = np.where(bt < bf, MODEL_TIED, MODEL_FULL).astype(np.int8)
    bg = np.where(model == MODEL_TIED, mt.min(axis=1), mf.min(axis=1))
    return {"bgmean": bg.astype(cells_scaled.dtype), "model": model,
            "n_iter": np.stack([it_t, it_f], axis=1), "converged": np.stack([cv_t, cv_f], axis=1)}


def denoise(cells_scaled, bgmean, ctrl_idx=None):
    """Step 4 (preproc.py:200-214): subtract the least-squares fit on the covariate (bgmean, or the first
    principal component of [isotype controls | bgmean]) without its intercept, in float64.

    The covariate is centred in both cases: the principal component is, and ``LinearRegression(copy_X=False)``
    centres ``bgmean`` in place during ``fit``, before the reference's ``predict``."""
    y = cells_scaled.astype(np.float64)
    if ctrl_idx is None:
        c = bgmean.astype(np.float64)
        c = c - c.mean()
    else:
        Z = np.hstack((y[:, ctrl_idx], bgmean.astype(np.float64)[:, None]))
        Zc = Z - Z.mean(axis=0)
        _, vecs = np.linalg.eigh(Zc.T @ Zc)
        c = Zc @ vecs[:, -1]
    beta = (c @ (y - y.mean(axis=0))) / (c @ c)
    out = y - np.outer(c, beta)
    return out.astype(cells_scaled.dtype, copy=False)


def dsb_ref(cells, empty, pseudocount=10, denoise_counts=True, ctrl_idx=None, scale_factor="standardize",
            quantile_clip=None, random_state=None):
    """DSB steps 2-5 on count matrices ``cells`` and ``empty`` (dense or scipy sparse).  ``ctrl_idx`` are the
    column indices of the isotype controls present; ``quantile_clip`` a pair of quantiles, or None for no clip.
    Returns a dict with ``out`` and, when denoising, ``bgmean``, ``model``, ``n_iter`` and ``converged``."""
    y = scale(cells, empty, pseudocount, scale_factor)
    res = {}
    if denoise_counts:
        res = background_means(y, random_state)
        y = denoise(y, res["bgmean"], ctrl_idx)
    if quantile_clip is not None:
        q = np.quantile(y, np.asarray(quantile_clip))
        np.clip(y, a_min=q.min(), a_max=q.max(), out=y)
    res["out"] = y
    return res


def synth_citeseq(n_cells, n_empty, n_prot, seed=0, dtype=np.float32, empty_density=0.1, chunk=1 << 17):
    """CITE-seq-like protein counts: (cells dense (n_cells, n_prot), empties CSR (n_empty, n_prot)).
    Every protein has an ambient level; each cell scales it by its own factor and expresses ~30 % of the
    proteins well above it.  Empty droplets hold a sparse sample of the ambient counts."""
    import scipy.sparse as sp
    rng = np.random.default_rng(seed)
    ambient = rng.gamma(2.0, 2.0, n_prot)
    cells = np.empty((n_cells, n_prot), dtype=dtype)
    for s in range(0, n_cells, chunk):
        e = min(n_cells, s + chunk)
        lam = ambient * rng.gamma(5.0, 0.2, (e - s, 1))
        lam = lam + (rng.random((e - s, n_prot)) < 0.3) * rng.gamma(2.0, 30.0, (e - s, n_prot))
        cells[s:e] = rng.poisson(lam)
    parts = []
    for s in range(0, n_empty, chunk):
        e = min(n_empty, s + chunk)
        mask = rng.random((e - s, n_prot), dtype=np.float32) < empty_density
        r, c = np.nonzero(mask)
        v = (1 + rng.poisson(0.5 * ambient[c])).astype(dtype)
        parts.append(sp.csr_matrix((v, c.astype(np.int32), np.concatenate(([0], np.cumsum(mask.sum(1))))),
                                   shape=(e - s, n_prot)))
    empty = sp.vstack(parts, format="csr") if parts else sp.csr_matrix((0, n_prot), dtype=dtype)
    return cells, empty


def load_reference_dsb():
    """Return the reference's own ``dsb`` (muon/_prot/preproc.py:17) executed in place through the container
    stubs of ``oracle._refload``; needs the reference checkout and scikit-learn."""
    from . import _refload
    import sys
    if not _refload.reference_available():
        raise FileNotFoundError(_refload.REF_ROOT)
    _refload._install_stubs()
    m = sys.modules.get("_refmuon_prot_preproc")
    if m is None:
        m = _refload._load("muon/_prot/preproc.py", "_refmuon_prot_preproc")
    return m.dsb
