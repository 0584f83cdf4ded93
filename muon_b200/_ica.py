"""``mu.tl.ica`` -- independent component analysis of an ``obsm`` representation: sklearn's FastICA on the GPU.

The reference (muon/_core/tools.py:1365-1386) hands ``data.obsm[basis]`` to ``sklearn.decomposition.FastICA`` and
stores ``fit_transform``'s sources in ``obsm["X_ica"]``.  Here ``FastICA._fit_transform`` (sklearn 1.9) is restated
step by step.  The passes over the n cells run in csrc/ica.cu; everything k x k or p x p stays on the host in float64:

  * moments  column means and the centred p x p Gram X_c^T X_c, float64 sums in a fixed order;
  * host     the whitening: eigh of the Gram, d = sqrt(eigenvalues) in descending order, ``u *= sign(u[0])``,
             K = (u / d)^T[:k];
  * project  X1 = sqrt(n) K (x - mean) per cell into an n x k float64 buffer (the raw X widened with whiten=False);
  * step     one fixed-point pass: sum_i g(W x1_i) x1_i^T and sum_i g'(W x1_i), r = k rows of W (parallel) or r = 1
             (deflation); the host finishes the update (symmetric decorrelation or Gram-Schmidt) and the stopping
             value, which is one (k^2 + k)-double copy per iteration;
  * sources  S = W x1 / sqrt(n) (or W x) in the output dtype, with the column std of the unit-variance rescale and of
             ``scale`` computed on the device and applied in the reference's order.

Divergences (DESIGN.md section 8): every sum is float64, also for float32 input, where sklearn works in float32; the
"svd" whitening is computed from the float64 Gram, so it agrees with LAPACK's SVD to float64 rounding x cond(X)^2, and
a Gram eigenvalue below 10 eps(float64) lambda_max is clamped there with a warning; a callable ``fun`` raises
NotImplementedError.  More than MUB_ICA_MAX_DIM = 128 features, and an X1 plus partials beyond free device memory,
raise NotImplementedError before any device work.  No float atomics: two calls return the same bits.
"""
from __future__ import annotations

import numbers
import warnings

import numpy as np

from ._lib import ICA_CUBE, ICA_EXP, ICA_LOGCOSH, ICA_MAX_DIM
from .prot.pp import ConvergenceWarning

FUNS = {"logcosh": ICA_LOGCOSH, "exp": ICA_EXP, "cube": ICA_CUBE}
FASTICA_KWARGS = ("algorithm", "whiten", "fun", "fun_args", "max_iter", "tol", "w_init", "whiten_solver")
NOT_CONVERGED = "FastICA did not converge. Consider increasing tolerance or the maximum number of iterations."


def _invalid(name, value, allowed):
    return ValueError(f"The {name!r} parameter of FastICA must be {allowed}. Got {value!r} instead.")


def _is_int(v):
    return isinstance(v, numbers.Integral) and not isinstance(v, (bool, np.bool_))


def check_params(n_components=None, *, algorithm="parallel", whiten="unit-variance", fun="logcosh", fun_args=None,
                 max_iter=200, tol=1e-4, w_init=None, whiten_solver="svd", random_state=None):
    """FastICA's parameter validation: ValueError for a value it refuses (sklearn's InvalidParameterError is one),
    NotImplementedError for a callable ``fun``.  Returns the contrast's alpha."""
    if n_components is not None and not (_is_int(n_components) and n_components >= 1):
        raise _invalid("n_components", n_components, "an int in the range [1, inf) or None")
    if not (isinstance(algorithm, str) and algorithm in ("parallel", "deflation")):
        raise _invalid("algorithm", algorithm, "a str among {'deflation', 'parallel'}")
    if not ((isinstance(whiten, str) and whiten in ("arbitrary-variance", "unit-variance"))
            or (isinstance(whiten, (bool, np.bool_)) and not whiten)):
        raise _invalid("whiten", whiten, "a str among {'arbitrary-variance', 'unit-variance'} or False")
    if callable(fun):
        raise NotImplementedError("mu.tl.ica runs FastICA on the GPU: a callable 'fun' cannot run there; use "
                                  "'logcosh', 'exp' or 'cube'")
    if not (isinstance(fun, str) and fun in FUNS):
        raise _invalid("fun", fun, "a str among {'cube', 'exp', 'logcosh'} or a callable")
    if fun_args is not None and not isinstance(fun_args, dict):
        raise _invalid("fun_args", fun_args, "an instance of 'dict' or None")
    if not (_is_int(max_iter) and max_iter >= 1):
        raise _invalid("max_iter", max_iter, "an int in the range [1, inf)")
    if not (isinstance(tol, numbers.Real) and not isinstance(tol, (bool, np.bool_)) and tol >= 0):
        raise _invalid("tol", tol, "a float in the range [0.0, inf)")
    if not (isinstance(whiten_solver, str) and whiten_solver in ("eigh", "svd")):
        raise _invalid("whiten_solver", whiten_solver, "a str among {'eigh', 'svd'}")
    if not (random_state is None or _is_int(random_state) or isinstance(random_state, np.random.RandomState)):
        raise _invalid("random_state", random_state, "an int, a numpy.random.RandomState instance or None")
    alpha = (fun_args or {}).get("alpha", 1.0)
    if not 1 <= alpha <= 2:
        raise ValueError("alpha must be in [1,2]")
    return float(alpha)


def as_input(X):
    """The dense float32 / float64 matrix FastICA fits (other dtypes become float64); sparse input is refused."""
    import scipy.sparse as sp
    if sp.issparse(X):
        raise TypeError("Sparse data was passed for X, but dense data is required. Use '.toarray()' to convert to "
                        "a dense numpy array.")
    X = np.asarray(X)
    if X.ndim != 2:
        raise ValueError(f"Expected a 2D array, got an array of shape {X.shape}")
    if X.dtype not in (np.float32, np.float64):
        X = X.astype(np.float64)
    n, p = X.shape
    if n < 2:
        raise ValueError(f"Found array with {n} sample(s) (shape={X.shape}) while a minimum of 2 is required by "
                         "FastICA.")
    if p < 1:
        raise ValueError(f"Found array with 0 feature(s) (shape={X.shape}) while a minimum of 1 is required by "
                         "FastICA.")
    return np.ascontiguousarray(X)


def n_components_of(n_components, whiten, n, p):
    """k as FastICA resolves it, with its warnings."""
    if not whiten and n_components is not None:
        n_components = None
        warnings.warn("Ignoring n_components with whiten=False.")
    if n_components is None:
        n_components = min(n, p)
    if n_components > min(n, p):
        n_components = min(n, p)
        warnings.warn("n_components is too large: it will be set to %s" % n_components)
    return int(n_components)


def generator(random_state):
    """sklearn's ``check_random_state``: None is numpy's global generator, an int seeds a new one."""
    if random_state is None:
        return np.random.mtrand._rand
    if isinstance(random_state, np.random.RandomState):
        return random_state
    return np.random.RandomState(random_state)


def device_bytes(n, p, k, itemsize):
    """Device bytes of one fit: X, X1, the output, the partials and the small buffers."""
    from ._lib import load
    ws = int(load().mub_ica_workspace_bytes(n, p, k))
    return n * p * itemsize + n * k * 8 + n * k * itemsize + ws + 8 * (p * p + 4 * k * k + 8 * p + 64)


def check_limits(n, p, k, itemsize):
    """Every refusal, before any device work."""
    if p > ICA_MAX_DIM:
        raise NotImplementedError(f"ICA of {p} features: at most {ICA_MAX_DIM} are supported on the GPU")
    from ._snf import free_device_bytes
    need = device_bytes(n, p, k, itemsize)
    free = free_device_bytes()
    if need > free:
        raise NotImplementedError(f"ICA of {n} cells x {p} features needs {need / 2**30:.1f} GiB of device memory; "
                                  f"{free / 2**30:.1f} GiB are free")


def whitening_of(gram, k, solver, in_dtype):
    """K [k x p] from the centred Gram, as sklearn's "eigh" solver computes it; "svd" takes the same route with a
    clamp at 10 eps(float64) lambda_max instead of 10 eps(input dtype)."""
    from scipy import linalg
    d, u = linalg.eigh(gram)
    order = np.argsort(d)[::-1]
    if solver == "eigh":
        eps = np.finfo(in_dtype).eps * 10
        if np.any(d < eps):
            warnings.warn("There are some small singular values, using whiten_solver = 'svd' might lead to more "
                          "accurate results.")
    else:
        eps = np.finfo(np.float64).eps * 10 * max(float(d.max()), 0.0)
        if np.any(d[order[:k]] < eps):
            warnings.warn("The centred data is numerically rank-deficient: Gram eigenvalues below 10 eps(float64) "
                          "times the largest were clamped, so the whitening differs from an SVD of the data.")
    d = np.sqrt(np.maximum(d, eps))
    d, u = d[order], u[:, order]
    u = u * np.sign(u[0])
    return (u / d).T[:k]


def sym_decorrelation(W):
    """(W W^T)^(-1/2) W."""
    from scipy import linalg
    s, u = linalg.eigh(W @ W.T)
    s = np.clip(s, a_min=np.finfo(W.dtype).tiny, a_max=None)
    return np.linalg.multi_dot([u * (1.0 / np.sqrt(s)), u.T, W])


class _Device:
    """The fit's device buffers and the calls on them."""

    def __init__(self, X, k):
        import torch

        from . import _device
        from ._lib import load
        _device.require_cuda()
        self.dev = torch.device("cuda", torch.cuda.current_device())
        self.n, self.p = X.shape
        self.k = k
        self.sfx = "f32" if X.dtype == np.float32 else "f64"
        self.tdt = torch.float32 if X.dtype == np.float32 else torch.float64
        self.X = torch.from_numpy(X).to(self.dev)
        ws = int(load().mub_ica_workspace_bytes(self.n, self.p, self.k))
        self.ws = torch.empty(max(ws, 8), dtype=torch.uint8, device=self.dev)
        self.status = torch.zeros(1, dtype=torch.int32, device=self.dev)
        self.step_out = torch.empty(k * k + k, dtype=torch.float64, device=self.dev)

    def _f64(self, a):
        import torch
        return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).to(self.dev)

    def _check_finite(self):
        if int(self.status.item()) & 1:
            raise ValueError("Input X contains NaN or infinity.")

    def moments(self):
        import torch

        from ._lib import call, ptr, stream_ptr
        p = self.p
        self.mean = torch.empty(p, dtype=torch.float64, device=self.dev)
        gram = torch.empty((p, p), dtype=torch.float64, device=self.dev)
        call(f"mub_ica_moments_{self.sfx}", ptr(self.X), self.n, p, ptr(self.ws), ptr(self.mean), ptr(gram),
             ptr(self.status), stream_ptr())
        self._check_finite()
        return self.mean.cpu().numpy(), gram.cpu().numpy()

    def project(self, K):
        import torch

        from ._lib import call, ptr, stream_ptr
        self.X1 = torch.empty((self.n, self.k), dtype=torch.float64, device=self.dev)
        Kt = None if K is None else self._f64((K * np.sqrt(self.n)).T)
        mean = getattr(self, "mean", None)
        call(f"mub_ica_project_{self.sfx}", ptr(self.X), self.n, self.p, ptr(mean if K is not None else None),
             ptr(Kt), self.k, ptr(self.X1), ptr(self.status), stream_ptr())
        self._check_finite()
        del self.X

    def step(self, W, fun, alpha):
        """(sum_i g(W x1_i) x1_i^T [r x k], sum_i g'(W x1_i) [r]) for W [r x k]."""
        from ._lib import call, ptr, stream_ptr
        r, k = W.shape
        Wd = self._f64(W)
        out = self.step_out[: r * k + r]
        call("mub_ica_step_f64", ptr(self.X1), self.n, k, ptr(Wd), r, FUNS[fun], alpha, ptr(self.ws), ptr(out),
             stream_ptr())
        h = out.cpu().numpy()
        return h[: r * k].reshape(r, k), h[r * k:]

    def sources(self, M, d1=None, d2=None, stats=False):
        import torch

        from ._lib import call, ptr, stream_ptr
        Mt = self._f64(M.T)
        d1 = None if d1 is None else self._f64(d1)
        d2 = None if d2 is None else self._f64(d2)
        if stats:
            st = torch.empty(2 * self.k, dtype=torch.float64, device=self.dev)
            call(f"mub_ica_sources_{self.sfx}", ptr(self.X1), self.n, self.k, ptr(Mt), ptr(d1), ptr(d2), None,
                 ptr(self.ws), ptr(st), stream_ptr())
            h = st.cpu().numpy()
            return h[: self.k], h[self.k:]
        out = torch.empty((self.n, self.k), dtype=self.tdt, device=self.dev)
        call(f"mub_ica_sources_{self.sfx}", ptr(self.X1), self.n, self.k, ptr(Mt), ptr(d1), ptr(d2), ptr(out),
             None, None, stream_ptr())
        return out.cpu().numpy()


def _parallel(dev, W0, fun, alpha, max_iter, tol, n):
    W = sym_decorrelation(W0)
    for ii in range(max_iter):
        G, gsum = dev.step(W, fun, alpha)
        W1 = sym_decorrelation(G / n - (gsum / n)[:, None] * W)
        lim = max(abs(abs(np.einsum("ij,ij->i", W1, W)) - 1))
        W = W1
        if lim < tol:
            break
    else:
        warnings.warn(NOT_CONVERGED, ConvergenceWarning)
    return W, ii + 1


def _deflation(dev, W0, fun, alpha, max_iter, tol, n):
    k = W0.shape[0]
    W = np.zeros((k, k))
    n_iter = []
    for j in range(k):
        w = W0[j, :].copy()
        w /= np.sqrt((w ** 2).sum())
        for i in range(max_iter):
            G, gsum = dev.step(w[None, :], fun, alpha)
            w1 = G[0] / n - (gsum[0] / n) * w
            w1 -= np.linalg.multi_dot([w1, W[:j].T, W[:j]])
            w1 /= np.sqrt((w1 ** 2).sum())
            lim = np.abs(np.abs((w1 * w).sum()) - 1)
            w = w1
            if lim < tol:
                break
        n_iter.append(i + 1)
        W[j, :] = w
    return W, max(n_iter)


def fit_transform(X, n_components=None, *, algorithm="parallel", whiten="unit-variance", fun="logcosh",
                  fun_args=None, max_iter=200, tol=1e-4, w_init=None, whiten_solver="svd", random_state=None,
                  scale=False):
    """``FastICA(...).fit_transform(X)`` on the GPU, then the reference's ``scale`` division.

    Returns ``(sources, info)``: the n x k sources in the dtype sklearn returns, and a dict with ``n_iter``,
    ``components``, ``mixing``, ``mean`` and ``whitening`` (None without whitening) and ``unmixing`` (FastICA's
    attributes of the same names, ``unmixing`` its ``_unmixing``), in the sources' dtype."""
    from scipy import linalg
    alpha = check_params(n_components, algorithm=algorithm, whiten=whiten, fun=fun, fun_args=fun_args,
                         max_iter=max_iter, tol=tol, w_init=w_init, whiten_solver=whiten_solver,
                         random_state=random_state)
    X = as_input(X)
    n, p = X.shape
    dt = X.dtype
    rs = generator(random_state)
    k = n_components_of(n_components, whiten, n, p)
    if w_init is not None:
        w_init = np.asarray(w_init)
        if w_init.shape != (k, k):
            raise ValueError("w_init has invalid shape -- should be %(shape)s" % {"shape": (k, k)})
    check_limits(n, p, k, dt.itemsize)

    dev = _Device(X, k)
    K = mean = None
    if whiten:
        mean, gram = dev.moments()
        K = whitening_of(gram, k, whiten_solver, dt)
    dev.project(K)
    if w_init is None:
        w_init = np.asarray(rs.normal(size=(k, k)), dtype=dt)
    W0 = np.asarray(w_init, dtype=np.float64)
    run = _parallel if algorithm == "parallel" else _deflation
    W, n_iter = run(dev, W0, fun, alpha, int(max_iter), float(tol), n)

    M = W / np.sqrt(n) if whiten else W
    d1 = d2 = None
    if whiten == "unit-variance":
        _, d1 = dev.sources(M, stats=True)
        W = W / d1[:, None]
    if scale:
        _, d2 = dev.sources(M, d1, stats=True)
    S = dev.sources(M, d1, d2)

    components = W @ K if whiten else W
    info = {"n_iter": int(n_iter), "components": components.astype(dt), "mixing": linalg.pinv(components).astype(dt),
            "mean": None if mean is None else mean.astype(dt), "whitening": None if K is None else K.astype(dt),
            "unmixing": W.astype(dt)}
    return S, info


def ica(data, basis="X_pca", n_components=None, *, random_state=None, scale=False, copy=False, return_info=False,
        **kwargs):
    """Independent component analysis of ``data.obsm[basis]`` -- ``muon.tl.ica`` (muon/_core/tools.py:1365-1386):
    the same arguments, ``**kwargs`` being FastICA's (``algorithm``, ``whiten``, ``fun``, ``fun_args``, ``max_iter``,
    ``tol``, ``w_init``, ``whiten_solver``; any other keyword raises TypeError), and the same slot: ``obsm["X_ica"]``,
    n x n_components, float32 for float32 input and float64 otherwise.  ``scale`` divides it by its ddof-0 column
    std after FastICA's own scaling.  With ``copy`` the result is stored on a copy, which is returned.

    ``return_info=True`` returns ``(result, info)``, ``info`` holding ``n_iter``, ``components``, ``mixing``, ``mean``,
    ``whitening`` and ``unmixing`` (W after the unit-variance rescale).  The passes over the cells run on the GPU in
    float64; a callable ``fun``, more than 128 features, and a fit that does not fit in free device memory raise
    NotImplementedError.  Two calls with the same random state return the same bits."""
    unknown = sorted(set(kwargs) - set(FASTICA_KWARGS))
    if unknown:
        raise TypeError(f"FastICA.__init__() got an unexpected keyword argument {unknown[0]!r}")
    x_ica, info = fit_transform(data.obsm[basis], n_components, random_state=random_state, scale=scale, **kwargs)
    data = data.copy() if copy else data
    data.obsm["X_ica"] = x_ica
    result = data if copy else None
    return (result, info) if return_info else result
