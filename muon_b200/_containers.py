"""Minimal stand-ins for ``anndata.AnnData`` / ``mudata.MuData``.

The drop-in boundary of this package is the Python call signature of
``mu.atac.pp.tfidf`` / ``mu.atac.tl.lsi`` / ``mu.tl.mofa`` plus the AnnData /
MuData slots those calls rebind (reference: muon/_atac/preproc.py:62-67,120-129,
muon/_atac/tools.py:42-69, muon/_core/tools.py:604-701).  ``anndata`` and
``mudata`` are not installable in the build container (no network), so the
shim is duck-typed: real AnnData/MuData objects are accepted when those
packages are importable, and these two small classes provide the same slots
(``X layers obs var obsm varm obsp uns shape is_view copy()``, ``mod``) for
tests, the benchmark and anyone who just wants to hand over arrays.

They implement container semantics only -- no numerics live here.
"""
from __future__ import annotations

import copy as _copy
from collections import OrderedDict
from typing import Mapping, Optional

import numpy as np

try:  # pandas is present in the image, but keep the containers usable without it
    import pandas as pd
except Exception:  # pragma: no cover
    pd = None


def _frame(index, n, prefix):
    names = [f"{prefix}{i}" for i in range(n)] if index is None else list(index)
    if pd is not None:
        return pd.DataFrame(index=pd.Index([str(x) for x in names]))
    return names


class SimpleAnnData:
    """Just enough of AnnData for the three hot-path entry points."""

    def __init__(self, X=None, obs=None, var=None, layers=None, obsm=None, varm=None,
                 uns=None, obsp=None, shape=None):
        if X is not None and not hasattr(X, "shape"):
            X = np.asarray(X)
        self._X = X
        if X is not None:
            n, d = X.shape
        elif shape is not None:
            n, d = shape
        elif layers:
            n, d = next(iter(layers.values())).shape
        else:
            n, d = (0 if obs is None else len(obs)), (0 if var is None else len(var))
        self._shape = (int(n), int(d))
        if pd is not None and isinstance(obs, pd.DataFrame):
            self.obs = obs
        else:
            self.obs = _frame(obs, n, "obs")
        if pd is not None and isinstance(var, pd.DataFrame):
            self.var = var
        else:
            self.var = _frame(var, d, "var")
        self.layers = dict(layers or {})
        self.obsm = dict(obsm or {})
        self.varm = dict(varm or {})
        self.obsp = dict(obsp or {})
        self.uns = OrderedDict(uns or {})
        self.is_view = False
        self.isbacked = False
        self._parent = None

    # -- AnnData-like surface ------------------------------------------------
    @property
    def X(self):
        return self._X

    @X.setter
    def X(self, value):
        if value is not None and tuple(value.shape) != self._shape:
            raise ValueError(f"X has shape {tuple(value.shape)}, expected {self._shape}")
        self._X = value

    @property
    def shape(self):
        return self._shape

    @property
    def n_obs(self):
        return self._shape[0]

    @property
    def n_vars(self):
        return self._shape[1]

    @property
    def obs_names(self):
        return self.obs.index if pd is not None else self.obs

    @property
    def var_names(self):
        return self.var.index if pd is not None else self.var

    def copy(self):
        def cp(v):
            return v.copy() if hasattr(v, "copy") else _copy.deepcopy(v)

        out = SimpleAnnData(
            X=None if self._X is None else cp(self._X),
            obs=cp(self.obs), var=cp(self.var),
            layers={k: cp(v) for k, v in self.layers.items()},
            obsm={k: cp(v) for k, v in self.obsm.items()},
            varm={k: cp(v) for k, v in self.varm.items()},
            obsp={k: cp(v) for k, v in self.obsp.items()},
            uns=_copy.deepcopy(self.uns), shape=self._shape)
        return out

    def __getitem__(self, key):
        """Row/column subsetting that yields a *view* (``is_view=True``) like AnnData does."""
        if not isinstance(key, tuple):
            key = (key, slice(None))
        rk, ck = key

        def names_to_idx(k, names):
            if isinstance(k, slice):
                return k
            arr = np.asarray(k)
            if arr.dtype.kind in "USO":
                lut = {str(nm): i for i, nm in enumerate(names)}
                return np.asarray([lut[str(a)] for a in arr.ravel()], dtype=np.int64)
            return arr

        rk = names_to_idx(rk, self.obs_names)
        ck = names_to_idx(ck, self.var_names)

        def sub(M):
            if M is None:
                return None
            out = M[rk] if isinstance(rk, slice) else M[np.asarray(rk)]
            return out[:, ck] if isinstance(ck, slice) else out[:, np.asarray(ck)]

        def rows(M):
            return M[rk] if isinstance(rk, slice) else M[np.asarray(rk)]

        def cols(M):
            return M[ck] if isinstance(ck, slice) else M[np.asarray(ck)]

        obs = self.obs.iloc[rk] if pd is not None else list(np.asarray(self.obs, dtype=object)[rk])
        var = self.var.iloc[ck] if pd is not None else list(np.asarray(self.var, dtype=object)[ck])
        n, d = len(obs), len(var)
        v = SimpleAnnData(X=sub(self._X), obs=obs, var=var,
                          layers={k: sub(M) for k, M in self.layers.items()},
                          obsm={k: rows(M) for k, M in self.obsm.items()},
                          varm={k: cols(M) for k, M in self.varm.items()},
                          uns=self.uns, shape=(n, d))
        v.is_view = True
        v._parent = self
        return v

    def _init_as_actual(self, other):
        """What ``scanpy._utils.view_to_actual`` does to a view (reference preproc.py:84)."""
        self.__dict__.update(other.__dict__)
        self.is_view = False
        self._parent = None

    def __repr__(self):
        return f"SimpleAnnData(n_obs={self.n_obs}, n_vars={self.n_vars})"


def view_to_actual(adata):
    """Turn a view into a real object in place (scanpy._utils.view_to_actual semantics)."""
    if getattr(adata, "is_view", False):
        if hasattr(adata, "_init_as_actual"):
            adata._init_as_actual(adata.copy())


class SimpleMuData:
    """Just enough of MuData: ``.mod`` mapping of modalities sharing observations."""

    def __init__(self, mod: Mapping[str, object]):
        if not isinstance(mod, Mapping):  # MuData(adata) wraps one modality (tools.py:425-431)
            mod = {"mod": mod}
        self.mod = OrderedDict(mod)
        self.obsm, self.varm, self.obsp = {}, {}, {}
        self.uns = OrderedDict()
        self.update()

    def update(self):
        """Recompute the union of observation / variable names; existing annotation columns are kept
        (like ``MuData.update_obs``), new names get NaN."""
        names, seen = [], set()
        for a in self.mod.values():
            for nm in a.obs_names:
                if nm not in seen:
                    seen.add(nm)
                    names.append(nm)
        vnames = [v for a in self.mod.values() for v in a.var_names]
        old_obs, old_var = getattr(self, "obs", None), getattr(self, "var", None)
        self.obs = _frame(names, len(names), "obs")
        self.var = _frame(vnames, len(vnames), "var")
        if pd is not None:
            if isinstance(old_obs, pd.DataFrame) and old_obs.shape[1]:
                self.obs = old_obs.reindex(self.obs.index)
            if isinstance(old_var, pd.DataFrame) and old_var.shape[1] and not old_var.index.has_duplicates:
                self.var = old_var.reindex(self.var.index)

    update_obs = update
    update_var = update

    @property
    def n_obs(self):
        return len(self.obs)

    @property
    def n_vars(self):
        return len(self.var)

    @property
    def shape(self):
        return (self.n_obs, self.n_vars)

    @property
    def obs_names(self):
        return self.obs.index if pd is not None else self.obs

    @property
    def var_names(self):
        return self.var.index if pd is not None else self.var

    def __getitem__(self, key):
        if isinstance(key, str):
            return self.mod[key]
        if isinstance(key, tuple):          # mdata[names, :] (muon/_prot/preproc.py:92)
            key, cols = key
            if not (isinstance(cols, slice) and cols == slice(None)):
                raise NotImplementedError("SimpleMuData selects observations only: use mdata[names, :]")
        out = SimpleMuData({k: a[[n for n in key if n in set(a.obs_names)]] for k, a in self.mod.items()})
        return out

    def copy(self):
        out = SimpleMuData({k: a.copy() for k, a in self.mod.items()})
        out.obs = self.obs.copy() if hasattr(self.obs, "copy") else list(self.obs)
        out.obsm = {k: v.copy() for k, v in self.obsm.items()}
        out.varm = {k: v.copy() for k, v in self.varm.items()}
        out.uns = _copy.deepcopy(self.uns)
        return out

    def __repr__(self):
        return f"SimpleMuData({', '.join(f'{k}: {a.n_obs}x{a.n_vars}' for k, a in self.mod.items())})"


def _real(cls_name: str, module: str) -> Optional[type]:
    try:
        mod = __import__(module)
        return getattr(mod, cls_name)
    except Exception:
        return None


def is_anndata(obj) -> bool:
    real = _real("AnnData", "anndata")
    if real is not None and isinstance(obj, real):
        return True
    return isinstance(obj, SimpleAnnData)


def is_mudata(obj) -> bool:
    real = _real("MuData", "mudata")
    if real is not None and isinstance(obj, real):
        return True
    return isinstance(obj, SimpleMuData)
