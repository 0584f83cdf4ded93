"""Generates the SNF fixtures by running the unmodified reference ``muon.tl.snf``:

    python tests/golden/make_golden_snf.py

The reference function is read from muon/_core/tools.py with ``ast`` and executed as written, with stand-ins for
its imports: the project's containers for MuData / AnnData, a ``_choose_representation`` that returns the
representation it is asked for, and the reference's own ``_sparse_csr_fast_knn`` (muon/_core/preproc.py) under
numba.  The reference cannot run on sparse distances (see DESIGN.md section 8), so every case gives it dense ones.

``snf_small.npz``: per case ``c<i>_``: ``X<m>`` the coordinates of modality m (the distances are
``scipy.spatial.distance.cdist(X, X)``), ``params`` (n_neighbors, n_iterations, sigma) and the reference's
``distances`` / ``connectivities`` as CSR (``_data``, ``_indices``, ``_indptr``, ``_shape``).
``snf_signature.json``: the reference signature of ``muon.tl.snf``.
"""
import ast
import json
import logging
import os
import sys
from datetime import datetime
from typing import Dict, Optional, Union

import numpy as np
import scipy.sparse as sp
from scipy.spatial.distance import cdist

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from muon_b200 import SimpleAnnData, SimpleMuData  # noqa: E402
from oracle._refload import REF_ROOT  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
TOOLS = os.path.join(REF_ROOT, "muon", "_core", "tools.py")
PREPROC = os.path.join(REF_ROOT, "muon", "_core", "preproc.py")

# (n_cells, n_modalities, n_neighbors, n_iterations, sigma)
CASES = [(300, 2, 20, 20, 0.5), (451, 3, 5, 7, 0.3), (333, 2, 1, 3, 0.5), (401, 3, 20, 20, 0.8),
         (360, 2, 5, 20, 0.5)]


def _function(path, names):
    src = open(path).read()
    tree = ast.parse(src)
    return [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in names]


def load_reference_snf():
    """The reference's own ``snf`` function object, executed from its source file."""
    import numba
    g = {"np": np, "issparse": sp.issparse, "csr_matrix": sp.csr_matrix, "csr_array": sp.csr_array,
         "logging": logging, "datetime": datetime, "Optional": Optional, "Union": Union, "Dict": Dict,
         "MuData": SimpleMuData, "njit": numba.njit, "prange": numba.prange,
         "_choose_representation": lambda adata, use_rep=None, n_pcs=None: adata.obsm[use_rep or "X_pca"]}
    for fn in _function(PREPROC, ("_sparse_csr_fast_knn_", "_sparse_csr_fast_knn")):
        exec(compile(ast.Module([fn], []), PREPROC, "exec"), g)
    (fn,) = _function(TOOLS, ("snf",))
    exec(compile(ast.Module([fn], []), TOOLS, "exec"), g)
    return g["snf"]


def planted_coords(n, n_mod, seed):
    rng = np.random.default_rng(seed)
    labels = np.arange(n) * 3 // n
    return [rng.normal(size=(n, 10)) + rng.normal(size=(3, 10))[labels] * 3 for _ in range(n_mod)]


def mudata_of(coords):
    mods = {}
    for m, X in enumerate(coords):
        a = SimpleAnnData(np.zeros((X.shape[0], 1)))
        a.obsm["X_pca"] = X
        a.obsp["distances"] = cdist(X, X)
        a.uns["neighbors"] = {"params": {"n_neighbors": 15, "use_rep": "X_pca"}, "distances_key": "distances",
                              "connectivities_key": "connectivities"}
        mods[f"m{m}"] = a
    return SimpleMuData(mods)


def dump_signature():
    (fn,) = _function(TOOLS, ("snf",))
    params = [a.arg for a in fn.args.args]
    defaults = [repr(eval(ast.unparse(d), {"np": np})) for d in fn.args.defaults]
    required = len(params) - len(defaults)
    out = {"snf": {"params": params, "defaults": [repr(None)] * required + defaults, "required": required}}
    json.dump(out, open(os.path.join(OUT, "snf_signature.json"), "w"), indent=1)


def main():
    snf = load_reference_snf()
    z = {}
    for c, (n, n_mod, k, iters, sigma) in enumerate(CASES):
        coords = planted_coords(n, n_mod, seed=c)
        md = mudata_of(coords)
        snf(md, n_neighbors=k, n_iterations=iters, sigma=sigma)
        for m, X in enumerate(coords):
            z[f"c{c}_X{m}"] = X
        z[f"c{c}_params"] = np.array([k, iters, sigma])
        for key in ("distances", "connectivities"):
            A = md.obsp[key]
            assert isinstance(A, sp.csr_array) and A.nnz == n * k
            z[f"c{c}_{key}_data"] = A.data
            z[f"c{c}_{key}_indices"] = A.indices
            z[f"c{c}_{key}_indptr"] = A.indptr
            z[f"c{c}_{key}_shape"] = np.array(A.shape)
        print(c, n, n_mod, k, iters, sigma, md.uns["neighbors"]["params"])
    path = os.path.join(OUT, "snf_small.npz")
    np.savez_compressed(path, n_cases=len(CASES), **z)
    print(os.path.basename(path), os.path.getsize(path))
    dump_signature()


if __name__ == "__main__":
    main()
