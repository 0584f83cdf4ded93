"""The inputs of the scOpen fixtures (tests/golden/scopen_small.npz), rebuilt from seeds.

Counts come from a planted topic model, so the leading singular values of the scaled pattern stand apart and the
NNDSVD init is well determined.  Every cell has at least one positive entry and the cells' counts differ, so every
scale is finite."""
import numpy as np
import scipy.sparse as sp

# name -> (seed, cells, peaks, topics, layout, kwargs of scopen)
CASES = {
    "csr_f32": (1, 100, 250, 8, "csr_f32", {"n_components": 10}),
    "dense_f64": (2, 90, 200, 5, "dense_f64", {"n_components": 5}),
    "csc_maxiter": (3, 110, 240, 8, "csc", {"n_components": 8, "max_iter": 15}),
    "mudata": (4, 80, 220, 6, "mudata", {"n_components": 6}),
    "k1": (5, 70, 180, 3, "csr_f32", {"n_components": 1}),
    "converges": (5, 70, 180, 3, "csr_f32", {"n_components": 3, "alpha": 10}),
    "k30": (6, 80, 150, 30, "csr_f32", {"n_components": 30}),
    "params": (7, 100, 230, 6, "csr_f32", {"n_components": 6, "min_rho": 0.1, "max_rho": 0.7, "alpha": 0.5}),
}


def planted_counts(seed, n, m, topics, density=0.12):
    """n x m non-negative integer counts (float64) with a planted rank-``topics`` pattern."""
    rng = np.random.default_rng(seed)
    theta = rng.gamma(0.3, size=(n, topics)) * np.linspace(2.0, 0.5, topics)[None, :]
    beta = (rng.random((topics, m)) < 0.25) * rng.gamma(2.0, size=(topics, m))
    p = theta @ beta + 0.05
    p *= density * n * m / p.sum()
    pattern = rng.random((n, m)) < np.minimum(p, 0.95)
    pattern[np.arange(n), rng.integers(0, m, n)] = True
    return pattern * rng.integers(1, 4, size=(n, m)).astype(np.float64)


def with_zeros_negatives_duplicates(C, seed):
    """C as a float32 CSR that also stores explicit zeros, negative entries, and duplicates whose sum keeps each
    entry's sign (one positive entry split as (v + 1, -1))."""
    rng = np.random.default_rng(seed + 1000)
    n, m = C.shape
    rows, cols, vals = [], [], []
    for i in range(n):
        nz = np.flatnonzero(C[i])
        zs = rng.choice(np.flatnonzero(C[i] == 0), size=2, replace=False)
        entries = [(j, C[i, j]) for j in nz] + [(zs[0], 0.0), (zs[1], -float(rng.integers(1, 3)))]
        if len(nz) > 1:
            j = nz[0]
            entries = [(jj, v) for jj, v in entries if jj != j] + [(j, C[i, j] + 1.0), (j, -1.0)]
        for j, v in entries:
            rows.append(i)
            cols.append(j)
            vals.append(v)
    order = np.lexsort((np.arange(len(rows)), np.asarray(rows)))
    rows, cols, vals = np.asarray(rows)[order], np.asarray(cols)[order], np.asarray(vals)[order]
    indptr = np.concatenate([[0], np.cumsum(np.bincount(rows, minlength=n))])
    X = sp.csr_matrix((vals.astype(np.float32), cols.astype(np.int32), indptr), shape=(n, m))
    X.has_canonical_format = False
    return X


def matrix(case):
    """The input ``X`` of a case (cells x peaks) and its layout."""
    seed, n, m, topics, layout, _ = CASES[case]
    C = planted_counts(seed, n, m, topics)
    if layout == "csr_f32":
        return with_zeros_negatives_duplicates(C, seed), layout
    if layout == "dense_f64":
        return C, layout
    if layout == "csc":
        return sp.csc_matrix(C), layout
    return sp.csr_matrix(C.astype(np.float32)), layout


def arguments(case, containers):
    """(data, adata, kwargs): the object scopen is called on, the AnnData it writes, and its keyword arguments.
    ``containers`` = (AnnData class, MuData class)."""
    AnnData, MuData = containers
    X, layout = matrix(case)
    ad = AnnData(X.copy())
    data = MuData({"atac": ad}) if layout == "mudata" else ad
    return data, ad, dict(CASES[case][5])


def sample_rows(n):
    """Every 16th row and the last."""
    return np.unique(np.concatenate([np.arange(0, n, 16), [n - 1]]))
