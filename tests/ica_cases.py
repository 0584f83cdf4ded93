"""Inputs of the ICA fixtures (tests/golden/ica_small.npz), rebuilt from seeds: legacy ``RandomState`` streams are
frozen, so the fixture stores only outputs.

Each case mixes planted non-Gaussian sources -- Laplace, uniform and a bimodal mixture, in turn -- into p features,
plus a little Gaussian noise so that every p is full rank.  ``random_state`` is an int, a fresh ``RandomState`` of
the seed ("rs"), or None with numpy's global generator seeded first ("global").
"""
import numpy as np

# name: (n, p, dtype, seed, random_state kind, scale, FastICA keywords)
CASES = {
    "p2_par_logcosh": (2001, 2, np.float64, 0, "int", False, {}),
    "p7_par_exp": (2001, 7, np.float64, 1, "int", False, {"fun": "exp"}),
    "p7_par_cube": (2001, 7, np.float64, 2, "rs", False, {"fun": "cube"}),
    "p7_def_logcosh_a15": (2001, 7, np.float64, 23, "int", False,
                           {"algorithm": "deflation", "fun_args": {"alpha": 1.5}}),
    "p7_def_exp_global": (2001, 7, np.float64, 4, "global", False, {"algorithm": "deflation", "fun": "exp"}),
    "p7_def_cube_k4": (2001, 7, np.float64, 25, "int", False,
                       {"algorithm": "deflation", "fun": "cube", "n_components": 4}),
    "p50_par_k10": (3001, 50, np.float64, 6, "int", False, {"n_components": 10}),
    "p7_arbitrary": (2001, 7, np.float64, 7, "int", False, {"whiten": "arbitrary-variance"}),
    "p7_nowhiten": (2001, 7, np.float64, 8, "int", False, {"whiten": False, "n_components": 3, "max_iter": 15}),
    "p7_eigh_a15": (2001, 7, np.float64, 9, "rs", False, {"whiten_solver": "eigh", "fun_args": {"alpha": 1.5}}),
    "p7_k_too_large": (2001, 7, np.float64, 10, "global", False, {"n_components": 12}),
    "p7_winit_scale": (2001, 7, np.float64, 11, "int", True, {"w_init": "given"}),
    "p7_capped": (2001, 7, np.float64, 12, "int", False, {"max_iter": 3}),
    "p128_par_k16": (1501, 128, np.float64, 13, "int", False, {"n_components": 16}),
    "p7_def_nowhiten": (2001, 7, np.float64, 14, "int", False,
                        {"algorithm": "deflation", "whiten": False, "tol": 1e-3}),
    "f32_p7_par": (2001, 7, np.float32, 15, "int", False, {}),
    "f32_p50_def_k5_scale": (3001, 50, np.float32, 16, "int", True, {"algorithm": "deflation", "n_components": 5}),
    "f32_p7_eigh_exp": (2001, 7, np.float32, 17, "rs", False, {"whiten_solver": "eigh", "fun": "exp"}),
    "f32_p7_arbitrary_cube": (2001, 7, np.float32, 18, "global", False,
                              {"whiten": "arbitrary-variance", "fun": "cube"}),
}


def planted(n, p, seed, dtype=np.float64, m=None):
    """(X [n x p] in dtype, planted sources [n x m] float64): X = [S | 0.1 gaussian] A + 0.05 noise, S of Laplace /
    uniform / bimodal columns.  m = p by default; a smaller m (the n_components of a case) puts the planted sources in
    the leading principal subspace."""
    m = p if m is None else m
    rs = np.random.RandomState(1000 + seed)
    S = 0.1 * rs.normal(size=(n, p))
    for j in range(m):
        kind = j % 3
        if kind == 0:
            S[:, j] = rs.laplace(size=n)
        elif kind == 1:
            S[:, j] = rs.uniform(-1.7, 1.7, size=n)
        else:
            S[:, j] = np.where(rs.uniform(size=n) < 0.5, -1.0, 1.0) + 0.3 * rs.normal(size=n)
    A = rs.normal(size=(p, p))
    X = S @ A + 0.05 * rs.normal(size=(n, p)) + rs.normal(size=p)
    return X.astype(dtype), S[:, :m]


def sample_rows(n):
    """The rows of X_ica the fixture keeps: every 16th and the last.  The whole output is checked against the
    float64 restatement (oracle/ica_ref.py), which reproduces the reference to 1e-10."""
    return np.unique(np.r_[np.arange(0, n, 16), n - 1])


def w_init_of(case):
    n, p, dtype, seed, rs_kind, scale, kw = CASES[case]
    k = kw.get("n_components") or p
    return np.random.RandomState(2000 + seed).normal(size=(k, k))


def arguments(case):
    """(X, sources, random_state, scale, FastICA keywords) of a case.  The generator is made fresh on every call;
    for "global", numpy's global generator is seeded here."""
    n, p, dtype, seed, rs_kind, scale, kw = CASES[case]
    m = kw.get("n_components") if kw.get("whiten", "unit-variance") else None
    X, S = planted(n, p, seed, dtype, None if m is None else min(m, p))
    kw = dict(kw)
    if kw.get("w_init") == "given":
        kw["w_init"] = w_init_of(case)
    if rs_kind == "int":
        rs = seed
    elif rs_kind == "rs":
        rs = np.random.RandomState(seed)
    else:
        np.random.seed(seed)
        rs = None
    return X, S, rs, scale, kw
