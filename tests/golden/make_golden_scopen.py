"""Generates the scOpen fixtures by running the unmodified reference ``muon.atac.pp.scopen``:

    python tests/golden/make_golden_scopen.py

The reference function is read from muon/_atac/preproc.py with ``ast`` and executed as written, with the project's
containers for AnnData / MuData and ``scopen.MF`` replaced by the stand-in of oracle/scopen_ref.py (exact-SVD NNDSVD,
coordinate descent bounded to [0, 1]).  Inputs are rebuilt from the seeds in tests/scopen_cases.py.

``scopen_small.npz`` holds ``cases`` and per case ``<name>_``:
  ``W0``, ``H0``          the NNDSVD init (from the exact SVD);
  ``W``, ``H``            the final factors of the reference run (bound 1), ``W_inf``, ``H_inf`` those of the same
                          fit with bound +inf (sklearn's), from the same init;
  ``n_iter``, ``n_iter_inf``, ``ratio``, ``ratio_inf``   iterations and the last violation ratio of both fits;
  ``M_rows``              the rows ``scopen_cases.sample_rows(m)`` of M = clip(W H, 0, 1) (the reference's ``X.T``);
  ``objective``           0.5 ||X - W H||^2 + 0.5 alpha (||W||^2 + ||H||^2) of the reference's factors;
  ``sens_M``, ``sens_W``, ``sens_obj``   how far M (absolute), W (relative to each column's max) and the objective
                          (relative) move when the init is scaled entrywise by 1 + 1e-5 N(0, 1);
  ``lines``, ``warnings`` the first three printed lines and the warning messages of the reference call.
Every violation ratio of both fits lies at least 1e-6 (relative) from tol, so the iteration counts do not depend on
rounding.  ``scopen_signature.json``: the reference signature of ``muon.atac.pp.scopen``.
"""
import contextlib
import io
import json
import os
import sys
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from scopen_cases import CASES, arguments, matrix, sample_rows  # noqa: E402
from muon_b200 import SimpleAnnData, SimpleMuData  # noqa: E402
from oracle import scopen_ref as R  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
DEFAULTS = {"n_components": 30, "max_iter": 500, "min_rho": 0.0, "max_rho": 0.5, "alpha": 1}
PERTURB = 1e-5


def _check_ratios(case, ratios):
    r = np.asarray(ratios)
    gap = np.min(np.abs(r - R.TOL)) / R.TOL if r.size else np.inf
    assert gap >= 1e-6, f"{case}: a violation ratio lies {gap:.2e} (relative) from tol"


def make_case(case, ref, out):
    data, ad, kw = arguments(case, (SimpleAnnData, SimpleMuData))
    kw_all = {**DEFAULTS, **kw}
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf), warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        ref(data, **kw)
    X, _ = matrix(case)
    r = R.scopen_ref(X, upper=1.0, **kw_all)
    assert np.array_equal(ad.varm["scopen"], r["W"]) and np.array_equal(ad.obsm["X_scopen"], r["H"].T)
    r_inf = R.scopen_ref(X, upper=np.inf, init=(r["W0"], r["H0"]), **kw_all)
    _check_ratios(case, r["ratios"])
    _check_ratios(case, r_inf["ratios"])
    Xd = R.dense_of(r["P"], r["s"])
    a = float(kw_all["alpha"])
    obj = R.objective(Xd, r["W"], r["H"], a)
    rng = np.random.default_rng(12345)
    init = tuple(A * (1 + PERTURB * rng.standard_normal(A.shape)) for A in (r["W0"], r["H0"]))
    p = R.scopen_ref(X, upper=1.0, init=init, **kw_all)
    M = np.asarray(ad.X).T
    m = M.shape[0]
    colmax = np.maximum(np.abs(r["W"]).max(axis=0), 1e-300)
    out.update({
        f"{case}_W0": r["W0"], f"{case}_H0": r["H0"], f"{case}_W": r["W"], f"{case}_H": r["H"],
        f"{case}_W_inf": r_inf["W"], f"{case}_H_inf": r_inf["H"],
        f"{case}_n_iter": r["n_iter"], f"{case}_n_iter_inf": r_inf["n_iter"],
        f"{case}_ratio": r["ratios"][-1], f"{case}_ratio_inf": r_inf["ratios"][-1],
        f"{case}_M_rows": M[sample_rows(m)], f"{case}_objective": obj,
        f"{case}_sens_M": np.abs(p["M"] - M).max(), f"{case}_sens_W": (np.abs(p["W"] - r["W"]) / colmax).max(),
        f"{case}_sens_obj": abs(R.objective(Xd, p["W"], p["H"], a) - obj) / obj,
        f"{case}_lines": np.array(buf.getvalue().splitlines()[:3]),
        f"{case}_warnings": np.array([str(w.message) for w in rec], dtype=str).reshape(-1),
    })
    print(case, "n_iter", r["n_iter"], r_inf["n_iter"], "sens M/W/obj", out[f"{case}_sens_M"], out[f"{case}_sens_W"],
          out[f"{case}_sens_obj"])


def main():
    ref = R.load_reference_scopen()
    out = {"cases": np.array(list(CASES))}
    for case in CASES:
        make_case(case, ref, out)
    np.savez_compressed(os.path.join(OUT, "scopen_small.npz"), **out)
    json.dump({"scopen": R.reference_signature()}, open(os.path.join(OUT, "scopen_signature.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
