"""Generates the ICA fixtures by running the unmodified reference ``muon.tl.ica``:

    python tests/golden/make_golden_ica.py

The reference function is read from muon/_core/tools.py with ``ast`` and executed as written, with sklearn's real
``FastICA`` and the project's containers for AnnData / MuData.  Inputs are rebuilt from the seeds in
tests/ica_cases.py, so the fixture holds only outputs.

``ica_small.npz``: ``sklearn_version``, ``cases`` (the case names) and per case ``<name>_``: ``X_ica`` (the
reference's slot at the rows ``ica_cases.sample_rows(n)``, to keep the file small), ``X_ica_shape``, ``n_iter``,
``components``, ``mixing``, ``unmixing`` and, with whitening, ``mean`` and ``whitening`` (FastICA's attributes from the same arguments and random state), and ``warnings`` (the messages the
reference call emitted, in order).  Float32 cases also hold ``f32_gap``: how far sklearn's float32 sources lie from
its own float64 run on the same values, relative to each column's scale (sklearn computes in float32 throughout; its
"eigh" whitening forms the Gram in float32, which costs about eps(float32) x cond(X)^2).  A case whose stopping
value comes within 1e-6 of ``tol`` at any iteration (in the float64 restatement, oracle/ica_ref.py) is refused,
because its iteration count would depend on rounding.
``ica_signature.json``: the reference signature of ``muon.tl.ica``.
"""
import ast
import json
import os
import sys
import warnings
from typing import Union

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from ica_cases import CASES, arguments, sample_rows  # noqa: E402
from muon_b200 import SimpleAnnData, SimpleMuData  # noqa: E402
from oracle._refload import REF_ROOT  # noqa: E402
from oracle.ica_ref import fastica_ref  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
TOOLS = os.path.join(REF_ROOT, "muon", "_core", "tools.py")


def _function(name):
    tree = ast.parse(open(TOOLS).read())
    (fn,) = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == name]
    return fn


def load_reference_ica():
    """The reference's own ``ica``; its ``from sklearn.decomposition import FastICA`` imports the real one."""
    g = {"np": np, "Union": Union, "AnnData": SimpleAnnData, "MuData": SimpleMuData}
    exec(compile(ast.Module([_function("ica")], []), TOOLS, "exec"), g)
    return g["ica"]


def dump_signature():
    fn = _function("ica")
    a = fn.args
    out = {"ica": {"params": [x.arg for x in a.args], "defaults": [ast.unparse(d) for d in a.defaults],
                   "kwonly": [x.arg for x in a.kwonlyargs], "kw_defaults": [ast.unparse(d) for d in a.kw_defaults],
                   "varkw": a.kwarg.arg if a.kwarg else None}}
    json.dump(out, open(os.path.join(OUT, "ica_signature.json"), "w"), indent=1)


def main():
    import sklearn
    from sklearn.decomposition import FastICA
    ica = load_reference_ica()
    z = {"sklearn_version": np.array(sklearn.__version__), "cases": np.array(list(CASES))}
    bad = []
    for name in CASES:
        X, _, rs, scale, kw = arguments(name)
        ad = SimpleAnnData(np.zeros((X.shape[0], 1)))
        ad.obsm["X_pca"] = X
        with warnings.catch_warnings(record=True) as rec:
            warnings.simplefilter("always")
            ica(ad, random_state=rs, scale=scale, **kw)
        msgs = [str(w.message) for w in rec]

        X, _, rs, scale, kw = arguments(name)
        est = FastICA(random_state=rs, **kw)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            S = est.fit_transform(X)
        if scale:
            S /= S.std(axis=0)
        assert np.array_equal(S, ad.obsm["X_ica"]) and S.dtype == ad.obsm["X_ica"].dtype, name
        if X.dtype == np.float32:
            X, _, rs, scale, kw = arguments(name)
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                S64 = FastICA(random_state=rs, **kw).fit_transform(X.astype(np.float64))
            if scale:
                S64 /= S64.std(axis=0)
            z[f"{name}_f32_gap"] = np.array(np.max(np.abs(S - S64) / np.max(np.abs(S64), axis=0)))

        X, _, rs, scale, kw = arguments(name)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            ref = fastica_ref(X, random_state=rs, **kw)
        tol = kw.get("tol", 1e-4)
        gap = float(np.min(np.abs(np.asarray(ref["lims"]) - tol)))
        if gap < 1e-6:
            bad.append(name)
            print(f"{name}: a stopping value lies {gap:.2e} from tol; choose another seed")
            continue
        assert ref["n_iter"] == est.n_iter_, (name, ref["n_iter"], est.n_iter_)

        z[f"{name}_X_ica"] = ad.obsm["X_ica"][sample_rows(X.shape[0])]
        z[f"{name}_X_ica_shape"] = np.array(ad.obsm["X_ica"].shape)
        z[f"{name}_n_iter"] = np.array(est.n_iter_)
        z[f"{name}_warnings"] = np.array(msgs, dtype=str)
        for attr in ("components", "mixing"):
            z[f"{name}_{attr}"] = getattr(est, attr + "_")
        z[f"{name}_unmixing"] = est._unmixing
        if kw.get("whiten", "unit-variance"):
            z[f"{name}_mean"] = est.mean_
            z[f"{name}_whitening"] = est.whitening_
        print(f"{name:24s} n_iter {est.n_iter_:3d}  gap {gap:.1e}  warnings {msgs}")
    if bad:
        raise SystemExit(f"refused cases: {bad}")
    path = os.path.join(OUT, "ica_small.npz")
    np.savez_compressed(path, **z)
    print(os.path.basename(path), os.path.getsize(path))
    dump_signature()


if __name__ == "__main__":
    main()
