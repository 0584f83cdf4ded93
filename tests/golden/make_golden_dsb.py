"""Generates the DSB fixtures by running the UNMODIFIED reference ``dsb`` (muon/_prot/preproc.py:17) on the
cases of tests/dsb_cases.py, through oracle.dsb_ref.load_reference_dsb (stubbed anndata/mudata, scikit-learn
as installed, nothing copied).

    python tests/golden/make_golden_dsb.py

Each ``dsb_<case>.npz`` holds the inputs, the call's keyword arguments (json), the normalised matrix, the
warnings the call raised and -- recorded by wrapping the reference's GaussianMixture, whose fits are left as
they are -- each cell's ``bgmean``, chosen model (0 tied, 1 full), iteration counts and convergence flags.
``dsb_signature.json`` holds the reference signature of ``dsb`` (read with ast).
"""
import ast
import json
import os
import sys
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from dsb_cases import CASES, build_call, make_inputs, pack, result_of  # noqa: E402
from muon_b200._containers import SimpleAnnData, SimpleMuData  # noqa: E402
from oracle.dsb_ref import load_reference_dsb  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))


def recording_dsb():
    """The reference ``dsb`` with its GaussianMixture replaced by a subclass that records every fit."""
    dsb = load_reference_dsb()
    mod = sys.modules[dsb.__module__]
    base = mod.GaussianMixture
    log = []

    class Recorder(base):
        def fit(self, X, y=None):
            out = super().fit(X, y)
            log.append({"type": self.covariance_type, "min_mean": float(np.min(self.means_)),
                        "n_iter": int(self.n_iter_), "converged": bool(self.converged_),
                        "bic": float(self.bic(X))})
            return out

    mod.GaussianMixture = Recorder
    return dsb, log


def run_case(dsb, log, name, z):
    log.clear()
    data, raw, kw = build_call(name, z, SimpleAnnData, SimpleMuData)
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        ret = dsb(data, raw, **kw)
    X, obs = result_of(name, data, raw, ret)
    res = {"out": X, "obs_names_out": obs,
           "warnings": np.array([f"{x.category.__name__}: {x.message}" for x in w
                                 if x.category.__name__ != "ConvergenceWarning"])}
    if log:
        t, f = log[0::2], log[1::2]
        assert all(r["type"] == "tied" for r in t) and all(r["type"] == "full" for r in f)
        model = np.array([0 if a["bic"] < b["bic"] else 1 for a, b in zip(t, f)], dtype=np.int8)
        res["bgmean"] = np.array([a["min_mean"] if m == 0 else b["min_mean"] for a, b, m in zip(t, f, model)])
        res["model"] = model
        res["n_iter"] = np.array([[a["n_iter"], b["n_iter"]] for a, b in zip(t, f)], dtype=np.int32)
        res["converged"] = np.array([[a["converged"], b["converged"]] for a, b in zip(t, f)])
    return res


def dump_signature():
    tree = ast.parse(open(os.path.join(os.environ.get("MUON_REFERENCE_ROOT", "/root/reference"),
                                       "muon/_prot/preproc.py")).read())
    fn = next(n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "dsb")
    params = [a.arg for a in fn.args.args]
    defaults = [ast.literal_eval(d) for d in fn.args.defaults]
    required = len(params) - len(defaults)
    out = {"dsb": {"params": params, "defaults": [repr(None)] * required + [repr(d) for d in defaults],
                   "required": required}}
    json.dump(out, open(os.path.join(OUT, "dsb_signature.json"), "w"), indent=1)


def main():
    dsb, log = recording_dsb()
    for name in CASES:
        arrays = make_inputs(name)
        z = pack(arrays)
        z["kwargs"] = np.array(json.dumps(CASES[name]["kw"]))
        z.update(run_case(dsb, log, name, z))
        path = os.path.join(OUT, f"dsb_{name}.npz")
        np.savez_compressed(path, **z)
        print(os.path.basename(path), os.path.getsize(path), list(z["warnings"]))
    dump_signature()


if __name__ == "__main__":
    main()
