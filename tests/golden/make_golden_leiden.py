"""Generates the clustering fixtures by running the unmodified reference driver (muon/_core/tools.py:928-1206) with
the stand-ins of tests/leiden_ref.py for leidenalg / louvain-igraph (their optimiser restated sequentially):

    python tests/golden/make_golden_leiden.py

``leiden_small.npz``: two modality graphs over the same 4 planted clusters of distinct sizes (80, 60, 45, 30), and
for each recorded call of ``leiden`` and ``louvain`` (the default, a resolution dict, mod_weights as a list,
partition_kwargs={"weights": "weight"}) the labels, the categories and ``uns[algorithm]["params"]`` as JSON.
``cluster_signature.json``: the reference signatures of ``leiden`` and ``louvain`` (read with ast).
"""
import ast
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

import leiden_ref as R  # noqa: E402

CALLS = R.REFERENCE_CALLS


def mudata(A, B):
    from muon_b200 import SimpleAnnData, SimpleMuData
    mods = {}
    for name, G in (("rna", A), ("atac", B)):
        ad = SimpleAnnData(np.zeros((G.shape[0], 1), np.float32))
        ad.obsp["connectivities"] = G
        ad.uns["neighbors"] = {"connectivities_key": "connectivities", "distances_key": "distances", "params": {}}
        mods[name] = ad
    return SimpleMuData(mods)


def dump_signature():
    tree = ast.parse(open(os.path.join(os.environ.get("MUON_REFERENCE_ROOT", "/root/reference"),
                                       "muon/_core/tools.py")).read())
    out = {}
    for name in ("leiden", "louvain"):
        fn = next(n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == name)
        params = [a.arg for a in fn.args.args]
        defaults = [ast.unparse(d) for d in fn.args.defaults]
        required = len(params) - len(defaults)
        out[name] = {"params": params, "defaults": ["None"] * required + defaults, "required": required,
                     "var_keyword": fn.args.kwarg.arg if fn.args.kwarg else None}
    json.dump(out, open(os.path.join(HERE, "cluster_signature.json"), "w"), indent=1)


def main():
    leiden, louvain = R.load_reference_cluster()
    labels, A, B = R.small_case()
    z = {"planted": labels.astype(np.int32)}
    for prefix, G in (("A", A), ("B", B)):
        z.update({f"{prefix}_data": G.data, f"{prefix}_indices": G.indices, f"{prefix}_indptr": G.indptr,
                  f"{prefix}_shape": np.array(G.shape)})
    for alg, fn in (("leiden", leiden), ("louvain", louvain)):
        for name, kw in CALLS.items():
            md = mudata(A, B)
            fn(md, **kw)
            cat = md.obs[alg if alg == "leiden" else "louvain"]
            got = np.asarray(cat.astype(int))
            assert np.array_equal(got, R.renumber_by_size(labels)), (alg, name)   # the planted partition
            z[f"{alg}_{name}_labels"] = got.astype(np.int32)
            z[f"{alg}_{name}_categories"] = np.array(list(cat.cat.categories))
            z[f"{alg}_{name}_params"] = np.array(json.dumps(md.uns[alg]["params"]))
            print(alg, name, md.uns[alg]["params"])
    np.savez_compressed(os.path.join(HERE, "leiden_small.npz"), **z)
    dump_signature()


if __name__ == "__main__":
    main()
