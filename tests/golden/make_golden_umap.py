"""Generates the UMAP fixtures from oracle/umap_ref.py (recalled umap-learn, numba on the CPU):

    python tests/golden/make_golden_umap.py

``umap_small.npz``: a planted-cluster graph (6 Gaussian clusters, 1500 cells in 10 dimensions, exact 15-NN,
umap connectivities from oracle._third_party.umap_connectivities) as CSR, its representation and labels, the
sequential umap-learn layout ``layout_ref`` (default arguments, random_state=42) and that layout's
trustworthiness and kNN label agreement (k = 15).
``umap_signature.json``: the reference signature of ``muon.tl.umap`` (read with ast).
"""
import ast
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle.umap_ref import find_ab, knn_label_agreement, layout_ref, planted_graph, trustworthiness  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
K = 15


def dump_signature():
    tree = ast.parse(open(os.path.join(os.environ.get("MUON_REFERENCE_ROOT", "/root/reference"),
                                       "muon/_core/tools.py")).read())
    fn = next(n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "umap")
    params = [a.arg for a in fn.args.args]
    defaults = [ast.literal_eval(d) for d in fn.args.defaults]
    required = len(params) - len(defaults)
    out = {"umap": {"params": params, "defaults": [repr(None)] * required + [repr(d) for d in defaults],
                    "required": required}}
    json.dump(out, open(os.path.join(OUT, "umap_signature.json"), "w"), indent=1)


def main():
    X, labels, W = planted_graph()
    a, b = find_ab(1.0, 0.5)
    Y = layout_ref(W, a=a, b=b, random_state=42)
    z = {"rep": X, "labels": labels.astype(np.int32), "layout_ref": Y,
         "W_data": W.data, "W_indices": W.indices, "W_indptr": W.indptr, "W_shape": np.array(W.shape),
         "trust_ref": trustworthiness(X, Y, K), "label_ref": knn_label_agreement(Y, labels, K)}
    path = os.path.join(OUT, "umap_small.npz")
    np.savez_compressed(path, **z)
    print(os.path.basename(path), os.path.getsize(path), float(z["trust_ref"]), float(z["label_ref"]))
    dump_signature()


if __name__ == "__main__":
    main()
