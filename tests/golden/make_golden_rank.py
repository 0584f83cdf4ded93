"""Generates the differential-accessibility fixtures by running the unmodified reference functions of
muon/_atac/tools.py (``add_peak_annotation`` and ``rank_peaks_groups``) with oracle/rank_ref.py standing in for
``scanpy.tl.rank_genes_groups``:

    python tests/golden/make_golden_rank.py

``rank_small.npz``: 360 cells x 800 peaks of small integer counts with 40 planted differential peaks per group over 5
groups of unequal sizes (the last 10 peaks all zero), and for every case of ``CASES`` the reference's
``uns["rank_genes_groups"]``, ranked names stored as peak indices.  Not stored, because they are functions of the
counts: the float64 ``scaled`` layer (``scaled_layer``) and the annotation table (``annotation_tsv``: multi-gene ``;``
rows and an intergenic row).  Case ``unannotated`` drops the annotation of a ranked peak: the reference raises after
writing the ranking.
``rank_signature.json``: the four reference signatures (read with ast) and the cases.
"""
import io
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

CASES = {
    "ttest": {},
    "overestim_bonferroni": {"method": "t-test_overestim_var", "corr_method": "bonferroni", "n_genes": 50},
    "wilcoxon_pts": {"method": "wilcoxon", "pts": True},
    "wilcoxon_tie_abs_layer": {"method": "wilcoxon", "tie_correct": True, "rankby_abs": True, "layer": "scaled"},
    "wilcoxon_ref": {"method": "wilcoxon", "reference": "1", "groups": ["3", "0", "1"], "tie_correct": True,
                     "pts": True, "n_genes": 300},
    "ttest_ref_types": {"method": "t-test", "reference": "2", "n_genes": 100, "add_peak_type": True,
                        "add_distance": True},
    "ttest_layer_pts": {"layer": "scaled", "pts": True, "n_genes": 200},
    "unannotated": {"method": "wilcoxon", "n_genes": 20},
}
SIZES = (120, 90, 70, 50, 30)
N_PEAKS = 800


def make_data(seed=7):
    import scipy.sparse as sp
    rng = np.random.default_rng(seed)
    n, d = sum(SIZES), N_PEAKS
    labels = np.repeat(np.arange(len(SIZES)), SIZES)
    rng.shuffle(labels)
    p = np.full((len(SIZES), d), 0.04)
    for g in range(len(SIZES)):
        p[g, 40 * g: 40 * g + 40] = 0.5
    p[:, d - 10:] = 0.0                                 # all-zero peaks
    P = p[labels]
    C = (rng.random((n, d)) < P) * rng.integers(1, 4, size=(n, d))
    X = sp.csr_matrix(C.astype(np.float32))
    return X, scaled_layer(X), labels


def scaled_layer(X):
    """float64 layer with negative values (ranked below the implicit zeros) and ties among them; dyadic values, so that
    every sum is exact in float64 and the fixture does not depend on summation order."""
    return np.choose(X.toarray().astype(np.int64), [0.0, -1.125, 2.5, 3.375]).astype(np.float64)


def peak_names(d):
    return [f"chr{1 + i // 1000}:{1000 * (i % 1000)}-{1000 * (i % 1000) + 500}" for i in range(d)]


def annotation_tsv(d, drop=None):
    rows = ["peak\tgene\tdistance\tpeak_type"]
    for i, name in enumerate(peak_names(d)):
        if i == drop:
            continue
        chrom, rest = name.split(":")
        start, end = rest.split("-")
        peak = f"{chrom}_{start}_{end}"
        if i % 7 == 0:
            rows.append(f"{peak}\tG{i};G{i + 1}\t-{i};{2 * i}\tpromoter;distal")
        elif i == 5:
            rows.append(f"{peak}\t\t12000\tintergenic")
        else:
            rows.append(f"{peak}\tG{i}\t{i % 300}\t{'promoter' if i % 2 else 'distal'}")
    return "\n".join(rows) + "\n"


def make_adata(X, scaled, labels):
    import pandas as pd

    from muon_b200 import SimpleAnnData
    ad = SimpleAnnData(X.copy(), var=peak_names(X.shape[1]), layers={"scaled": scaled.copy()})
    ad.obs["leiden"] = pd.Categorical([str(v) for v in labels], categories=[str(i) for i in range(len(SIZES))])
    return ad


def flatten(prefix, uns, z):
    """uns["rank_genes_groups"] -> npz entries (ranked names as peak indices, other strings as unicode arrays)."""
    index = {name: i for i, name in enumerate(peak_names(N_PEAKS))}
    for key, val in uns.items():
        if key == "params":
            z[f"{prefix}|params"] = np.array(json.dumps(val))
        elif key in ("pts", "pts_rest"):
            assert list(val.index) == peak_names(N_PEAKS)
            z[f"{prefix}|{key}"] = val.to_numpy()
            z[f"{prefix}|{key}|columns"] = np.array(list(val.columns))
        elif isinstance(val, dict):                  # peak_type / distance, or genes when building them raised
            for g, arr in val.items():
                z[f"{prefix}|{key}|{g}"] = np.array([str(x) for x in arr])
        else:                                        # recarrays
            for g in val.dtype.names:
                col = val[g]
                if key == "names":
                    col = np.array([index[x] for x in col], dtype=np.int16)
                elif col.dtype == object:
                    col = np.array([str(x) for x in col])
                z[f"{prefix}|{key}|{g}"] = col


def main():
    from oracle.rank_ref import load_reference_rank_peaks_groups, rank_genes_groups, reference_signatures
    rank_peaks_groups, _, add_peak_annotation, _ = load_reference_rank_peaks_groups()
    import pandas as pd
    X, scaled, labels = make_data()
    z = {"X_data": X.data.astype(np.uint8), "X_indices": X.indices.astype(np.int16), "X_indptr": X.indptr,
         "X_shape": np.array(X.shape), "labels": labels.astype(np.int8)}
    for name, kw in CASES.items():
        kw = dict(kw)
        ad = make_adata(X, scaled, labels)
        drop = None
        if name == "unannotated":                    # group 0's best peak: in its top list, not in the others'
            probe = make_adata(X, scaled, labels)
            rank_genes_groups(probe, "leiden", **kw)
            drop = peak_names(X.shape[1]).index(probe.uns["rank_genes_groups"]["names"]["0"][0])
            z["unannotated_drop"] = np.array(drop)
        add_peak_annotation(ad, pd.read_csv(io.StringIO(annotation_tsv(X.shape[1], drop)), sep="\t"))
        try:
            rank_peaks_groups(ad, "leiden", **kw)
            z[f"{name}|error"] = np.array("")
        except Exception as e:                       # noqa: BLE001 -- the case records which exception the reference raises
            z[f"{name}|error"] = np.array(type(e).__name__)
            print(name, "raised", type(e).__name__, e)
        flatten(name, ad.uns["rank_genes_groups"], z)
        print(name, "ok")
    np.savez_compressed(os.path.join(HERE, "rank_small.npz"), **z)
    sig = reference_signatures()
    json.dump({"signatures": sig, "cases": CASES}, open(os.path.join(HERE, "rank_signature.json"), "w"), indent=1)


def load_counts(z):
    """The fixture's count matrix (float32 CSR) and labels."""
    import scipy.sparse as sp
    X = sp.csr_matrix((z["X_data"].astype(np.float32), z["X_indices"].astype(np.int32), z["X_indptr"]),
                      shape=tuple(z["X_shape"]))
    return X, z["labels"].astype(np.int64)


if __name__ == "__main__":
    main()
