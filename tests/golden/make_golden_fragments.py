"""Generates the fragments-file fixtures by running the unmodified reference functions of muon/_atac/tools.py
(``locate_fragments``, ``count_fragments_features``, ``tss_enrichment``, ``nucleosome_signal``) with the pysam
stand-in of oracle/fragments_ref.py:

    python tests/golden/make_golden_fragments.py

``fragments_small.npz``: a synthetic, coordinate-sorted fragments file of ~1e5 fragments on three contigs (two ``#``
header lines, scores 1-5, a nucleosomal length mixture, 300 obs cells plus 50 foreign barcodes, fragments piled up
around planted TSSs, one obs cell without fragments), stored as columns (``make_text`` rebuilds the text; tests write
it as BGZF + ``.tbi``, plain gzip or plain text), and the reference's output for every case of ``CASES``:
  count|<case>|{data,indices,indptr}  the reference's X, canonicalised (duplicates summed, indices sorted)
  tss|<case>|{score,shape,X_sha256}  obs["tss_score"], and the shape and sha256 of the returned float64 X
  nuc|<case>  obs["nucleosome_signal"]
A case the reference raises on stores the exception type in ``fragments_signature.json`` instead.
``fragments_signature.json``: the four reference signatures (read with ast) and the cases.
"""
import ast
import hashlib
import json
import os
import sys
import tempfile
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

CONTIGS = ("chr1", "chr2", "chr3")
CONTIG_LEN = (600_000, 400_000, 300_000)
N_FRAG = 100_000
N_CELLS, N_FOREIGN = 300, 50
HEADER = ("# id=synthetic-fragments", "# description=tests/golden/make_golden_fragments.py")

COUNT_CASES = {
    "default": {},
    "fragments": {"count_reads": False},
    "ext_0_0": {"extend_upstream": 0, "extend_downstream": 0},
    "ext_2000_500": {"extend_upstream": 2000, "extend_downstream": 500},
    "strand_true": {"stranded": True, "features": "strand"},
    "strand_false": {"stranded": False, "features": "strand"},
    "near_start": {"features": "near_start"},
    "absent_contig": {"features": "absent"},
    "from_rna": {"features": None},
}
TSS_CASES = {
    "all": {},
    "sample": {"n_tss": 15, "random_state": 3},
    "barcodes": {"barcodes": "bc"},
    "nan": {"extend_upstream": 500, "extend_downstream": 500},
    "narrow": {"extend_upstream": 300, "extend_downstream": 300},
    "no_return": {"return_tss": False},
}
NUC_CASES = {
    "n20000": {"n": 20000},
    "bounds": {"n": 50000, "nucleosome_free_upper_bound": 100, "mononuleosomal_upper_bound": 250},
    "barcodes": {"n": 30000.0, "barcodes": "bc"},
    "default_n": {},
}


def barcodes():
    return [f"CELL{i:04d}-1" for i in range(N_CELLS)] + [f"FOREIGN{i:03d}-1" for i in range(N_FOREIGN)]


def make_genes(seed=5):
    """Gene table: Chromosome, Start, End, Strand; overlapping genes on the three contigs (Start >= 2000)."""
    import pandas as pd
    rng = np.random.default_rng(seed)
    rows = []
    for c, L in zip(CONTIGS, CONTIG_LEN):
        for _ in range(20):
            s = int(rng.integers(2_000, L - 40_000))
            rows.append((c, s, s + int(rng.integers(1_500, 30_000)), "+" if rng.random() < 0.5 else "-"))
    rows.append(("chr1", 100_000, 130_000, "+"))          # overlaps planted genes
    rows.append(("chr1", 110_000, 112_000, "-"))
    g = pd.DataFrame(rows, columns=["Chromosome", "Start", "End", "Strand"])
    g.index = [f"gene{i}" for i in range(len(g))]
    return g


def features_for(kind):
    g = make_genes()
    if kind == "strand":
        return g
    base = g.drop(columns="Strand")
    if kind == "near_start":
        extra = base.iloc[:1].copy()
        extra.iloc[0] = ["chr2", 800, 5_000]
        extra.index = ["gene_near_start"]
        return __import__("pandas").concat([base, extra])
    if kind == "absent":
        extra = base.iloc[:2].copy()
        extra["Chromosome"] = "chr9"
        extra.index = ["gene_chr9a", "gene_chr9b"]
        return __import__("pandas").concat([base, extra])
    return base


def tss_features():
    """TSS table (Chromosome, Start, End): every gene, plus three on a contig the file lacks."""
    import pandas as pd
    g = make_genes().drop(columns="Strand")
    extra = pd.DataFrame({"Chromosome": ["chr9"] * 3, "Start": [5_000, 9_000, 20_000], "End": [6_000, 10_000, 21_000]},
                         index=["t9a", "t9b", "t9c"])
    return pd.concat([g, extra])


def make_fragments(seed=11):
    rng = np.random.default_rng(seed)
    genes = make_genes()
    n_cell_bc = N_CELLS - 1                                  # the last obs cell has no fragment
    contig, start, length, bc, score = [], [], [], [], []
    per = np.array(CONTIG_LEN) / sum(CONTIG_LEN)
    counts = rng.multinomial(N_FRAG, per)
    for ci, (c, L, n) in enumerate(zip(CONTIGS, CONTIG_LEN, counts)):
        tss = genes.loc[genes.Chromosome == c, "Start"].to_numpy()
        near = rng.random(n) < 0.5
        s = rng.integers(0, L - 1000, n)
        s[near] = np.clip(rng.choice(tss, near.sum()) + rng.normal(0, 120, near.sum()).astype(np.int64) - 60, 0,
                          L - 1000)
        s[:3] = [0, 5, 40]                                   # fragments at the contig start
        kind = rng.random(n)
        ln = np.where(kind < 0.6, np.clip(rng.normal(80, 30, n), 20, 146),
                      np.where(kind < 0.9, rng.integers(147, 295, n), rng.integers(295, 800, n))).astype(np.int64)
        b = np.where(rng.random(n) < 0.9, rng.integers(0, n_cell_bc, n), rng.integers(N_CELLS, N_CELLS + N_FOREIGN, n))
        order = np.argsort(s, kind="stable")
        contig.append(np.full(n, ci, np.uint8))
        start.append(s[order])
        length.append(ln[order])
        bc.append(b[order])
        score.append(rng.integers(1, 6, n)[order])
    return {"contig": np.concatenate(contig), "start": np.concatenate(start).astype(np.int32),
            "length": np.concatenate(length).astype(np.uint16), "bc": np.concatenate(bc).astype(np.uint16),
            "score": np.concatenate(score).astype(np.uint8)}


def make_text(Z, header=True) -> bytes:
    from oracle.fragments_ref import format_text
    names = np.array(barcodes(), dtype=object)
    st = Z["start"].astype(np.int64)
    return format_text(np.array(CONTIGS, dtype=object)[Z["contig"]], st, st + Z["length"], names[Z["bc"]], Z["score"],
                       HEADER if header else ())


def obs_frame():
    """obs of the ATAC AnnData: index = the obs barcodes; column ``bc`` = a permutation of them with one repeat."""
    import pandas as pd
    names = barcodes()[:N_CELLS]
    rng = np.random.default_rng(3)
    bc = list(np.array(names)[rng.permutation(N_CELLS)])
    bc[7] = bc[200]                                          # a repeated barcode: the later row wins
    return pd.DataFrame({"bc": bc}, index=pd.Index(names))


def make_adata(path=None):
    from muon_b200._containers import SimpleAnnData
    ad = SimpleAnnData(np.zeros((N_CELLS, 1), np.float32), obs=obs_frame())
    if path is not None:
        ad.uns["files"] = {"fragments": str(path)}
    return ad


def make_mudata(path=None):
    import pandas as pd

    from muon_b200._containers import SimpleAnnData, SimpleMuData
    g = features_for("plain")
    var = pd.DataFrame({"gene_ids": [f"ENSG{i:05d}" for i in range(len(g))],
                        "interval": [f"{c}:{s}-{e}" for c, s, e in zip(g.Chromosome, g.Start, g.End)]}, index=g.index)
    rna = SimpleAnnData(np.zeros((N_CELLS, len(g)), np.float32), obs=obs_frame(), var=var)
    return SimpleMuData({"atac": make_adata(path), "rna": rna})


def csr_parts(X):
    import scipy.sparse as sp
    m = sp.csr_matrix(X, dtype=np.int64)
    m.sum_duplicates()
    m.sort_indices()
    return m.data, m.indices, m.indptr


def signatures():
    src = open(os.path.join(os.environ.get("MUON_REFERENCE_ROOT", "/root/reference"), "muon", "_atac", "tools.py")).read()
    out = {}
    for node in ast.parse(src).body:
        if isinstance(node, ast.FunctionDef) and node.name in ("locate_fragments", "count_fragments_features",
                                                               "tss_enrichment", "nucleosome_signal"):
            a = node.args
            out[node.name] = {"params": [p.arg for p in a.args], "required": len(a.args) - len(a.defaults),
                              "defaults": [ast.unparse(d) for d in a.defaults]}
    return out


def main():
    from oracle.fragments_ref import load_reference_fragments, write_fragments
    os.environ.setdefault("TQDM_DISABLE", "1")
    ref = load_reference_fragments()
    Z = make_fragments()
    out = dict(Z)
    errors = {}
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "fragments.tsv.gz")
        write_fragments(path, make_text(Z))
        for name, kw in COUNT_CASES.items():
            kw = dict(kw)
            kind = kw.pop("features", "plain")
            data = make_mudata() if kind is None else make_adata()
            ref.locate_fragments(data, path)
            feats = None if kind is None else features_for(kind)
            try:
                with warnings.catch_warnings():
                    warnings.simplefilter("ignore")
                    res = ref.count_fragments_features(data, feats, **kw)
            except Exception as e:   # noqa: BLE001
                errors[f"count|{name}"] = type(e).__name__
                continue
            for k, v in zip(("data", "indices", "indptr"), csr_parts(res.X)):
                out[f"count|{name}|{k}"] = v
        for name, kw in TSS_CASES.items():
            ad = make_adata()
            ref.locate_fragments(ad, path)
            try:
                with warnings.catch_warnings():
                    warnings.simplefilter("ignore")
                    res = ref.tss_enrichment(ad, tss_features(), **kw)
            except Exception as e:   # noqa: BLE001
                errors[f"tss|{name}"] = type(e).__name__
                continue
            out[f"tss|{name}|score"] = ad.obs["tss_score"].to_numpy()
            if res is not None:
                X = np.ascontiguousarray(res.X, dtype=np.float64)
                out[f"tss|{name}|X_sha256"] = np.array(hashlib.sha256(X.tobytes()).hexdigest())
                out[f"tss|{name}|shape"] = np.array(X.shape)
        for name, kw in NUC_CASES.items():
            ad = make_adata()
            ref.locate_fragments(ad, path)
            try:
                ref.nucleosome_signal(ad, **kw)
            except Exception as e:   # noqa: BLE001
                errors[f"nuc|{name}"] = type(e).__name__
                continue
            out[f"nuc|{name}"] = ad.obs["nucleosome_signal"].to_numpy()
    np.savez_compressed(os.path.join(HERE, "fragments_small.npz"), **out)
    sig = {"signatures": signatures(), "count": COUNT_CASES, "tss": TSS_CASES, "nucleosome": NUC_CASES,
           "errors": errors}
    with open(os.path.join(HERE, "fragments_signature.json"), "w") as fh:
        json.dump(sig, fh, indent=1, default=str)
    print("errors:", errors)
    print("npz bytes:", os.path.getsize(os.path.join(HERE, "fragments_small.npz")))


if __name__ == "__main__":
    main()
