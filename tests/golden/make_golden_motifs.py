"""Generates the motif-scanning fixtures by running the unmodified reference functions of muon/_atac/tools.py
(``get_sequences``, ``_parse_motif_ids``, ``_parse_motif_matrices``, ``_prepare_motif_scanner``, ``scan_sequences``)
with the MOODS and pybedtools stand-ins of oracle/motif_ref.py:

    python tests/golden/make_golden_motifs.py

``motifs_small.npz``:
  fasta                the synthetic genome as FASTA bytes (uint8): four contigs with line widths 60, 50, 80 and 70,
                       uneven final lines, runs of N and soft-masked (lowercase) stretches
  peaks                the ATAC feature names ``chrX:S-E`` (one past the end of chr3, one on the absent chr9)
  seq_text, seq_len    the reference's ``get_sequences`` output, concatenated, and each sequence's length
  pfm_name, pfm_len, pfm_counts   the .pfm files of the scans (40 JASPAR matrices and the edge motifs), in order;
                       the counts of all files side by side (4 x sum of lengths)
  meta_id, meta_gene   the JASPAR motif_to_gene table
  <case>|seq, |motif, |position, |score, |gene, |gene_na   the reference's hit table for each case of ``CASES``
                       (sequence index into the sequences, motif index into the files, tf_gene_name when joined)
``motifs_signature.json``: the reference signatures (read with ast), the cases, the frames' columns and dtypes, and
the exception type of every case that raises.
``jaspar_pfm.npz``: all 746 JASPAR count matrices (``names``, ``lengths``, ``counts`` 4 x 8983) and the
motif_to_gene table, a data fixture for the benchmark and the large tests.
"""
import ast
import json
import os
import sys
import tempfile
import warnings
from glob import glob

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
REF = os.environ.get("MUON_REFERENCE_ROOT", "/root/reference")
JASPAR = os.path.join(REF, "muon", "_atac", "_ref", "jaspar")

CONTIGS = (("chr1", 20_000, 60), ("chr2", 15_003, 50), ("chr3", 8_011, 80), ("chrM", 1_999, 70))
N_JASPAR = 40
# edge motifs: one column; longer than the shortest sequences; a constant (uninformative) column.  The names show the
# reference's character-set strip: "edge_len1.pfm" -> "edge_len1", "long_pfm.pfm" -> "long_"
EDGES = {
    "edge_len1.pfm": np.array([[9.0], [1.0], [1.0], [9.0]]),
    "long_pfm.pfm": None,          # filled by make_edges: 30 columns
    "const_map.pfm": None,         # a JASPAR-like motif with a constant middle column
}
CASES = {
    "default": {"pvalue": 0.0001},
    "p1e-3": {"pvalue": 0.001},
    "background": {"pvalue": 0.0005, "background": [0.3, 0.2, 0.2, 0.3]},
    "scanner": {"pvalue": 0.0001, "scanner": True},
    "pvalue_one": {"pvalue": 1.0, "subset": True},
    "no_hits": {"pvalue": 0.0001, "all_n": True},
}
SIGNATURE_NAMES = ("_parse_motif_ids", "_parse_motif_matrices", "_prepare_motif_scanner", "scan_sequences",
                   "get_sequences", "locate_file", "locate_genome")


def make_genome(seed=21):
    rng = np.random.default_rng(seed)
    lines, seqs = [], {}
    for name, length, width in CONTIGS:
        s = rng.choice(np.array(list("ACGT")), length, p=[0.3, 0.2, 0.2, 0.3])
        for a in rng.integers(0, length - 300, 4):            # runs of N
            s[a:a + int(rng.integers(5, 200))] = "N"
        for a in rng.integers(0, length - 500, 5):            # soft-masked repeats
            b = a + int(rng.integers(20, 400))
            s[a:b] = np.char.lower(s[a:b])
        s = "".join(s)
        seqs[name] = s
        lines.append(f">{name} synthetic contig")
        lines += [s[i:i + width] for i in range(0, length, width)]
    return ("\n".join(lines) + "\n").encode(), seqs


def make_peaks(seqs, seed=22):
    rng = np.random.default_rng(seed)
    peaks = []
    for name, length, _ in CONTIGS:
        for _ in range(12):
            w = int(rng.choice([8, 20, 29, 150, 500, 613]))
            a = int(rng.integers(0, length - w))
            peaks.append(f"{name}:{a}-{a + w}")
    peaks.insert(5, f"chr3:{CONTIGS[2][1] - 100}-{CONTIGS[2][1] + 50}")   # past the end of chr3
    peaks.insert(9, "chr9:100-400")                                      # contig absent from the FASTA
    peaks.append(f"chr1:0-{CONTIGS[0][2] * 3 + 7}")                      # from the contig start, across lines
    peaks.append(f"chrM:{CONTIGS[3][1] - 61}-{CONTIGS[3][1]}")           # up to the contig end (uneven last line)
    return peaks


def make_edges():
    rng = np.random.default_rng(23)
    long_ = rng.integers(0, 40, (4, 30)).astype(np.float64)
    long_[rng.integers(0, 4, 30), np.arange(30)] += 200
    const = rng.integers(0, 30, (4, 9)).astype(np.float64)
    const[np.argmax(rng.random((4, 9)), 0), np.arange(9)] += 150
    const[:, 4] = 25.0
    return {"edge_len1.pfm": EDGES["edge_len1.pfm"], "long_pfm.pfm": long_, "const_map.pfm": const}


def write_pfm(path, counts):
    with open(path, "w") as fh:
        for row in counts:
            fh.write(" ".join(f"{int(v)}" for v in row) + "\n")


def read_counts(path):
    with open(path) as fh:
        return np.array([line.split() for line in fh if line.strip()], dtype=np.float64)


def signatures():
    src = open(os.path.join(REF, "muon", "_atac", "tools.py")).read()
    out = {}
    for node in ast.parse(src).body:
        if isinstance(node, ast.FunctionDef) and node.name in SIGNATURE_NAMES:
            a = node.args
            out[node.name] = {"params": [p.arg for p in a.args], "required": len(a.args) - len(a.defaults),
                              "defaults": [ast.unparse(d) for d in a.defaults]}
    return out


def jaspar_files():
    return sorted(glob(os.path.join(JASPAR, "*.pfm")))[:N_JASPAR]


def write_jaspar_fixture():
    files = sorted(glob(os.path.join(JASPAR, "*.pfm")))
    counts = [read_counts(f) for f in files]
    meta = np.loadtxt(os.path.join(JASPAR, "motif_to_gene.txt"), dtype=str, delimiter="\t")
    np.savez_compressed(os.path.join(HERE, "jaspar_pfm.npz"), names=np.array([os.path.basename(f) for f in files]),
                        lengths=np.array([c.shape[1] for c in counts]), counts=np.concatenate(counts, axis=1),
                        meta_id=meta[:, 0], meta_gene=meta[:, 1])


def main():
    import pandas as pd

    from muon_b200._containers import SimpleAnnData
    from oracle.motif_ref import load_reference_motifs
    ref = load_reference_motifs()
    fasta, genome = make_genome()
    peaks = make_peaks(genome)
    out = {"fasta": np.frombuffer(fasta, np.uint8), "peaks": np.array(peaks)}
    errors, frames = {}, {}
    with tempfile.TemporaryDirectory() as tmp:
        fa = os.path.join(tmp, "genome.fa")
        with open(fa, "wb") as fh:
            fh.write(fasta)
        ad = SimpleAnnData(np.zeros((2, len(peaks)), np.float32), var=pd.DataFrame(index=pd.Index(peaks)))
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            seqs = ref.get_sequences(ad, None, fa)
        assert len(w) == 2, [str(x.message) for x in w]
        out["seq_text"] = np.array("".join(seqs))
        out["seq_len"] = np.array([len(s) for s in seqs])
        files = jaspar_files()
        for name, counts in make_edges().items():
            files.append(os.path.join(tmp, name))
            write_pfm(files[-1], counts)
        counts = [read_counts(f) for f in files]
        out["pfm_name"] = np.array([os.path.basename(f) for f in files])
        out["pfm_len"] = np.array([c.shape[1] for c in counts])
        out["pfm_counts"] = np.concatenate(counts, axis=1)
        meta = ref._parse_motif_ids(os.path.join(JASPAR, "motif_to_gene.txt"))
        out["meta_id"] = meta.index.to_numpy().astype(str)
        out["meta_gene"] = meta["tf_gene_name"].to_numpy().astype(str)
        for case, kw in CASES.items():
            bg = kw.get("background", 4)
            mm = ref._parse_motif_matrices(files=files, background=bg)
            ids, mats = mm["motifs"], mm["matrices"]
            case_seqs = seqs
            if kw.get("subset"):
                case_seqs = [s for s in seqs if len(s) <= 150][:6]
                ids, mats = [ids[0], ids[-3], ids[-1]], [mats[0], mats[-3], mats[-1]]
                out[f"{case}|motif_pick"] = np.array([0, len(files) - 3, len(files) - 1])
            if kw.get("all_n"):
                case_seqs = ["N" * 40, "nNRY" * 5, ""]
            try:
                if kw.get("scanner"):
                    sc = ref._prepare_motif_scanner(mats, background=bg, pvalue=kw["pvalue"])
                    df = ref.scan_sequences(case_seqs, motif_scanner=sc, motifs=ids)
                else:
                    df = ref.scan_sequences(case_seqs, matrices=mats, motifs=ids, motif_meta=meta, background=bg,
                                            pvalue=kw["pvalue"])
            except Exception as e:   # noqa: BLE001
                errors[case] = [type(e).__name__, str(e)]
                continue
            frames[case] = {"columns": list(df.columns), "dtypes": [str(t) for t in df.dtypes]}
            index_of = {id(s): i for i, s in enumerate(case_seqs)}
            out[f"{case}|seq"] = np.array([index_of[id(s)] for s in df["sequence"]], dtype=np.int64) \
                if df["sequence"].dtype == object else \
                np.array([case_seqs.index(s) for s in df["sequence"]], dtype=np.int64)
            out[f"{case}|motif"] = np.array([ids.index(m) for m in df["motif_id"]], dtype=np.int64)
            out[f"{case}|position"] = df["position"].to_numpy(np.int64)
            out[f"{case}|score"] = df["score"].to_numpy(np.float64)
            if "tf_gene_name" in df.columns:
                g = df["tf_gene_name"]
                out[f"{case}|gene"] = g.fillna("").to_numpy().astype(str)
                out[f"{case}|gene_na"] = g.isna().to_numpy()
        for case, call in (("assert_matrices", lambda: ref.scan_sequences(seqs[:2], matrices=[mats[0]])),
                           ("assert_scanner", lambda: ref.scan_sequences(seqs[:2], motif_scanner=object())),
                           ("bed_and_file", lambda: ref.get_sequences(ad, "chr1\t0\t10", fa, bed_file=fa))):
            try:
                call()
                errors[case] = None
            except Exception as e:   # noqa: BLE001
                errors[case] = [type(e).__name__, str(e)]
    np.savez_compressed(os.path.join(HERE, "motifs_small.npz"), **out)
    sig = {"signatures": signatures(), "cases": CASES, "frames": frames, "errors": errors}
    with open(os.path.join(HERE, "motifs_signature.json"), "w") as fh:
        json.dump(sig, fh, indent=1)
    write_jaspar_fixture()
    print("errors:", errors)
    print({k: len(v) for k, v in out.items() if k.endswith("|position")})
    print("npz bytes:", os.path.getsize(os.path.join(HERE, "motifs_small.npz")))


if __name__ == "__main__":
    main()
