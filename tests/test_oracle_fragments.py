"""CPU: the fragments oracle (pysam stand-in, BGZF and .tbi writers, numpy restatement) against brute force and the
reference-driver fixture; the host reader's chunking and index; signatures and the errors raised before device work."""
import gzip
import hashlib
import inspect
import json
import os
import sys
import warnings

import numpy as np
import pytest

from conftest import GOLDEN
from oracle import fragments_ref as O

sys.path.insert(0, GOLDEN)
import make_golden_fragments as M  # noqa: E402

Z = np.load(os.path.join(GOLDEN, "fragments_small.npz"))
SIG = json.load(open(os.path.join(GOLDEN, "fragments_signature.json")))
TEXT = M.make_text(Z)


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    d = tmp_path_factory.mktemp("frag")
    out = {}
    for kind in ("bgzf", "gzip", "plain"):
        out[kind] = str(O.write_fragments(str(d / f"f_{kind}.tsv.gz"), TEXT, kind=kind, block_size=4096))
    return out


def records():
    return O.parse_text(TEXT)


def oracle_records(index_of):
    return O.Records(records(), index_of)


def test_fetch_equals_brute_force(files):
    tf = O.TabixFile(files["bgzf"], parser=O.asBed())
    r = records()
    rng = np.random.default_rng(0)
    for _ in range(40):
        c = str(rng.choice(M.CONTIGS))
        a = int(rng.integers(0, 300_000))
        b = a + int(rng.integers(0, 5_000))
        got = [(f.start, f.end, f.name) for f in tf.fetch(c, a, b)]
        m = (r["contig"] == c) & (r["start"] < b) & (r["end"] > a)
        assert got == list(zip(r["start"][m].tolist(), r["end"][m].tolist(), r["name"][m].tolist()))
    assert list(tf.fetch(M.CONTIGS[0], 2e3, 4e3)) is not None
    with pytest.raises(ValueError):
        tf.fetch("chr1", -1, 10)
    with pytest.raises(ValueError):
        tf.fetch("chr9", 0, 10)
    assert tf.contigs == list(M.CONTIGS)
    assert sum(1 for _ in tf.fetch()) == len(Z["start"])


def test_bgzf_reads_back_with_gzip(files):
    for kind in ("bgzf", "gzip"):
        with gzip.open(files[kind], "rb") as fh:
            assert fh.read() == TEXT


def test_tbi_linear_index(files):
    from muon_b200 import _fragments as F
    path = files["bgzf"]
    ioff = F.read_tbi(path + ".tbi")
    coff, uoff = O.write_bgzf(path + ".again", TEXT, 4096)
    want = O.tbi_index(TEXT, coff, uoff)
    assert list(ioff) == [c for c, _, _ in want]
    for c, _, lin in want:
        assert np.array_equal(ioff[c], lin)
    # no record overlapping window w lies before ioff[w]
    starts = np.concatenate([[0], np.flatnonzero(np.frombuffer(TEXT, np.uint8) == 10)[:-1] + 1])
    blk = np.searchsorted(uoff, starts, side="right") - 1
    voff = (coff[blk].astype(np.uint64) << np.uint64(16)) | (starts - uoff[blk]).astype(np.uint64)
    r = records()
    voff = voff[len(M.HEADER):]
    for c in M.CONTIGS:
        m = r["contig"] == c
        s, e, v = r["start"][m], r["end"][m], voff[m]
        for w in range(len(ioff[c])):
            ov = (s < (w + 1) << 14) & (e > w << 14)
            if ov.any():
                assert v[ov].min() >= ioff[c][w]


@pytest.mark.parametrize("chunk", [37, 4096, 1 << 20])
def test_chunking_keeps_every_line(files, chunk):
    from concurrent.futures import ThreadPoolExecutor

    from muon_b200 import _fragments as F
    for kind, path in files.items():
        with ThreadPoolExecutor(4) as pool:
            parts = list(F.text_chunks(F.file_pieces(path, pool), chunk))
        assert all(p.endswith(b"\n") for p in parts)
        assert b"".join(parts) == TEXT, kind


def test_indexed_text_covers_windows(files):
    from muon_b200 import _fragments as F
    path = files["bgzf"]
    ioff = F.read_tbi(path + ".tbi")
    feats = M.tss_features()
    feats = feats[feats.Chromosome.isin(list(ioff))]
    windows = [(c, int(s) - 1000, int(s) + 1000) for c, s in zip(feats.Chromosome, feats.Start)]
    text = F.indexed_text(path, windows, ioff)
    sub = O.parse_text(text)
    full = records()
    key = lambda r, i: (r["contig"][i], int(r["start"][i]), int(r["end"][i]), r["name"][i])  # noqa: E731
    from collections import Counter
    got = Counter(key(sub, i) for i in range(len(sub["start"])))
    have = Counter(key(full, i) for i in range(len(full["start"])))
    assert all(have[k] == n for k, n in got.items())          # no record read twice (the file has exact repeats)
    for c, lo, hi in windows:
        m = np.flatnonzero((full["contig"] == c) & (full["start"] < hi) & (full["end"] > lo))
        assert all(key(full, i) in got for i in m)
    assert len(text) < len(TEXT)


def test_corrupt_tbi_falls_back(files, tmp_path):
    import shutil

    from muon_b200 import _fragments as F
    path = str(tmp_path / "c.tsv.gz")
    shutil.copy(files["bgzf"], path)
    ioff = F.read_tbi(files["bgzf"] + ".tbi")
    bad = {c: v + np.uint64(3) for c, v in ioff.items()}
    with pytest.warns(UserWarning):
        assert F.indexed_text(path, [("chr1", 100_000, 102_000)], bad) is None


def index_of_obs(ad, barcodes=None):
    from muon_b200.atac.tl import _barcode_rows
    return _barcode_rows(ad, barcodes)


@pytest.mark.parametrize("case", list(SIG["count"]))
def test_numpy_count_equals_fixture(case):
    import scipy.sparse as sp
    if f"count|{case}" in SIG["errors"]:
        pytest.skip("the reference raises")
    kw = dict(SIG["count"][case])
    kind = kw.pop("features", "plain")
    feats = M.features_for(kind) if kind is not None else M.features_for("plain")
    up, down = kw.get("extend_upstream", 2000), kw.get("extend_downstream", 0)
    windows = [(c, s - up, e + down) for c, s, e in zip(feats.Chromosome, feats.Start, feats.End)]
    R = oracle_records(index_of_obs(M.make_adata()))
    got = O.count_ref(R, windows, M.N_CELLS, kw.get("count_reads", True))
    want = sp.csr_matrix((Z[f"count|{case}|data"], Z[f"count|{case}|indices"], Z[f"count|{case}|indptr"]),
                         shape=got.shape)
    assert (got != want).nnz == 0


@pytest.mark.parametrize("case", ["all", "barcodes", "nan", "no_return"])
def test_numpy_tss_equals_fixture(case):
    kw = SIG["tss"][case]
    up, down = kw.get("extend_upstream", 1000), kw.get("extend_downstream", 1000)
    feats = M.tss_features()
    feats = feats[feats.Chromosome.isin(M.CONTIGS)]
    R = oracle_records(index_of_obs(M.make_adata(), kw.get("barcodes")))
    X, score, _ = O.tss_ref(R, list(zip(feats.Chromosome, feats.Start)), M.N_CELLS, up, down)
    assert np.array_equal(score, Z[f"tss|{case}|score"], equal_nan=True)
    if f"tss|{case}|X_sha256" in Z.files:
        assert hashlib.sha256(np.ascontiguousarray(X).tobytes()).hexdigest() == str(Z[f"tss|{case}|X_sha256"])


@pytest.mark.parametrize("case", list(SIG["nucleosome"]))
def test_numpy_nucleosome_equals_fixture(case):
    kw = dict(SIG["nucleosome"][case])
    n = int(kw.pop("n", M.N_CELLS * 1e4))
    R = oracle_records(index_of_obs(M.make_adata(), kw.pop("barcodes", None)))
    if f"nuc|{case}" in SIG["errors"]:
        with pytest.raises(StopIteration):
            O.nucleosome_ref(R, n, M.N_CELLS)
        return
    got = O.nucleosome_ref(R, n, M.N_CELLS, kw.get("nucleosome_free_upper_bound", 147),
                           kw.get("mononuleosomal_upper_bound", 294))
    assert np.array_equal(got, Z[f"nuc|{case}"])


def test_fixture_expected_errors():
    assert SIG["errors"] == {"count|strand_false": "KeyError", "count|near_start": "ValueError",
                             "count|absent_contig": "ValueError", "tss|narrow": "ValueError",
                             "nuc|default_n": "StopIteration"}


@pytest.mark.parametrize("name", ["locate_fragments", "count_fragments_features", "tss_enrichment",
                                  "nucleosome_signal"])
def test_signature_matches_reference(name):
    import muon_b200 as mu
    ref = SIG["signatures"][name]
    sig = inspect.signature(getattr(mu.atac.tl, name))
    pos = [p for p in sig.parameters.values() if p.kind == p.POSITIONAL_OR_KEYWORD]
    assert [p.name for p in pos] == ref["params"]
    for i, p in enumerate(pos):
        if i < ref["required"]:
            assert p.default is inspect.Parameter.empty
        else:
            assert repr(p.default) == ref["defaults"][i - ref["required"]], (name, p.name)
    assert all(p.kind == p.KEYWORD_ONLY for p in sig.parameters.values() if p.kind != p.POSITIONAL_OR_KEYWORD)


def test_errors_before_device_work(files):
    import muon_b200 as mu
    from muon_b200._containers import SimpleMuData
    tl = mu.atac.tl
    with pytest.raises(TypeError):
        tl.count_fragments_features(np.zeros(3), M.features_for("plain"))
    with pytest.raises(TypeError):
        tl.nucleosome_signal(SimpleMuData({"rna": M.make_adata()}))
    with pytest.raises(ValueError):
        tl.count_fragments_features(M.make_adata(files["bgzf"]))
    with pytest.raises(ValueError):
        tl.tss_enrichment(M.make_adata(files["bgzf"]))
    with pytest.raises(KeyError):
        tl.count_fragments_features(M.make_adata(), M.features_for("plain"))
    with pytest.raises(KeyError):
        tl.tss_enrichment(M.make_adata(), M.tss_features())
    with pytest.raises(KeyError):
        tl.nucleosome_signal(M.make_adata())
    with pytest.warns(FutureWarning), pytest.raises(KeyError):
        tl.count_fragments_features(M.make_adata(files["bgzf"]), M.features_for("strand"))
    with pytest.warns(FutureWarning), pytest.raises(ValueError):
        tl.count_fragments_features(M.make_adata(files["bgzf"]), M.features_for("near_start"))
    with pytest.raises(ValueError):
        tl.count_fragments_features(M.make_adata(files["bgzf"]), M.features_for("plain").drop(columns="End"),
                                    count_reads=False)
    ad = M.make_adata(files["bgzf"])
    ad.obs.index = ["same"] * M.N_CELLS
    with pytest.raises(ValueError):
        tl.count_fragments_features(ad, M.features_for("plain"), count_reads=False)


def test_locate_fragments_prints(files, capsys):
    import muon_b200 as mu
    ad = M.make_adata()
    assert mu.atac.tl.locate_fragments(ad, files["bgzf"]) is None
    assert ad.uns["files"]["fragments"] == files["bgzf"]
    assert mu.atac.tl.locate_fragments(ad, files["bgzf"] + ".missing") is None
    assert "missing" in capsys.readouterr().out
    assert ad.uns["files"]["fragments"] == files["bgzf"]
    mu.atac.tl.locate_fragments(np.zeros(2), files["bgzf"])
    assert "Expected AnnData" in capsys.readouterr().out
    try:
        import pysam  # noqa: F401
    except ImportError:
        assert mu.atac.tl.locate_fragments(ad, files["bgzf"], return_fragments=True) is None
        assert "pysam" in capsys.readouterr().out


def test_gene_annotation_from_rna_matches_reference():
    try:
        ref = O.load_reference_fragments()
    except FileNotFoundError:
        pytest.skip("reference sources not present")
    from muon_b200.atac.tl import _gene_annotation_from_rna
    md = M.make_mudata()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        want = ref.get_gene_annotation_from_rna(md)
    got = _gene_annotation_from_rna(md)
    assert list(got.columns) == list(want.columns)
    assert list(got.index) == list(want.index)
    for c in got.columns:
        assert list(got[c]) == list(want[c])
