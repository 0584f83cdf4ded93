"""CPU: the motif oracle (MOODS / pybedtools stand-ins, array restatement) against the reference-driver fixture; the
threshold DP against brute-force enumeration; log-odds; the FASTA / .fai reader; signatures; every refusal raised
before device work; the missing-database path."""
import importlib.util
import inspect
import itertools
import os
import warnings

import numpy as np
import pytest

import motif_cases as C
from muon_b200 import _motifs as T
from oracle import motif_ref as O

SEQS = C.sequences()


@pytest.fixture(scope="module")
def pfm(tmp_path_factory):
    return C.write_pfms(tmp_path_factory.mktemp("pfm"))


def test_stand_in_reproduces_fixture(pfm):
    for case, kw in C.SIG["cases"].items():
        if case in C.SIG["errors"] or kw.get("subset"):
            continue
        bg = T.background_of(kw.get("background", 4))
        mats = [O.pfm_to_log_odds(f, bg, 0.0001) for f in pfm]
        thr = [O.threshold_from_p(m, bg, kw["pvalue"]) for m in mats]
        sc = O.Scanner(10)
        sc.set_motifs(mats, bg, thr)
        rows = [(si, mi, r.pos, r.score) for si, s in enumerate(SEQS) for mi, rs in enumerate(sc.scan(s)) for r in rs]
        z = C.Z
        got = np.array([r[:3] for r in rows])
        assert np.array_equal(got[:, 2], z[f"{case}|position"]) and np.array_equal(got[:, 1], z[f"{case}|motif"])
        assert np.array_equal(np.array([r[3] for r in rows]), z[f"{case}|score"])


def test_log_odds_formula(pfm):
    bg = np.array([0.3, 0.2, 0.2, 0.3])
    for f in pfm[:5] + pfm[-3:]:
        c = T.read_pfm(f)
        s = T.log_odds(c, bg, 0.01)
        for b, j in itertools.product(range(4), range(c.shape[1])):
            want = np.log((c[b, j] + 0.01 * bg[b]) / (c[:, j].sum() + 0.01)) - np.log(bg[b])
            assert abs(s[b, j] - want) <= 1e-12 * max(1.0, abs(want))
        assert np.array_equal(s, O.pfm_to_log_odds(f, bg, 0.01))


@pytest.mark.parametrize("p", [1e-4, 1e-3, 0.05, 1.0])
def test_threshold_against_enumeration(pfm, p):
    bg = np.array([0.25, 0.25, 0.25, 0.25])
    checked = 0
    for f in pfm:
        m = T.log_odds(T.read_pfm(f), bg, 0.0001)
        L = m.shape[1]
        if L > 10:
            continue
        t = T.threshold_from_p(m, bg, p)
        words = np.stack(np.unravel_index(np.arange(4 ** L), (4,) * L), axis=1)
        S = m[words, np.arange(L)].sum(1)
        mass = bg[words].prod(1)
        tail = lambda x: mass[S >= x].sum()                      # noqa: E731
        d = T.THRESHOLD_GRID
        best = S.max()
        if mass[S >= best - 1e-12].sum() > p:                    # even the best word has mass > p: only it hits
            assert t == pytest.approx(best, abs=1e-9)
        else:
            assert tail(t + L * d) <= p * (1 + 1e-9)
            assert p == 1.0 or tail(t - d) > p
        if p == 1.0:
            assert S.min() >= t
        checked += 1
    assert checked >= 5


def test_threshold_refusals():
    m = np.zeros((4, 3))
    for p in (0.0, -1.0, 1.5):
        with pytest.raises(ValueError):
            T.threshold_from_p(m, np.full(4, 0.25), p)
    with pytest.raises(ValueError):
        T.background_of([0.5, 0.5])
    with pytest.raises(ValueError):
        T.background_of([0.3, 0.3, 0.3, 0.3])


def test_read_pfm_rejects_malformed(tmp_path):
    for text in ("1 2 3\n4 5 6\n7 8 9\n", "1 2\n3 4\n5 6\n7\n", "a b\n1 2\n3 4\n5 6\n", ""):
        p = tmp_path / "bad.pfm"
        p.write_text(text)
        with pytest.raises(ValueError):
            T.read_pfm(str(p))


def test_motif_ids_strip_like_reference(pfm):
    ids = T.parse_motif_matrices(pfm)["motifs"]
    assert ids == [os.path.basename(f).rstrip(".pfm") for f in pfm]
    assert "long_" in ids


def write_fai(path):
    """A samtools-style .fai of ``path``, from the oracle's whole-file read and the line layout."""
    text = open(path, "rb").read()
    lines = text.split(b"\n")
    off, rows, i = 0, [], 0
    while i < len(lines):
        line = lines[i]
        off += len(line) + 1
        i += 1
        if line.startswith(b">"):
            name = line[1:].split()[0].decode()
            start = off
            lb = len(lines[i]) if i < len(lines) else 0
            n = 0
            while i < len(lines) and not lines[i].startswith(b">") and lines[i]:
                n += len(lines[i])
                off += len(lines[i]) + 1
                i += 1
            rows.append(f"{name}\t{n}\t{start}\t{lb}\t{lb + 1}\n")
    with open(path + ".fai", "w") as fh:
        fh.writelines(rows)


@pytest.mark.parametrize("with_fai", [False, True])
def test_fasta_reader_matches_fixture(tmp_path, with_fai):
    fa = C.write_fasta(tmp_path)
    if with_fai:
        write_fai(fa)
    bed = "track name=peaks\n#comment\n" + "\n".join(
        p.replace(":", "-", 1).replace("-", "\t", 2) for p in map(str, C.Z["peaks"]))
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        got = T.get_fasta(bed, fa)
    assert len([x for x in w if issubclass(x.category, UserWarning)]) == 2
    assert got == SEQS
    genome = O.read_fasta(fa)
    fasta = T.Fasta(fa)
    for name, s in genome.items():
        assert fasta.index[name][0] == len(s)
        for a, b in ((0, len(s)), (len(s) - 1, len(s)), (59, 61), (0, 0)):
            assert fasta.fetch(name, a, b) == s[a:b]
    assert os.path.exists(fa + ".fai") == with_fai          # no .fai is written


def test_fasta_refusals(tmp_path):
    import gzip
    gz = tmp_path / "g.fa.gz"
    with gzip.open(gz, "wb") as fh:
        fh.write(b">c\nACGT\n")
    with pytest.raises(NotImplementedError, match="decompress"):
        T.get_fasta("c\t0\t2\n", str(gz))
    uneven = tmp_path / "u.fa"
    uneven.write_bytes(b">c\nACGT\nAC\nACGT\n")
    with pytest.raises(ValueError):
        T.get_fasta("c\t0\t2\n", str(uneven))
    ok = tmp_path / "ok.fa"
    ok.write_bytes(b">c\nACGT\nAC\n>d\nAAA\n")
    assert T.get_fasta("c\t1\t6\nd\t0\t3\n", str(ok)) == ["CGTAC", "AAA"]
    with pytest.raises(ValueError):
        T.get_fasta("c\t4\t2\n", str(ok))


def test_signatures_match_reference():
    import muon_b200 as mu
    for name, ref in C.SIG["signatures"].items():
        fn = getattr(mu.atac.tl, name)
        pos = [p for p in inspect.signature(fn).parameters.values() if p.kind == p.POSITIONAL_OR_KEYWORD]
        assert [p.name for p in pos] == ref["params"], name
        for i, (p, d) in enumerate(zip(pos[ref["required"]:], ref["defaults"])):
            assert repr(p.default) == d, (name, p.name)
        assert all(p.kind in (p.POSITIONAL_OR_KEYWORD, p.KEYWORD_ONLY) for p in inspect.signature(fn).parameters.values())


def test_refusals_before_device_work(pfm, monkeypatch):
    import muon_b200 as mu
    from muon_b200 import _lib

    def no_device(*a, **k):
        raise AssertionError("device work before the refusal")
    monkeypatch.setattr(_lib, "call", no_device)
    monkeypatch.setattr(T, "_cuda", no_device)
    mats = T.parse_motif_matrices(pfm)["matrices"]
    with pytest.raises(AssertionError, match=C.SIG["errors"]["assert_matrices"][1]):
        mu.atac.tl.scan_sequences(SEQS[:2], matrices=[mats[0]])
    with pytest.raises(AssertionError, match="motif scanner was built on"):
        mu.atac.tl.scan_sequences(SEQS[:2], motif_scanner=T.MotifScanner(mats[:2]))
    with pytest.raises(TypeError):
        mu.atac.tl.scan_sequences(SEQS[:2], motif_scanner=object(), motifs=["a"])
    with pytest.raises(NotImplementedError, match="longer than 64"):
        mu.atac.tl.scan_sequences(SEQS[:2], matrices=[np.zeros((4, 65))], motifs=["a"], motif_meta=False)
    with pytest.raises(ValueError):
        mu.atac.tl.scan_sequences(SEQS[:2], matrices=mats[:2], motifs=["a", "b"], pvalue=0.0, motif_meta=False)
    with pytest.raises(ValueError):
        mu.atac.tl.scan_sequences(SEQS[:2], matrices=[np.zeros((3, 5))], motifs=["a"], motif_meta=False)
    with pytest.raises(TypeError):
        mu.atac.tl.scan_sequences([b"ACGT"], matrices=mats[:1], motifs=["a"], motif_meta=False)
    with pytest.raises(NotImplementedError):
        monkeypatch.setattr(T, "MAX_MOTIFS", 1)
        T.MotifScanner(mats[:2])


def test_missing_database(monkeypatch, tmp_path, pfm):
    real = importlib.util.find_spec
    monkeypatch.setattr(importlib.util, "find_spec", lambda n, *a: None if n == "muon" else real(n, *a))
    import muon_b200 as mu
    with pytest.raises(FileNotFoundError, match="files="):
        mu.atac.tl._parse_motif_matrices()
    with pytest.raises(FileNotFoundError):
        mu.atac.tl._parse_motif_ids()
    with pytest.raises(FileNotFoundError):
        mu.atac.tl.scan_sequences(SEQS[:2])
    # an importable muon package with the database: the default path globs it
    pkg = tmp_path / "muon"
    jas = pkg / "_atac" / "_ref" / "jaspar"
    jas.mkdir(parents=True)
    (pkg / "__init__.py").write_text("")
    files = C.write_pfms(jas)
    C.write_meta(jas)
    spec = importlib.util.spec_from_file_location("muon", str(pkg / "__init__.py"),
                                                  submodule_search_locations=[str(pkg)])
    monkeypatch.setattr(importlib.util, "find_spec", lambda n, *a: spec if n == "muon" else real(n, *a))
    mm = mu.atac.tl._parse_motif_matrices()
    assert sorted(mm["motifs"]) == sorted(os.path.basename(f).rstrip(".pfm") for f in files)
    assert list(mu.atac.tl._parse_motif_ids().columns) == ["tf_gene_name"]


def test_locate_and_get_sequences_flow(tmp_path):
    import pandas as pd

    import muon_b200 as mu
    from muon_b200._containers import SimpleAnnData
    fa = C.write_fasta(tmp_path)
    ad = SimpleAnnData(np.zeros((1, 2), np.float32), var=pd.DataFrame(index=pd.Index(["chr1:0-10", "chr2:5-9"])))
    with pytest.raises(FileNotFoundError):
        mu.atac.tl.get_sequences(ad, None, None)
    with pytest.raises(FileNotFoundError):
        mu.atac.tl.locate_genome(ad, str(tmp_path / "missing.fa"))
    assert mu.atac.tl.get_sequences(ad, None, fa) == [O.read_fasta(fa)["chr1"][:10], O.read_fasta(fa)["chr2"][5:9]]
    assert ad.uns["files"]["genome"] == fa
    assert mu.atac.tl.get_sequences(ad, "chr1\t1\t3\n", "/nonexistent.fa") == [O.read_fasta(fa)["chr1"][1:3]]
    bed = tmp_path / "p.bed"
    bed.write_text("chr1\t2\t4\tname\n")
    assert mu.atac.tl.get_sequences(ad, None, None, bed_file=str(bed)) == [O.read_fasta(fa)["chr1"][2:4]]
    with pytest.raises(AssertionError):
        mu.atac.tl.get_sequences(ad, "chr1\t0\t1\n", None, bed_file=str(bed))
