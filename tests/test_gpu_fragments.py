"""GPU: ``count_fragments_features``, ``tss_enrichment`` and ``nucleosome_signal`` reproduce the reference run recorded
in tests/golden/fragments_small.npz exactly, from BGZF (full pass and through the .tbi), plain gzip and plain text, with
lines straddling tiny chunks; the parse equals a host parse; repeated calls are bit-identical; a 1e7-fragment file
matches the numpy restatement."""
import hashlib
import json
import os
import sys
import warnings

import numpy as np
import pytest
import scipy.sparse as sp

from conftest import GOLDEN
from oracle import fragments_ref as O

pytestmark = pytest.mark.gpu
sys.path.insert(0, GOLDEN)
import make_golden_fragments as M  # noqa: E402

Z = np.load(os.path.join(GOLDEN, "fragments_small.npz"))
SIG = json.load(open(os.path.join(GOLDEN, "fragments_signature.json")))
TEXT = M.make_text(Z)
READS = [("bgzf", None), ("bgzf", 4096), ("gzip", None), ("plain", 777)]     # (encoding, chunk_bytes)


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    d = tmp_path_factory.mktemp("fraggpu")
    return {k: str(O.write_fragments(str(d / f"f_{k}.tsv.gz"), TEXT, kind=k, block_size=8192))
            for k in ("bgzf", "gzip", "plain")}


def expect_error(key):
    return {"KeyError": KeyError, "ValueError": ValueError, "StopIteration": StopIteration}[SIG["errors"][key]]


@pytest.mark.parametrize("kind,chunk", READS)
@pytest.mark.parametrize("case", list(SIG["count"]))
def test_count_matches_fixture(cuda, files, case, kind, chunk):
    import muon_b200 as mu
    kw = dict(SIG["count"][case])
    feat = kw.pop("features", "plain")
    data = M.make_mudata(files[kind]) if feat is None else M.make_adata(files[kind])
    feats = None if feat is None else M.features_for(feat)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", FutureWarning)
        if f"count|{case}" in SIG["errors"]:
            with pytest.raises(expect_error(f"count|{case}")):
                mu.atac.tl.count_fragments_features(data, feats, **kw, chunk_bytes=chunk)
            return
        res = mu.atac.tl.count_fragments_features(data, feats, **kw, chunk_bytes=chunk)
    X = res.X
    assert sp.isspmatrix_csr(X) and X.dtype == np.int64 and X.has_canonical_format
    assert np.array_equal(X.data, Z[f"count|{case}|data"])
    assert np.array_equal(X.indices, Z[f"count|{case}|indices"])
    assert np.array_equal(X.indptr, Z[f"count|{case}|indptr"])
    assert list(res.obs.index) == list(M.obs_frame().index)
    assert res.var.shape[0] == X.shape[1]


@pytest.mark.parametrize("kind,chunk,use_index", [("bgzf", None, True), ("bgzf", 5000, False), ("gzip", None, True),
                                                  ("plain", 999, True)])
@pytest.mark.parametrize("case", list(SIG["tss"]))
def test_tss_matches_fixture(cuda, files, case, kind, chunk, use_index):
    import muon_b200 as mu
    kw = SIG["tss"][case]
    ad = M.make_adata(files[kind])
    if f"tss|{case}" in SIG["errors"]:
        with pytest.raises(expect_error(f"tss|{case}")):
            mu.atac.tl.tss_enrichment(ad, M.tss_features(), **kw, use_index=use_index, chunk_bytes=chunk)
        return
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        res = mu.atac.tl.tss_enrichment(ad, M.tss_features(), **kw, use_index=use_index, chunk_bytes=chunk)
    assert np.array_equal(ad.obs["tss_score"].to_numpy(), Z[f"tss|{case}|score"], equal_nan=True)
    if kw.get("return_tss", True):
        X = np.ascontiguousarray(res.X)
        assert X.dtype == np.float64 and X.shape == tuple(Z[f"tss|{case}|shape"])
        assert hashlib.sha256(X.tobytes()).hexdigest() == str(Z[f"tss|{case}|X_sha256"])
        assert list(res.var.index) == [str(i) for i in range(X.shape[1])]
        assert res.var["TSS_position"].iloc[0] == -kw.get("extend_upstream", 1000)
        assert np.array_equal(res.obs["tss_score"].to_numpy(), Z[f"tss|{case}|score"], equal_nan=True)
    else:
        assert res is None


@pytest.mark.parametrize("kind,chunk", READS)
@pytest.mark.parametrize("case", list(SIG["nucleosome"]))
def test_nucleosome_matches_fixture(cuda, files, case, kind, chunk):
    import muon_b200 as mu
    ad = M.make_adata(files[kind])
    kw = SIG["nucleosome"][case]
    if f"nuc|{case}" in SIG["errors"]:
        with pytest.raises(expect_error(f"nuc|{case}")):
            mu.atac.tl.nucleosome_signal(ad, **kw, chunk_bytes=chunk)
        return
    assert mu.atac.tl.nucleosome_signal(ad, **kw, chunk_bytes=chunk) is None
    assert np.array_equal(ad.obs["nucleosome_signal"].to_numpy(), Z[f"nuc|{case}"])


def test_corrupt_tbi_warns_and_matches(cuda, files, tmp_path):
    import shutil

    import muon_b200 as mu
    path = str(tmp_path / "c.tsv.gz")
    shutil.copy(files["bgzf"], path)
    coff, uoff = O.write_bgzf(str(tmp_path / "tmp.gz"), TEXT, 8192)
    idx = O.tbi_index(TEXT, coff, uoff)
    idx = [(c, bins, lin + np.uint64(5)) for c, bins, lin in idx]        # in-block offsets off the line starts
    import struct
    nm = b"".join(c.encode() + b"\0" for c, _, _ in idx)
    body = [b"TBI\x01", struct.pack("<iiiiiiii", len(idx), O.TBX_UCSC, 1, 2, 3, ord("#"), 0, len(nm)), nm]
    for _, _, lin in idx:
        body += [struct.pack("<i", 0), struct.pack("<i", len(lin)), lin.astype("<u8").tobytes()]
    with open(path + ".tbi", "wb") as fh:
        fh.write(O.bgzf_block(b"".join(body)) + O.BGZF_EOF)
    ad = M.make_adata(path)
    with pytest.warns(UserWarning):
        mu.atac.tl.tss_enrichment(ad, M.tss_features())
    assert np.array_equal(ad.obs["tss_score"].to_numpy(), Z["tss|all|score"], equal_nan=True)


def test_unsorted_file_raises(cuda, tmp_path):
    import muon_b200 as mu
    lines = TEXT.split(b"\n")
    body = lines[len(M.HEADER):-1]
    swapped = body[:100] + [body[200]] + body[101:200] + [body[100]] + body[201:]
    path = O.write_fragments(str(tmp_path / "u.tsv"), b"\n".join(swapped) + b"\n", kind="plain")
    with pytest.raises(ValueError):
        mu.atac.tl.nucleosome_signal(M.make_adata(path), n=1000)
    # a contig that comes back after another one
    c1 = [ln for ln in body if ln.startswith(b"chr1\t")]
    c2 = [ln for ln in body if ln.startswith(b"chr2\t")]
    path = O.write_fragments(str(tmp_path / "u2.tsv"), b"\n".join(c1[:50] + c2 + c1[50:]) + b"\n", kind="plain")
    with pytest.raises(ValueError):
        mu.atac.tl.count_fragments_features(M.make_adata(path), M.features_for("plain"), count_reads=False)


def test_parse_equals_host_parse(cuda, files):
    import torch

    from muon_b200 import _fragments as F
    ad = M.make_adata()
    index_of = {k: v for v, k in enumerate(ad.obs.index)}
    for chunk in (None, 3000):
        R = F.read_records(files["bgzf"], index_of, cuda, chunk_bytes=chunk or F.CHUNK_BYTES)
        torch.cuda.synchronize()
        r = O.parse_text(TEXT)
        assert np.array_equal(R.start.cpu().numpy(), r["start"])
        assert np.array_equal(R.end.cpu().numpy(), r["end"])
        assert np.array_equal(R.score.cpu().numpy(), r["score"])
        assert np.array_equal(R.cell.cpu().numpy(), [index_of.get(n, -1) for n in r["name"]])
        spans = {}
        for i, c in enumerate(r["contig"]):
            spans.setdefault(c, [i, i])[1] = i + 1
        assert {k: list(v) for k, v in R.contigs.items()} == spans
        assert R.lmax == int((r["end"] - r["start"]).max())


def test_two_calls_identical_bits(cuda, files):
    import muon_b200 as mu
    outs = []
    for _ in range(2):
        ad = M.make_adata(files["bgzf"])
        X = mu.atac.tl.count_fragments_features(ad, M.features_for("plain"), count_reads=False).X
        T = mu.atac.tl.tss_enrichment(ad, M.tss_features()).X
        mu.atac.tl.nucleosome_signal(ad, n=60000)
        outs.append((X.data.tobytes(), X.indices.tobytes(), T.tobytes(), ad.obs["nucleosome_signal"].values.tobytes()))
    assert outs[0] == outs[1]


def test_malformed_line_raises(cuda, tmp_path):
    import muon_b200 as mu
    bad = TEXT[:5000].rsplit(b"\n", 1)[0] + b"\nchr3\t12\tx\tCELL0001-1\t1\n"
    path = O.write_fragments(str(tmp_path / "m.tsv"), bad, kind="plain")
    with pytest.raises(ValueError):
        mu.atac.tl.nucleosome_signal(M.make_adata(path), n=10_000)


def big_file(tmp, n=10_000_000, n_cells=2_000, seed=2):
    """1e7 fragments on 4 contigs, plain text (the numpy restatement parses it with numpy, not line by line)."""
    rng = np.random.default_rng(seed)
    contigs = ["chr1", "chr2", "chr3", "chrX"]
    L = 50_000_000
    per = rng.multinomial(n, [0.4, 0.3, 0.2, 0.1])
    cols = {"contig": [], "start": [], "end": [], "cell": [], "score": []}
    for ci, k in enumerate(per):
        s = np.sort(rng.integers(0, L, k))
        ln = np.where(rng.random(k) < 0.6, rng.integers(30, 147, k), rng.integers(147, 700, k))
        cols["contig"].append(np.full(k, ci))
        cols["start"].append(s)
        cols["end"].append(s + ln)
        cols["cell"].append(rng.integers(0, n_cells + 100, k))
        cols["score"].append(rng.integers(1, 5, k))
    cols = {k: np.concatenate(v) for k, v in cols.items()}
    names = np.array([f"BC{i:06d}-1" for i in range(n_cells + 100)])
    path = os.path.join(tmp, "big.tsv")
    with open(path, "w") as fh:
        for lo in range(0, n, 1_000_000):
            sl = slice(lo, lo + 1_000_000)
            fh.write("\n".join(np.char.add(np.char.add(np.char.add(np.char.add(
                np.array(contigs)[cols["contig"][sl]], "\t"), cols["start"][sl].astype(str)), "\t"),
                np.char.add(np.char.add(cols["end"][sl].astype(str), "\t"),
                            np.char.add(np.char.add(names[cols["cell"][sl]], "\t"), cols["score"][sl].astype(str)))))
                     + "\n")
    return path, contigs, cols, names, n_cells


def test_large_file_matches_numpy(cuda, tmp_path):
    import pandas as pd

    import muon_b200 as mu
    from muon_b200._containers import SimpleAnnData
    path, contigs, cols, names, n_cells = big_file(str(tmp_path))
    rec = {"contig": np.array(contigs, dtype=object)[cols["contig"]], "start": cols["start"], "end": cols["end"],
           "name": names[cols["cell"]], "score": cols["score"]}
    obs = pd.DataFrame(index=pd.Index(names[:n_cells]))
    index_of = {k: v for v, k in enumerate(obs.index)}
    R = O.Records(rec, index_of)
    ad = SimpleAnnData(np.zeros((n_cells, 1), np.float32), obs=obs)
    ad.uns["files"] = {"fragments": path}
    mu.atac.tl.nucleosome_signal(ad, n=len(cols["start"]))
    assert np.array_equal(ad.obs["nucleosome_signal"].to_numpy(), O.nucleosome_ref(R, len(cols["start"]), n_cells))
    rng = np.random.default_rng(4)
    tss = pd.DataFrame({"Chromosome": np.array(contigs)[rng.integers(0, 4, 300)],
                        "Start": rng.integers(5_000, 49_000_000, 300)})
    tss["End"] = tss["Start"] + 1000
    res = mu.atac.tl.tss_enrichment(ad, tss, n_tss=2000)
    X, score, _ = O.tss_ref(R, list(zip(tss.Chromosome, tss.Start)), n_cells, 1000, 1000)
    assert np.array_equal(ad.obs["tss_score"].to_numpy(), score, equal_nan=True)
    assert np.array_equal(res.X, X, equal_nan=True)
    g = pd.DataFrame({"Chromosome": np.array(contigs)[rng.integers(0, 4, 500)],
                      "Start": rng.integers(5_000, 49_000_000, 500)})
    g["End"] = g["Start"] + rng.integers(1_000, 100_000, 500)
    got = mu.atac.tl.count_fragments_features(ad, g, count_reads=False).X
    want = O.count_ref(R, [(c, s - 2000, e) for c, s, e in zip(g.Chromosome, g.Start, g.End)], n_cells, False)
    assert (got != want).nnz == 0
