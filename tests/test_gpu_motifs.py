"""GPU: ``scan_sequences`` reproduces the reference run recorded in tests/golden/motifs_small.npz exactly (row order,
the caller's sequence objects, ids, positions, bit-equal scores, tf_gene_name), and matches the array restatement on
the full JASPAR set over 1e6 random bases and on one 5e7-base sequence; pvalue=1 keeps every valid window; short,
empty and all-N sequences; a reused scanner; bit-identical repeated calls."""
import warnings

import numpy as np
import pytest

import motif_cases as C
from oracle import motif_ref as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pfm(tmp_path_factory):
    d = tmp_path_factory.mktemp("pfm")
    return C.write_pfms(d), C.write_meta(d)


def check_case(df, case, seqs, ids, joined):
    z = C.Z
    frame = C.SIG["frames"][case]
    assert list(df.columns) == frame["columns"]
    want = [("object" if c == "sequence" else t) for c, t in zip(frame["columns"], frame["dtypes"])]
    assert [str(t) for t in df.dtypes] == want
    si = z[f"{case}|seq"]
    assert len(df) == len(si)
    col = df["sequence"].to_numpy()
    assert all(col[r] is seqs[i] for r, i in enumerate(si))
    assert list(df["motif_id"]) == [ids[i] for i in z[f"{case}|motif"]]
    assert np.array_equal(df["position"].to_numpy(), z[f"{case}|position"])
    assert np.array_equal(df["score"].to_numpy().view(np.int64), z[f"{case}|score"].view(np.int64))
    if joined:
        g = df["tf_gene_name"]
        assert np.array_equal(g.isna().to_numpy(), z[f"{case}|gene_na"])
        assert list(g.fillna("").astype(str)) == list(z[f"{case}|gene"])


@pytest.mark.parametrize("case", list(C.SIG["cases"]))
def test_golden_case(cuda, pfm, case):
    import muon_b200 as mu
    files, meta_file = pfm
    kw = C.SIG["cases"][case]
    bg = kw.get("background", 4)
    seqs = C.sequences()
    mm = mu.atac.tl._parse_motif_matrices(files=files, background=bg)
    ids, mats = mm["motifs"], mm["matrices"]
    if kw.get("subset"):
        pick = C.Z[f"{case}|motif_pick"]
        seqs = [s for s in seqs if len(s) <= 150][:6]
        ids, mats = [ids[i] for i in pick], [mats[i] for i in pick]
    if kw.get("all_n"):
        seqs = ["N" * 40, "nNRY" * 5, ""]
    meta = mu.atac.tl._parse_motif_ids(meta_file)
    run = (lambda: mu.atac.tl.scan_sequences(seqs, motif_scanner=mu.atac.tl._prepare_motif_scanner(
        mats, background=bg, pvalue=kw["pvalue"]), motifs=ids)) if kw.get("scanner") else \
        (lambda: mu.atac.tl.scan_sequences(seqs, matrices=mats, motifs=ids, motif_meta=meta, background=bg,
                                           pvalue=kw["pvalue"]))
    if case in C.SIG["errors"]:
        with pytest.raises(ValueError, match=C.SIG["errors"][case][1]):
            run()
        return
    df = run()
    check_case(df, case, seqs, ids, joined=not kw.get("scanner"))


def restated_frame(seqs, mats, thresholds, device=None):
    """(seq, motif, pos, score) of the array restatement in the reference's row order.  The sequences are scanned as
    one text with an N between them, so no window spans two; with ``device`` the arrays are torch tensors there."""
    import torch
    tabs = O.tables(mats)
    lens = np.array([len(s) for s in seqs], dtype=np.int64)
    start = np.concatenate([[0], np.cumsum(lens + 1)])[:-1]
    codes = O.codes_of("N".join(seqs))
    if device is not None:
        tabs = [torch.from_numpy(t).to(device) for t in tabs]
        codes = torch.from_numpy(codes).to(device)
    rows = [[], [], []]
    for mi, (pos, sc) in enumerate(O.scan_restated(codes, tabs, thresholds)):
        if device is not None:
            pos, sc = pos.cpu().numpy(), sc.cpu().numpy()
        rows[0].append(np.full(len(pos), mi))
        rows[1].append(np.asarray(pos, np.int64))
        rows[2].append(np.asarray(sc, np.float64))
    mot, pos, score = (np.concatenate(r) for r in rows)
    seq = np.searchsorted(start, pos, side="right") - 1
    pos = pos - start[seq]
    order = np.lexsort((pos, mot, seq))
    return seq[order], mot[order], pos[order], score[order]


def jaspar_matrices(bg=4):
    from muon_b200._motifs import background_of, log_odds
    b = background_of(bg)
    return [log_odds(c, b, 0.0001) for c in C.counts_list(C.JASPAR, "names", "lengths", "counts")]


def assert_hits_equal(hits, want):
    seq_i, mot_i, pos, score = hits
    assert len(pos) == len(want[2])
    assert np.array_equal(seq_i, want[0]) and np.array_equal(mot_i, want[1]) and np.array_equal(pos, want[2])
    assert np.array_equal(score.view(np.int64), want[3].view(np.int64))


def test_full_jaspar_on_1e6_bases(cuda):
    from muon_b200._motifs import MotifScanner, scan_hits
    mats = jaspar_matrices()
    sc = MotifScanner(mats, 4, 0.0001)
    g = C.random_genome(1_000_000, seed=5)
    rng = np.random.default_rng(6)
    cuts = np.sort(rng.choice(np.arange(1, len(g)), 1999, replace=False))     # peaks of varied length
    seqs = [g[a:b] for a, b in zip(np.r_[0, cuts], np.r_[cuts, len(g)])]
    hits = scan_hits(seqs, sc)
    assert len(hits[2]) > 10_000
    assert_hits_equal(hits, restated_frame(seqs, mats, sc.thresholds, cuda))
    assert_hits_equal(scan_hits(seqs, sc), hits)                               # two calls, identical bits


def test_one_5e7_sequence(cuda):
    from muon_b200._lib import MOTIF_TILE
    from muon_b200._motifs import MotifScanner, scan_hits
    mats = jaspar_matrices()[::7][:100]
    sc = MotifScanner(mats, 4, 0.001)
    g = C.random_genome(50_000_000, seed=7, n_runs=20_000, lower_runs=20_000)
    hits = scan_hits([g], sc)
    want = restated_frame([g], mats, sc.thresholds, cuda)
    assert_hits_equal(hits, want)
    L = np.array([m.shape[1] for m in mats])[hits[1]]
    assert np.any(hits[2] // MOTIF_TILE != (hits[2] + L - 1) // MOTIF_TILE)  # hits spanning tile boundaries


def test_pvalue_one_keeps_every_valid_window(cuda):
    from muon_b200._motifs import MotifScanner, scan_hits
    mats = jaspar_matrices()[:61]                    # two groups, the second partly filled
    sc = MotifScanner(mats, 4, 1.0)
    assert sc.n_groups > 1
    seqs = [C.random_genome(3000, seed=s, n_runs=5, lower_runs=5) for s in range(4)]
    seqs += ["ACG", "", "N" * 700, "acgtNacgt" * 70]
    hits = scan_hits(seqs, sc)
    want = restated_frame(seqs, mats, sc.thresholds)
    assert_hits_equal(hits, want)
    valid = 0
    for s in seqs:
        bad = np.concatenate([[0], np.cumsum(O.codes_of(s) == 4)])
        for m in mats:
            L = m.shape[1]
            if len(s) >= L:
                valid += int(np.sum(bad[L:] - bad[:-L] == 0))
    assert len(hits[2]) == valid


def test_short_empty_all_n_and_reused_scanner(cuda, pfm):
    import muon_b200 as mu
    files, _ = pfm
    mm = mu.atac.tl._parse_motif_matrices(files=files)
    sc = mu.atac.tl._prepare_motif_scanner(mm["matrices"], pvalue=0.01)
    seqs = C.sequences()
    short = ["", "A", "NNNNNNNNNN", "acgtacg"] + seqs[:20]
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        a = mu.atac.tl.scan_sequences(short, sc, motifs=mm["motifs"])
        b = mu.atac.tl.scan_sequences(short, sc, motifs=mm["motifs"])
    assert a.equals(b) and np.array_equal(a["score"].to_numpy().view(np.int64), b["score"].to_numpy().view(np.int64))
    assert set(a["sequence"].map(short.index)) <= set(range(1, len(short)))
    want = restated_frame(short, mm["matrices"], sc.thresholds)
    assert np.array_equal(a["position"].to_numpy(), want[2])
    assert list(a["motif_id"]) == [mm["motifs"][i] for i in want[1]]


def test_custom_matrices_without_meta_warn_once(cuda, pfm, monkeypatch):
    import importlib.util

    import muon_b200 as mu
    files, _ = pfm
    mm = mu.atac.tl._parse_motif_matrices(files=files)
    real = importlib.util.find_spec
    monkeypatch.setattr(importlib.util, "find_spec", lambda n, *a: None if n == "muon" else real(n, *a))
    with pytest.warns(UserWarning) as rec:
        df = mu.atac.tl.scan_sequences(C.sequences(), matrices=mm["matrices"], motifs=mm["motifs"])
    assert len([r for r in rec if "motif_to_gene" in str(r.message)]) == 1
    assert list(df.columns) == ["sequence", "motif_id", "position", "score"]
    with pytest.raises(TypeError):
        mu.atac.tl.scan_sequences(["ACGT"], motif_scanner=object(), motifs=["x"])


def test_get_sequences_matches_fixture(cuda, tmp_path):
    import pandas as pd

    import muon_b200 as mu
    from muon_b200._containers import SimpleAnnData
    fa = C.write_fasta(tmp_path)
    ad = SimpleAnnData(np.zeros((2, len(C.Z["peaks"])), np.float32),
                       var=pd.DataFrame(index=pd.Index([str(p) for p in C.Z["peaks"]])))
    with pytest.warns(UserWarning):
        seqs = mu.atac.tl.get_sequences(ad, None, fa)
    assert seqs == C.sequences()
