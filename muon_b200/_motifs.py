"""Motif scanning and sequence extraction (muon/_atac/tools.py:381-618) for ``mu.atac.tl``.

Host side: the JASPAR ``.pfm`` parser, MOODS' log-odds and p-value thresholds (restated: MOODS is not a dependency),
a FASTA / ``.fai`` reader standing in for ``bedtools getfasta``, and the DataFrame assembly.  Device side
(``csrc/motifs.cu``): every window of every sequence is scored against every motif in float64, and the hits are
compacted in the reference's row order (sequence, motif, position) from per-(sequence, motif, tile) counts.

The MOODS and bedtools behaviours restated here are recalled, not checked against those tools; DESIGN.md §8 lists
them.
"""
from __future__ import annotations

import importlib.util
import os
import warnings
from collections.abc import Iterable
from glob import glob

import numpy as np

from ._lib import MOTIF_CODES, MOTIF_GROUP_COLS, MOTIF_MAX_LEN, MOTIF_TILE

# Grid of the threshold DP, in nats.  A power of two, so every grid score is exact in float64 (see threshold_from_p).
THRESHOLD_GRID = 2.0 ** -10
MAX_MOTIFS = (1 << 31) - 1            # motif ids are int32 on the device


# ---- the bundled JASPAR database -------------------------------------------------------------------------------------
def jaspar_dir():
    """``<muon>/_atac/_ref/jaspar`` of an importable ``muon`` package, or None.  The database is muon's package data
    and is looked up at run time, never copied."""
    spec = importlib.util.find_spec("muon")
    if spec is None or not spec.submodule_search_locations:
        return None
    for root in spec.submodule_search_locations:
        d = os.path.join(root, "_atac", "_ref", "jaspar")
        if os.path.isdir(d):
            return d
    return None


def _require_jaspar(what):
    d = jaspar_dir()
    if d is None:
        raise FileNotFoundError(f"The bundled JASPAR database is muon's package data and no `muon` package is "
                                f"importable: {what}")
    return d


# ---- MOODS' arithmetic ---------------------------------------------------------------------------------------------------
def flat_bg(n):
    """MOODS.tools.flat_bg: a uniform background over ``n`` letters."""
    return [1.0 / n] * n


def background_of(background):
    """The reference's ``flat_bg(background)`` for a number, the iterable as given otherwise; 4 entries summing to 1."""
    bg = flat_bg(background) if not isinstance(background, Iterable) else list(background)
    bg = np.asarray(bg, dtype=np.float64)
    if bg.shape != (4,) or not np.all(bg > 0) or abs(bg.sum() - 1.0) > 1e-9:
        raise ValueError(f"background must be 4 positive frequencies summing to 1 (A, C, G, T), got {bg.tolist()}")
    return bg


def read_pfm(path):
    """A count matrix: 4 whitespace-separated rows (A, C, G, T), one column per position, as float64 (4, L)."""
    with open(path) as fh:
        rows = [line.split() for line in fh if line.strip()]
    try:
        m = np.array([[float(v) for v in r] for r in rows], dtype=np.float64) if rows else None
    except ValueError:
        raise ValueError(f"{path}: not a count matrix (non-numeric entry)") from None
    if m is None or m.ndim != 2 or m.shape[0] != 4 or m.shape[1] == 0:
        raise ValueError(f"{path}: a .pfm file needs 4 rows (A, C, G, T) of equal, non-zero length")
    return m


def log_odds(counts, bg, pseudocount):
    """MOODS.tools/parsers ``pfm_to_log_odds``: s[b, j] = ln((c[b, j] + ps bg[b]) / (sum_b c[b, j] + ps)) - ln bg[b]."""
    c = np.asarray(counts, dtype=np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        s = np.log((c + pseudocount * bg[:, None]) / (c.sum(0) + pseudocount)) - np.log(bg)[:, None]
    if not np.all(np.isfinite(s)):
        raise ValueError("log-odds are not finite: a zero count needs a positive pseudocount")
    return s


def _matrix(mat):
    m = np.asarray(mat, dtype=np.float64)
    if m.ndim != 2 or m.shape[0] != 4 or m.shape[1] == 0:
        raise ValueError(f"a log-odds matrix has 4 rows (A, C, G, T) and at least one column, got shape {m.shape}")
    if not np.all(np.isfinite(m)):
        raise ValueError("a log-odds matrix must be finite")
    return m


def threshold_from_p(mat, bg, p):
    """The score threshold at which the upper tail of the motif's score under ``bg`` has mass ``p``.

    MOODS computes this from a DP over column scores rounded to an integer grid; so does this restatement, with
    q[b, j] = floor(s[b, j] / d) for d = THRESHOLD_GRID.  Q = sum_j q[b_j, j] has the exact distribution below, and
    the threshold is t = k d for the smallest k with P(Q >= k) <= p.  Since Q d <= S < Q d + L d for a window's real
    score S, P(S >= t + L d) <= p and P(S >= t - d) > p: only windows scoring in [t - d, t + L d] can fall on the
    other side of an exact-tail threshold.  d is a power of two, so t and every grid sum are exact and a window with
    Q >= k also has a float64 column-order score >= t; with p = 1 every window is a hit."""
    m = _matrix(mat)
    if not (0.0 < p <= 1.0):
        raise ValueError(f"pvalue must be in (0, 1], got {p}")
    q = np.floor(m / THRESHOLD_GRID)
    q -= q * THRESHOLD_GRID > m                                   # never above the real score
    q = q.astype(np.int64)
    lo = int(q.min(0).sum())
    hi = int(q.max(0).sum())
    dist = np.zeros(hi - lo + 1, dtype=np.float64)
    dist[0] = 1.0
    span = 0                                                      # dist[0 .. span] may be non-zero
    qmin = q.min(0)
    for j in range(m.shape[1]):
        rel = q[:, j] - qmin[j]
        w = int(rel.max())
        new = np.zeros(span + w + 1, dtype=np.float64)
        for b in range(4):
            new[rel[b]:rel[b] + span + 1] += bg[b] * dist[:span + 1]
        span += w
        dist[:span + 1] = new
    tail = np.cumsum(dist[::-1])[::-1]                            # tail[i] = P(Q >= lo + i)
    k = np.flatnonzero(tail <= p) if p < 1.0 else [0]
    if len(k) == 0:                      # the best word alone has mass > p (short motifs): only it is a hit
        best = 0.0
        for j in range(m.shape[1]):
            best += m[:, j].max()
        return float(best)
    return float((lo + int(k[0])) * THRESHOLD_GRID)


# ---- the reference's helpers ---------------------------------------------------------------------------------------------
def parse_motif_ids(filename=None):
    import pandas as pd
    if filename is None:
        filename = os.path.join(_require_jaspar("pass `filename=` (a tab-separated motif_id / tf_gene_name table)"),
                                "motif_to_gene.txt")
    motifs = pd.read_csv(filename, sep="\t", header=None)
    motifs.columns = ["motif_id", "tf_gene_name"]
    return motifs.set_index("motif_id")


def parse_motif_matrices(files=None, background=4, pseudocount=0.0001):
    if files is None:
        files = glob(os.path.join(_require_jaspar("pass `files=` (a list of .pfm files) to _parse_motif_matrices"),
                                  "*.pfm"))
    bg = background_of(background)
    matrices = [log_odds(read_pfm(f), bg, pseudocount) for f in files]
    return {"motifs": [os.path.basename(f).rstrip(".pfm") for f in files], "matrices": matrices}


class MotifScanner:
    """Log-odds tables, thresholds and the scan groups of a list of motifs, resident on one CUDA device.  Built by
    ``_prepare_motif_scanner``; ``scan_sequences(..., motif_scanner=s, motifs=ids)`` reuses it without uploading."""

    def __init__(self, matrices, background=4, pvalue=0.0001):
        mats = [_matrix(m) for m in matrices]
        bg = background_of(background)
        if not (0.0 < pvalue <= 1.0):
            raise ValueError(f"pvalue must be in (0, 1], got {pvalue}")
        if len(mats) > MAX_MOTIFS:
            raise NotImplementedError(f"{len(mats)} motifs: at most {MAX_MOTIFS} (int32 motif ids)")
        lengths = np.array([m.shape[1] for m in mats], dtype=np.int64)
        if len(mats) and lengths.max() > MOTIF_MAX_LEN:
            raise NotImplementedError(f"motifs longer than {MOTIF_MAX_LEN} columns are not supported "
                                      f"(got {int(lengths.max())})")
        if lengths.sum() > (1 << 31) - 1:
            raise NotImplementedError("more than 2^31 - 1 matrix columns in total")
        self.background = bg
        self.lengths = lengths
        self.thresholds = np.array([threshold_from_p(m, bg, pvalue) for m in mats], dtype=np.float64)
        col_off = np.zeros(len(mats) + 1, dtype=np.int64)
        np.cumsum(lengths, out=col_off[1:])
        tab = np.full((int(col_off[-1]), MOTIF_CODES), -np.inf, dtype=np.float64)
        if len(mats):
            tab[:, :4] = np.concatenate(mats, axis=1).T
        # groups of consecutive motifs whose columns fit the kernel's shared-memory table
        group_m0 = [0]
        for i in range(len(mats)):
            if col_off[i + 1] - col_off[group_m0[-1]] > MOTIF_GROUP_COLS:
                group_m0.append(i)
        group_m0.append(len(mats))
        if len(mats) == 0:
            group_m0 = [0]
        self.n_motifs = len(mats)
        self.n_groups = len(group_m0) - 1
        self._host = {"tab": tab.reshape(-1), "col_off": col_off.astype(np.int32), "thr": self.thresholds,
                      "group_m0": np.asarray(group_m0, dtype=np.int32)}
        self._dev = None
        self.device = None

    def upload(self, device):
        import torch
        if self._dev is None or self.device != device:
            self._dev = {k: torch.from_numpy(np.ascontiguousarray(v)).to(device) for k, v in self._host.items()}
            self.device = device
        return self._dev


def prepare_motif_scanner(matrices=None, background=4, pvalue=0.0001, max_hits=10):
    if matrices is None:
        matrices = parse_motif_matrices(files=None, background=background)["matrices"]
    s = MotifScanner(matrices, background, pvalue)
    s.upload(_cuda())
    return s


def _cuda():
    import torch
    if not torch.cuda.is_available():
        from ._lib import MuonB200Error
        raise MuonB200Error("scan_sequences runs on a CUDA device and none is available")
    return torch.device("cuda", torch.cuda.current_device())


# ---- the scan ------------------------------------------------------------------------------------------------------------
def _sequence_bytes(seqs):
    """The concatenated sequences as bytes (one byte per character: anything outside ASCII becomes ``?``, which
    scores like N) and their int64 offsets."""
    for s in seqs:
        if not isinstance(s, str):
            raise TypeError(f"sequences must be str, got {type(s).__name__}")
    lengths = np.fromiter(map(len, seqs), dtype=np.int64, count=len(seqs))
    if len(seqs) and lengths.max() > (1 << 31) - 1:
        raise NotImplementedError("sequences longer than 2^31 - 1 bases are not supported")
    off = np.zeros(len(seqs) + 1, dtype=np.int64)
    np.cumsum(lengths, out=off[1:])
    return "".join(seqs).encode("ascii", "replace"), off


def scan_hits(seqs, scanner, timings=None):
    """Every hit of ``scanner`` in ``seqs`` as host arrays (seq int32, motif int32, pos int32, score float64), in
    (sequence, motif, position) order.  ``timings`` (a dict) receives upload / kernels / download seconds."""
    import time

    import torch

    from ._lib import call, ptr, stream_ptr
    text, off = _sequence_bytes(seqs)
    if len(seqs) >= (1 << 31) - 1:
        raise NotImplementedError("more than 2^31 - 2 sequences")
    tiles = (np.diff(off) + MOTIF_TILE - 1) // MOTIF_TILE
    tile0 = np.zeros(len(seqs) + 1, dtype=np.int64)
    np.cumsum(tiles, out=tile0[1:])
    n_tiles = int(tile0[-1])
    M = scanner.n_motifs
    if n_tiles > (1 << 31) - 1 or n_tiles * M > (1 << 62):
        raise NotImplementedError(f"{n_tiles} tiles of {MOTIF_TILE} bases: too many for one scan")
    empty = (np.zeros(0, np.int32), np.zeros(0, np.int32), np.zeros(0, np.int32), np.zeros(0, np.float64))
    if n_tiles == 0 or M == 0:
        return empty
    device = _cuda()
    torch.cuda.synchronize(device)
    t0 = time.perf_counter()
    tabs = scanner.upload(device)
    pinned = torch.empty(max(len(text), 1), dtype=torch.uint8, pin_memory=True)
    pinned.numpy()[:len(text)] = np.frombuffer(text, dtype=np.uint8)
    codes = pinned[:len(text)].to(device, non_blocking=True)
    seq_off = torch.from_numpy(off).to(device)
    seq_tile0 = torch.from_numpy(tile0).to(device)
    tile_seq = torch.from_numpy(np.repeat(np.arange(len(seqs), dtype=np.int32), tiles)).to(device)
    torch.cuda.synchronize(device)
    t1 = time.perf_counter()
    st = stream_ptr()
    geo = (ptr(codes), ptr(seq_off), ptr(tile_seq), ptr(seq_tile0), n_tiles, ptr(tabs["tab"]), ptr(tabs["col_off"]),
           ptr(tabs["thr"]), ptr(tabs["group_m0"]), scanner.n_groups, M)
    call("mub_motif_encode", ptr(codes), len(text), st)
    counts = torch.empty(n_tiles * M, dtype=torch.int32, device=device)
    call("mub_motif_count", *geo, ptr(counts), st)
    incl = torch.cumsum(counts, 0, dtype=torch.int64)
    n_hits = int(incl[-1])
    free, _ = torch.cuda.mem_get_info(device)
    need = n_hits * (3 * 4 + 8)
    if need > free:
        raise NotImplementedError(f"{n_hits} hits need {need / 2**30:.1f} GiB of device memory and "
                                  f"{free / 2**30:.1f} GiB are free: scan fewer sequences at a time")
    out_seq = torch.empty(n_hits, dtype=torch.int32, device=device)
    out_motif = torch.empty(n_hits, dtype=torch.int32, device=device)
    out_pos = torch.empty(n_hits, dtype=torch.int32, device=device)
    out_score = torch.empty(n_hits, dtype=torch.float64, device=device)
    if n_hits:
        incl -= counts
        call("mub_motif_fill", *geo, ptr(counts), ptr(incl), ptr(out_seq), ptr(out_motif), ptr(out_pos),
             ptr(out_score), st)
    del counts, incl, codes
    torch.cuda.synchronize(device)
    t2 = time.perf_counter()
    res = tuple(t.cpu().numpy() for t in (out_seq, out_motif, out_pos, out_score))
    t3 = time.perf_counter()
    if timings is not None:
        timings.update(upload=t1 - t0, kernels=t2 - t1, download=t3 - t2)
    return res


def hits_frame(seqs, motifs, hits):
    """The reference's ``matches`` frame: sequence (the caller's own str objects), motif_id, position, score."""
    import pandas as pd
    seq_i, mot_i, pos, score = hits
    if len(pos) == 0:
        matches = pd.DataFrame([])
        matches.columns = ["sequence", "motif_id", "position", "score"]     # raises, as the reference does
    seq_col = np.empty(len(seqs), dtype=object)
    seq_col[:] = seqs
    mot_col = np.empty(len(motifs), dtype=object)
    mot_col[:] = list(motifs)
    return pd.DataFrame({"sequence": pd.Series(seq_col.take(seq_i), dtype=object, copy=False),
                         "motif_id": mot_col.take(mot_i), "position": pos.astype(np.int64), "score": score})


def scan_sequences(sequences, motif_scanner=None, matrices=None, motifs=None, motif_meta=None, background=4,
                   pvalue=0.0001, max_hits=10, timings=None):
    if motifs is None:
        assert matrices is None, ("Both a list of matrices and a corresponding list of motif IDs should be provided "
                                  "— or none to use the built-in ones, unless a scanner is provided.")
    if motif_scanner is None:
        if matrices is None:
            motifs = parse_motif_matrices(files=None, background=background)["motifs"]
        else:
            assert motifs is not None, "A list of motif IDs should be provided if building a scanner from matrices"
        seqs = list(sequences)
        _sequence_bytes(seqs)                                     # refuse bad sequences before any device work
        motif_scanner = MotifScanner(
            parse_motif_matrices(files=None, background=background)["matrices"] if matrices is None else matrices,
            background, pvalue)
        if motif_meta is None:
            if matrices is None or jaspar_dir() is not None:
                motif_meta = parse_motif_ids()
            else:
                warnings.warn("scan_sequences: no `muon` package is importable, so the JASPAR motif_to_gene table is "
                              "absent; pass `motif_meta=` to add tf_gene_name", UserWarning, stacklevel=3)
    else:
        if not isinstance(motif_scanner, MotifScanner):
            raise TypeError(f"motif_scanner must be a MotifScanner from muon_b200's _prepare_motif_scanner (it runs "
                            f"on the GPU; there is no CPU scanner), got {type(motif_scanner).__name__}")
        assert motifs is not None, ("A list of motif IDs should be provided that corresponds to the matrices that the "
                                    "motif scanner was built on.")
        seqs = list(sequences)
    if len(motifs) < motif_scanner.n_motifs:
        raise IndexError(f"{len(motifs)} motif ids for a scanner of {motif_scanner.n_motifs} motifs")
    import time
    hits = scan_hits(seqs, motif_scanner, timings)
    t0 = time.perf_counter()
    matches = hits_frame(seqs, motifs, hits)
    t1 = time.perf_counter()
    if motif_meta is not None:
        matches = matches.set_index("motif_id").join(motif_meta, how="left").reset_index()
    if timings is not None:
        timings.update(frame=t1 - t0, join=time.perf_counter() - t1)
    return matches


# ---- bedtools getfasta ---------------------------------------------------------------------------------------------------
class Fasta:
    """Random access to an uncompressed FASTA file through its ``.fai`` (name, length, offset, line bases, line
    width) or, without one, through an index built in memory (no ``.fai`` is written)."""

    def __init__(self, path):
        with open(path, "rb") as fh:
            head = fh.read(2)
        if head == b"\x1f\x8b":
            raise NotImplementedError(f"{path} is compressed: decompress it (e.g. `gunzip -k`) before get_sequences")
        self.path = path
        size = os.path.getsize(path)
        self.mm = np.memmap(path, dtype=np.uint8, mode="r") if size else np.zeros(0, np.uint8)
        fai = path + ".fai"
        self.index = self._read_fai(fai) if os.path.isfile(fai) else self._build_index()

    @staticmethod
    def _read_fai(fai):
        index = {}
        with open(fai) as fh:
            for line in fh:
                f = line.rstrip("\n").split("\t")
                if len(f) < 5:
                    raise ValueError(f"{fai}: malformed line {line!r}")
                index[f[0]] = tuple(int(v) for v in f[1:5])
        return index

    def _build_index(self):
        mm = self.mm
        nl = np.flatnonzero(mm == 10)
        starts = np.concatenate([[0], nl + 1])
        ends = np.concatenate([nl, [len(mm)]])
        keep = starts < len(mm)
        starts, ends = starts[keep], ends[keep]
        index = {}
        heads = np.flatnonzero(mm[starts] == ord(">")) if len(starts) else np.zeros(0, np.int64)
        for h, a in enumerate(heads):
            b = heads[h + 1] if h + 1 < len(heads) else len(starts)
            name = bytes(mm[starts[a] + 1:ends[a]]).decode().split()[0] if ends[a] > starts[a] + 1 else ""
            ls, le = starts[a + 1:b], ends[a + 1:b]
            cr = (le > ls) & (mm[np.maximum(le - 1, 0)] == 13) if len(ls) else np.zeros(0, bool)
            bases = le - ls - cr
            while len(bases) and bases[-1] == 0:                  # blank lines closing the record
                bases, ls, cr = bases[:-1], ls[:-1], cr[:-1]
            offset = int(ls[0]) if len(ls) else int(ends[a] + 1)
            if len(bases) == 0:
                index[name] = (0, offset, 0, 0)
                continue
            lb, lw = int(bases[0]), int(bases[0] + 1 + cr[0])
            if np.any(bases[:-1] != lb) or bases[-1] > lb or np.any(np.diff(ls) != lw):
                raise ValueError(f"{self.path}: different line length in sequence '{name}'")
            index[name] = (int(bases.sum()), offset, lb, lw)
        return index

    def fetch(self, name, start, end):
        length, offset, lb, lw = self.index[name]
        if end <= start:
            return ""

        def at(p):
            return offset + (p // lb) * lw + p % lb
        raw = bytes(self.mm[at(start):at(end - 1) + 1])
        return raw.replace(b"\n", b"").replace(b"\r", b"").decode("ascii", "replace")


def parse_bed(text):
    """(chrom, start, end) of every interval of a BED text; ``track``, ``browser`` and ``#`` lines are skipped."""
    out = []
    for line in text.splitlines():
        if not line.strip() or line.startswith(("track", "browser", "#")):
            continue
        f = line.split("\t") if "\t" in line else line.split()
        if len(f) < 3:
            raise ValueError(f"BED line with fewer than 3 columns: {line!r}")
        try:
            start, end = int(f[1]), int(f[2])
        except ValueError:
            raise ValueError(f"BED line with non-integer coordinates: {line!r}") from None
        if start > end:
            raise ValueError(f"BED interval with start > end: {line!r}")
        if start < 0:
            raise ValueError(f"BED interval with a negative start: {line!r}")
        out.append((f[0], start, end))
    return out


def get_fasta(bed_text, fasta_file):
    """``bedtools getfasta -fi fasta_file`` over the BED text: one sequence per interval, case preserved; an interval
    on a contig missing from the FASTA or past the end of its contig is skipped with a warning."""
    fa = Fasta(fasta_file)
    seqs = []
    for chrom, start, end in parse_bed(bed_text):
        if chrom not in fa.index:
            warnings.warn(f"chromosome {chrom!r} was not found in the FASTA file; skipping {chrom}:{start}-{end}",
                          UserWarning, stacklevel=3)
            continue
        if end > fa.index[chrom][0]:
            warnings.warn(f"{chrom}:{start}-{end} is beyond the length of {chrom} ({fa.index[chrom][0]}); skipping",
                          UserWarning, stacklevel=3)
            continue
        seqs.append(fa.fetch(chrom, start, end))
    return seqs
