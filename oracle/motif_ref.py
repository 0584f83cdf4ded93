"""TEST INFRASTRUCTURE ONLY -- the motif-scanning oracle.

* A MOODS stand-in (``MOODS.tools``, ``MOODS.parsers``, ``MOODS.scan``) and a pybedtools stand-in (``BedTool``) for
  running the unmodified reference functions of muon/_atac/tools.py:381-566 without either package.  Each behaviour
  below is recalled from MOODS / bedtools, not checked against them (neither is installed where this was written):
    - [recalled] ``flat_bg(n)`` is ``[1/n] * n``.
    - [recalled] ``pfm_to_log_odds(file, bg, ps)`` reads 4 whitespace-separated rows (A, C, G, T), one column per
      position, and returns s[b][j] = ln((c[b][j] + ps bg[b]) / (sum_b c[b][j] + ps)) - ln(bg[b]) (natural log).
    - [recalled] ``threshold_from_p(mat, bg, p)`` is the score whose upper tail under ``bg`` has mass p, from a DP over
      column scores rounded to an integer grid.  The grid and rounding are this project's
      (``muon_b200._motifs.threshold_from_p``, checked against brute-force enumeration in the tests).
    - [recalled] ``Scanner(window).set_motifs(matrices, bg, thresholds)`` then ``scan(seq)`` returns, per motif in
      list order, the hits of the forward strand only, by ascending position: ``.pos`` the 0-based window start,
      ``.score`` the window's score; a hit is ``score >= threshold``; ``a/c/g/t`` score like ``A/C/G/T`` and a window
      holding any other character is not scored.  The score here is the float64 sum over the columns in order from
      0.0 (MOODS may add them in another order, so its scores can differ in the last bits).
    - [recalled] ``BedTool(text, from_string=True).sequence(fi=fasta).seqfn`` is a FASTA file with one ``>`` header
      line and one sequence line per BED interval (``bedtools getfasta``): 0-based half-open, ``track`` / ``browser``
      / ``#`` lines skipped, first three columns used, FASTA case preserved; an interval past the end of its contig or
      on a contig the FASTA lacks is skipped with a warning; start > end is an error.
* ``scan_restated``: the scan restated with array operations (numpy, or torch tensors on any device: every step is
  an elementwise IEEE float64 add or compare, so both give the same bits).
* ``load_reference_motifs()``: the reference's motif and sequence functions, loaded unmodified with these stand-ins.
"""
from __future__ import annotations

import os
import sys
import tempfile
import types
import warnings

import numpy as np

CODE = np.full(256, 4, dtype=np.int64)
for _i, _b in enumerate("ACGT"):
    CODE[ord(_b)] = CODE[ord(_b.lower())] = _i


# ---- MOODS stand-in ------------------------------------------------------------------------------------------------------
def flat_bg(n):
    return [1.0 / n] * n


def pfm_to_log_odds(path, bg, ps):
    with open(path) as fh:
        rows = [line.split() for line in fh if line.strip()]
    if len(rows) != 4 or len({len(r) for r in rows}) != 1 or not rows[0]:
        raise ValueError(f"{path}: not a 4-row count matrix")
    c = np.array(rows, dtype=np.float64)
    bg = np.asarray(bg, dtype=np.float64)
    return np.log((c + ps * bg[:, None]) / (c.sum(0) + ps)) - np.log(bg)[:, None]


def threshold_from_p(mat, bg, p):
    from muon_b200._motifs import threshold_from_p as t
    return t(mat, np.asarray(bg, dtype=np.float64), p)


def codes_of(seq: str):
    return CODE[np.frombuffer(seq.encode("ascii", "replace"), dtype=np.uint8)]


def tables(matrices):
    """Per motif an (L, 5) table: the 4 log-odds of each column, then -inf for any other character."""
    out = []
    for m in matrices:
        m = np.asarray(m, dtype=np.float64)
        t = np.full((m.shape[1], 5), -np.inf)
        t[:, :4] = m.T
        out.append(t)
    return out


def scan_restated(codes, tabs, thresholds):
    """Hits of every motif in one coded sequence: list (per motif) of (positions, scores).  ``codes`` and ``tabs`` are
    numpy arrays, or torch tensors on one device (``codes`` int64)."""
    torch_mode = not isinstance(codes, np.ndarray)
    out = []
    for t, th in zip(tabs, thresholds):
        L = t.shape[0]
        n = len(codes) - L + 1
        if n <= 0:
            out.append((codes[:0], t[:0, 0]))
            continue
        score = 0.0 + t[0][codes[0:n]]
        for j in range(1, L):
            score = score + t[j][codes[j:j + n]]
        hit = score >= th
        pos = hit.nonzero().flatten() if torch_mode else np.flatnonzero(hit)
        out.append((pos, score[pos]))
    return out


class _Hit:
    __slots__ = ("pos", "score")

    def __init__(self, pos, score):
        self.pos, self.score = pos, score


class Scanner:
    def __init__(self, window_size):
        self.window_size = window_size

    def set_motifs(self, matrices, bg, thresholds):
        self._tabs = tables(matrices)
        self._thr = list(thresholds)

    def scan(self, seq):
        return [[_Hit(int(p), float(s)) for p, s in zip(pos, sc)]
                for pos, sc in scan_restated(codes_of(seq), self._tabs, self._thr)]


def moods_module():
    m = types.ModuleType("MOODS")
    m.__path__ = []
    m.tools = types.ModuleType("MOODS.tools")
    m.tools.flat_bg, m.tools.threshold_from_p = flat_bg, threshold_from_p
    m.parsers = types.ModuleType("MOODS.parsers")
    m.parsers.pfm_to_log_odds = pfm_to_log_odds
    m.scan = types.ModuleType("MOODS.scan")
    m.scan.Scanner = Scanner
    return m


# ---- pybedtools stand-in -------------------------------------------------------------------------------------------------
def read_fasta(path):
    """{name: sequence} of a plain FASTA file, read whole."""
    seqs, name, parts = {}, None, []
    with open(path, "rb") as fh:
        text = fh.read().decode()
    for line in text.splitlines():
        if line.startswith(">"):
            if name is not None:
                seqs[name] = "".join(parts)
            name, parts = line[1:].split()[0], []
        else:
            parts.append(line.strip())
    if name is not None:
        seqs[name] = "".join(parts)
    return seqs


class BedTool:
    def __init__(self, text, from_string=False):
        assert from_string
        self.text = text

    def sequence(self, fi):
        genome = read_fasta(fi)
        fd, path = tempfile.mkstemp(suffix=".fa")
        with os.fdopen(fd, "w") as out:
            for line in self.text.splitlines():
                if not line.strip() or line.startswith(("track", "browser", "#")):
                    continue
                chrom, start, end = line.split("\t")[:3]
                start, end = int(start), int(end)
                if start > end:
                    raise ValueError(f"start > end: {line}")
                if chrom not in genome or end > len(genome[chrom]):
                    warnings.warn(f"skipping {chrom}:{start}-{end}", UserWarning)
                    continue
                out.write(f">{chrom}:{start}-{end}\n{genome[chrom][start:end]}\n")
        res = types.SimpleNamespace(seqfn=path)
        return res


def pybedtools_module():
    m = types.ModuleType("pybedtools")
    m.BedTool = BedTool
    return m


# ---- the reference functions ---------------------------------------------------------------------------------------------
def load_reference_motifs():
    """``_parse_motif_ids``, ``_parse_motif_matrices``, ``_prepare_motif_scanner``, ``scan_sequences``,
    ``get_sequences``, ``locate_file`` and ``locate_genome`` of the unmodified muon/_atac/tools.py, with the stand-ins
    above as ``MOODS`` and ``pybedtools``."""
    from . import _refload as RL
    if not RL.reference_available():
        raise FileNotFoundError(RL.REF_ROOT)
    RL._install_stubs()
    from muon_b200._containers import SimpleMuData
    moods = moods_module()
    for name, mod in (("MOODS", moods), ("MOODS.tools", moods.tools), ("MOODS.parsers", moods.parsers),
                      ("MOODS.scan", moods.scan), ("pybedtools", pybedtools_module())):
        sys.modules[name] = mod
    for name in ("_refmotif", "_refmotif._atac", "_refmotif._rna"):
        if name not in sys.modules:
            p = types.ModuleType(name)
            p.__path__ = []
            sys.modules[name] = p
    sys.modules["_refmotif"].MuData = SimpleMuData
    au = types.ModuleType("_refmotif._atac.utils")
    sys.modules["_refmotif._atac.utils"] = au
    sys.modules["_refmotif._atac"].utils = au
    ru = types.ModuleType("_refmotif._rna.utils")
    ru.get_gene_annotation_from_rna = lambda *a, **k: None
    sys.modules["_refmotif._rna.utils"] = ru
    tools = sys.modules.get("_refmotif._atac.tools") or RL._load("muon/_atac/tools.py", "_refmotif._atac.tools")
    names = ("_parse_motif_ids", "_parse_motif_matrices", "_prepare_motif_scanner", "scan_sequences", "get_sequences",
             "locate_file", "locate_genome")
    return types.SimpleNamespace(**{n: getattr(tools, n) for n in names}, module=tools)
