"""TEST INFRASTRUCTURE ONLY -- the fragments-file oracle.

* A pysam stand-in (``TabixFile``, ``asBed``) for running the unmodified reference functions of
  muon/_atac/tools.py:640-1201 without pysam.  Each behaviour below is recalled from pysam / htslib, not checked
  against them (pysam is not installed where this was written); each is marked [recalled]:
    - [recalled] ``fetch(contig, start, stop)`` yields the records with ``record.start < stop`` and
      ``record.end > start`` (0-based, half-open BED), in file order.
    - [recalled] it accepts integral floats as bounds (the reference passes ``start - 2e3``).
    - [recalled] it raises ValueError for ``start < 0`` ("start out of range"), for ``start > stop`` and for a contig
      that is not in the file.
    - [recalled] ``fetch()`` with no region walks every record in file order and skips ``#`` header lines.
    - [recalled] ``contigs`` lists the contigs of the file, in file order.
    - [recalled] ``asBed()`` records carry ``contig, start, end, name, score``.
* A BGZF writer and a tabix (``.tbi``) writer for the fixtures.  The ``.tbi`` layout is [recalled] from the htslib
  format description: magic ``TBI\\1``, n_ref, format, col_seq/beg/end, meta, skip, names; per reference the binning
  index (bin, chunks) and the linear index of 16 kb windows holding the smallest virtual offset of a record that
  overlaps the window (empty windows take the previous window's offset); the whole file BGZF-compressed.
* A vectorised numpy restatement of ``count_fragments_features``, ``_tss_pileup`` / ``_calculate_tss_score`` and
  ``nucleosome_signal`` for inputs too large for the reference's per-fragment loops.
* ``load_reference_fragments()``: the four reference functions, loaded unmodified with this stand-in as ``pysam``.
"""
from __future__ import annotations

import bisect
import gzip
import os
import struct
import sys
import types
import zlib

import numpy as np

BGZF_BLOCK = 0xFF00
BGZF_EOF = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")
TBX_UCSC = 0x10000
LIDX_SHIFT = 14


# ---- reading the text -------------------------------------------------------------------------------------------------
def read_text(path) -> bytes:
    with open(path, "rb") as fh:
        head = fh.read(2)
    if head == b"\x1f\x8b":
        with gzip.open(path, "rb") as fh:
            return fh.read()
    with open(path, "rb") as fh:
        return fh.read()


def parse_text(text: bytes):
    """Records of a fragments text: dict of numpy columns (contig names, start, end, name, score) in file order."""
    contigs, start, end, name, score = [], [], [], [], []
    for line in text.split(b"\n"):
        if not line or line.startswith(b"#"):
            continue
        f = line.split(b"\t")
        contigs.append(f[0].decode())
        start.append(int(f[1]))
        end.append(int(f[2]))
        name.append(f[3].decode())
        score.append(int(f[4]))
    return {"contig": np.array(contigs, dtype=object), "start": np.array(start, dtype=np.int64),
            "end": np.array(end, dtype=np.int64), "name": np.array(name, dtype=object),
            "score": np.array(score, dtype=np.int64)}


def format_text(contig, start, end, name, score, header=()) -> bytes:
    lines = [h for h in header]
    lines += [f"{c}\t{s}\t{e}\t{n}\t{v}" for c, s, e, n, v in zip(contig, start, end, name, score)]
    return ("\n".join(lines) + "\n").encode()


# ---- pysam stand-in -------------------------------------------------------------------------------------------------
class BedRecord:
    __slots__ = ("contig", "start", "end", "name", "score")

    def __init__(self, contig, start, end, name, score):
        self.contig, self.start, self.end, self.name, self.score = contig, start, end, name, score


class asBed:  # noqa: N801 -- pysam's name
    pass


def _coord(v, what):
    if isinstance(v, float):
        if not v.is_integer():
            raise TypeError(f"{what} must be integral, got {v}")
        v = int(v)
    return int(v)


class TabixFile:
    def __init__(self, path, parser=None):
        self.path = os.fspath(path)
        r = parse_text(read_text(self.path))
        self._rec = r
        self._order = []
        self._by = {}
        for i, c in enumerate(r["contig"]):
            if c not in self._by:
                self._order.append(c)
                self._by[c] = [i, i + 1]
            else:
                self._by[c][1] = i + 1
        self._lmax = int((r["end"] - r["start"]).max()) if len(r["start"]) else 0

    @property
    def contigs(self):
        return list(self._order)

    def _make(self, i):
        r = self._rec
        return BedRecord(r["contig"][i], int(r["start"][i]), int(r["end"][i]), r["name"][i], int(r["score"][i]))

    def fetch(self, contig=None, start=None, stop=None):
        if contig is None and start is None and stop is None:
            return (self._make(i) for i in range(len(self._rec["start"])))
        a = 0 if start is None else _coord(start, "start")
        b = (1 << 31) - 1 if stop is None else _coord(stop, "stop")
        if a > b:
            raise ValueError(f"invalid coordinates: start ({a}) > stop ({b})")
        if a < 0:
            raise ValueError(f"start out of range ({a})")
        if contig not in self._by:
            raise ValueError(f"could not create iterator for region '{contig}:{a + 1}-{b}'")
        lo, hi = self._by[contig]
        st = self._rec["start"]
        j = lo + bisect.bisect_left(st[lo:hi], a - self._lmax + 1) if self._lmax else lo
        out = []
        while j < hi and st[j] < b:
            if self._rec["end"][j] > a:
                out.append(self._make(j))
            j += 1
        return iter(out)

    def close(self):
        pass


def pysam_module():
    m = types.ModuleType("pysam")
    m.TabixFile, m.asBed = TabixFile, asBed
    m.__stub__ = True
    return m


# ---- BGZF and .tbi writers -------------------------------------------------------------------------------------------
def bgzf_block(data: bytes) -> bytes:
    c = zlib.compressobj(6, zlib.DEFLATED, -15)
    payload = c.compress(data) + c.flush()
    bsize = 18 + len(payload) + 8
    head = struct.pack("<BBBBIBBHBBHH", 0x1F, 0x8B, 8, 4, 0, 0, 0xFF, 6, ord("B"), ord("C"), 2, bsize - 1)
    return head + payload + struct.pack("<II", zlib.crc32(data) & 0xFFFFFFFF, len(data))


def write_bgzf(path, text: bytes, block_size=BGZF_BLOCK):
    """BGZF-compress ``text`` in blocks of ``block_size`` bytes (cut anywhere, as bgzip does).  Returns the compressed
    offset of each block and the text offset it starts at."""
    coff, uoff = [], []
    with open(path, "wb") as fh:
        pos = 0
        for k in range(0, len(text), block_size):
            coff.append(pos)
            uoff.append(k)
            blk = bgzf_block(text[k:k + block_size])
            fh.write(blk)
            pos += len(blk)
        fh.write(BGZF_EOF)
    return np.array(coff, dtype=np.int64), np.array(uoff, dtype=np.int64)


def write_plain_gzip(path, text: bytes):
    with gzip.open(path, "wb") as fh:
        fh.write(text)


def reg2bin(beg, end):
    end -= 1
    for shift, off in ((14, 4681), (17, 585), (20, 73), (23, 9), (26, 1)):
        if beg >> shift == end >> shift:
            return off + (beg >> shift)
    return 0


def tbi_index(text: bytes, coff, uoff):
    """The tabix index of a BGZF file of ``text``: names and, per contig, the bins and the linear index."""
    starts = np.concatenate([[0], np.flatnonzero(np.frombuffer(text, np.uint8) == 10)[:-1] + 1])
    names, refs = [], {}
    for ls in starts:
        le = text.index(b"\n", ls)
        line = text[ls:le]
        if not line or line.startswith(b"#"):
            continue
        f = line.split(b"\t")
        c, beg, end = f[0].decode(), int(f[1]), int(f[2])
        end = max(end, beg + 1)
        blk = int(np.searchsorted(uoff, ls, side="right") - 1)
        voff = (int(coff[blk]) << 16) | int(ls - uoff[blk])
        le_blk = int(np.searchsorted(uoff, le + 1, side="right") - 1)
        vend = (int(coff[le_blk]) << 16) | int(le + 1 - uoff[le_blk])
        if c not in refs:
            names.append(c)
            refs[c] = {"bins": {}, "lin": {}}
        r = refs[c]
        b = reg2bin(beg, end)
        chunks = r["bins"].setdefault(b, [])
        if chunks and chunks[-1][1] == voff:
            chunks[-1][1] = vend
        else:
            chunks.append([voff, vend])
        for w in range(beg >> LIDX_SHIFT, ((end - 1) >> LIDX_SHIFT) + 1):
            r["lin"].setdefault(w, voff)
    out = []
    for c in names:
        lin = refs[c]["lin"]
        n = max(lin) + 1
        ioff = np.zeros(n, dtype=np.uint64)
        prev = 0
        for w in range(n):
            prev = lin.get(w, prev)
            ioff[w] = prev
        out.append((c, refs[c]["bins"], ioff))
    return out


def write_tbi(path, text: bytes, coff, uoff):
    idx = tbi_index(text, coff, uoff)
    nm = b"".join(c.encode() + b"\0" for c, _, _ in idx)
    body = [b"TBI\x01", struct.pack("<iiiiiiii", len(idx), TBX_UCSC, 1, 2, 3, ord("#"), 0, len(nm)), nm]
    for _, bins, ioff in idx:
        body.append(struct.pack("<i", len(bins)))
        for b in sorted(bins):
            body.append(struct.pack("<Ii", b, len(bins[b])))
            for a, e in bins[b]:
                body.append(struct.pack("<QQ", a, e))
        body.append(struct.pack("<i", len(ioff)))
        body.append(ioff.astype("<u8").tobytes())
    raw = b"".join(body)
    with open(path, "wb") as fh:
        for k in range(0, len(raw), BGZF_BLOCK):
            fh.write(bgzf_block(raw[k:k + BGZF_BLOCK]))
        fh.write(BGZF_EOF)
    return idx


def write_fragments(path, text: bytes, kind="bgzf", block_size=BGZF_BLOCK, index=True):
    """Write ``text`` as ``kind`` in ("bgzf", "gzip", "plain"); a ``.tbi`` next to a BGZF file when ``index``."""
    if kind == "bgzf":
        coff, uoff = write_bgzf(path, text, block_size)
        if index:
            write_tbi(str(path) + ".tbi", text, coff, uoff)
    elif kind == "gzip":
        write_plain_gzip(path, text)
    else:
        with open(path, "wb") as fh:
            fh.write(text)
    return path


# ---- numpy restatement ------------------------------------------------------------------------------------------------
class Records:
    """Start-sorted records per contig with their obs row (-1 when the barcode is not an obs name)."""

    def __init__(self, rec, index_of):
        self.rec = rec
        self.cell = np.array([index_of.get(n, -1) for n in rec["name"]], dtype=np.int64)
        self.span = {}
        for i, c in enumerate(rec["contig"]):
            if c not in self.span:
                self.span[c] = [i, i + 1]
            else:
                self.span[c][1] = i + 1
        self.lmax = int((rec["end"] - rec["start"]).max()) if len(rec["start"]) else 0

    def hits(self, contig, lo, hi):
        a, b = self.span[contig]
        st = self.rec["start"][a:b]
        j0 = a + np.searchsorted(st, lo - self.lmax + 1)
        j1 = a + np.searchsorted(st, hi)
        j = np.arange(j0, max(j0, j1))
        j = j[(self.rec["end"][j] > lo) & (self.cell[j] >= 0)]
        return j


def count_ref(R: Records, windows, n_obs, count_reads=True):
    """cells x features int64 counts; ``windows`` = (contig, lo, hi) per feature."""
    import scipy.sparse as sp
    rows, cols, vals = [], [], []
    for f, (c, lo, hi) in enumerate(windows):
        j = R.hits(c, lo, hi)
        rows.append(R.cell[j])
        cols.append(np.full(len(j), f))
        vals.append(R.rec["score"][j] if count_reads else np.ones(len(j), np.int64))
    cat = (lambda v: np.concatenate(v) if v else np.zeros(0, np.int64))
    m = sp.csr_matrix((cat(vals), (cat(rows), cat(cols))), shape=(n_obs, len(windows)), dtype=np.int64)
    m.sum_duplicates()
    m.sort_indices()
    return m


def tss_ref(R: Records, tss, n_obs, up, down):
    """``_tss_pileup`` + ``_calculate_tss_score``: (X float64, tss_score); ``tss`` = (contig, Start) per feature."""
    width = up + down + 1
    diff = np.zeros((n_obs, width + 1), dtype=np.int64)
    for c, s in tss:
        lo = s - up
        j = R.hits(c, lo, s + down)
        cs = np.maximum(R.rec["start"][j] - lo, 0)
        ce = np.minimum(R.rec["end"][j] - lo, width)
        np.add.at(diff, (R.cell[j], cs), R.rec["score"][j])
        np.add.at(diff, (R.cell[j], ce), -R.rec["score"][j])
    pile = np.cumsum(diff[:, :width], axis=1)
    if 1001 > width:
        raise ValueError(f"`center_size` (1001) must smaller than the piled up region ({width}).")
    flank = np.hstack((pile[:, :100], pile[:, -100:])).mean(axis=1)
    flank[flank == 0] = flank.mean()
    cd = (width - 1001) // 2
    with np.errstate(invalid="ignore", divide="ignore"):
        import warnings
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", RuntimeWarning)
            center = pile[:, cd:-cd].mean(axis=1)
        return pile / flank[:, None], center / flank, pile


def nucleosome_ref(R: Records, n, n_obs, free_ub=147, mono_ub=294):
    """``nucleosome_signal`` over the first ``n`` records (StopIteration when the file holds fewer)."""
    if len(R.cell) < n:
        raise StopIteration
    cell = R.cell[:n]
    length = (R.rec["end"] - R.rec["start"])[:n]
    keep = cell >= 0
    mat = np.zeros((n_obs, 2), dtype=np.int64)
    free = keep & (length < free_ub)
    mono = keep & ~(length < free_ub) & (length < mono_ub)
    np.add.at(mat[:, 0], cell[free], 1)
    np.add.at(mat[:, 1], cell[mono], 1)
    mat[mat[:, 0] == 0, :] += 1
    return mat[:, 1] / mat[:, 0]


# ---- the reference functions ------------------------------------------------------------------------------------------
def load_reference_fragments():
    """``locate_fragments``, ``count_fragments_features``, ``tss_enrichment`` and ``nucleosome_signal`` of the
    unmodified muon/_atac/tools.py (and ``get_gene_annotation_from_rna`` of muon/_rna/utils.py), with this module as
    ``pysam`` and an ``AnnData`` stand-in that accepts ``dtype=``."""
    from . import _refload as RL
    if not RL.reference_available():
        raise FileNotFoundError(RL.REF_ROOT)
    RL._install_stubs()
    from muon_b200._containers import SimpleAnnData, SimpleMuData

    class _Meta(type):
        def __instancecheck__(cls, obj):
            return isinstance(obj, SimpleAnnData)

    class RefAnnData(SimpleAnnData, metaclass=_Meta):
        def __init__(self, X=None, obs=None, var=None, dtype=None, **kw):
            if dtype is not None and X is not None:
                X = X.astype(dtype)
            super().__init__(X=X, obs=obs, var=var, **kw)

    sys.modules["pysam"] = pysam_module()
    pkgs = ("_reffrag", "_reffrag._atac", "_reffrag._rna")
    for name in pkgs:
        if name not in sys.modules:
            p = types.ModuleType(name)
            p.__path__ = []
            sys.modules[name] = p
    sys.modules["_reffrag"].MuData = SimpleMuData
    au = types.ModuleType("_reffrag._atac.utils")
    sys.modules["_reffrag._atac.utils"] = au
    sys.modules["_reffrag._atac"].utils = au
    ru = sys.modules.get("_reffrag._rna.utils") or RL._load("muon/_rna/utils.py", "_reffrag._rna.utils")
    tools = sys.modules.get("_reffrag._atac.tools") or RL._load("muon/_atac/tools.py", "_reffrag._atac.tools")
    tools.AnnData = RefAnnData
    ru.AnnData = RefAnnData
    return types.SimpleNamespace(locate_fragments=tools.locate_fragments,
                                 count_fragments_features=tools.count_fragments_features,
                                 tss_enrichment=tools.tss_enrichment, nucleosome_signal=tools.nucleosome_signal,
                                 get_gene_annotation_from_rna=ru.get_gene_annotation_from_rna, module=tools)
