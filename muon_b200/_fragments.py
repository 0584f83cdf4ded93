"""The fragments file on the GPU: ``count_fragments_features``, ``tss_enrichment`` and ``nucleosome_signal`` of
muon/_atac/tools.py:746-1201 without a per-fragment Python loop.

The host inflates the file into text chunks cut at their last newline.  A BGZF file (the tabix format) is split into
its blocks, which a thread pool inflates (``zlib`` releases the GIL); any other gzip stream is inflated sequentially,
and plain text is read as is.  Each chunk goes through a pinned buffer to the device, where csrc/fragments.cu finds
the line starts, parses the five fields of every line, looks its barcode up in an open-addressing table and marks
where a new chromosome begins.  The host reads back only those contig runs and checks that the file is
coordinate-sorted.  The records then stay on the device for the counting kernels.

``tss_enrichment`` reads only the windows it needs when ``<path>.tbi`` exists: each window starts at the linear-index
offset of its first 16 kb bin, windows whose byte ranges overlap are merged so that each block is inflated once, and
reading stops at the first record past the window.  Every virtual offset used is checked (a BGZF header at the block
offset, a line start at the in-block offset); a check that fails warns and falls back to a full pass.
"""
from __future__ import annotations

import os
import struct
import warnings
import zlib
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from ._lib import call, load, phase, ptr, stream_ptr

CHUNK_BYTES = 256 << 20          # text per device chunk
READ_BYTES = 64 << 20            # compressed bytes read per batch of BGZF blocks
LIDX_SHIFT = 14                  # tabix linear index: 16 kb windows
_M = (1 << 63) - 1


def threads() -> int:
    return max(1, min(32, os.cpu_count() or 1))


# ---- inflating -----------------------------------------------------------------------------------------------------
def _bgzf_block_size(buf, off):
    """Total size of the BGZF block at ``buf[off:]``, or None when no BGZF header sits there."""
    if len(buf) - off < 18 or buf[off] != 0x1F or buf[off + 1] != 0x8B or buf[off + 2] != 8 or not buf[off + 3] & 4:
        return None
    xlen = struct.unpack_from("<H", buf, off + 10)[0]
    p, end = off + 12, off + 12 + xlen
    while p + 4 <= end:
        si1, si2, slen = buf[p], buf[p + 1], struct.unpack_from("<H", buf, p + 2)[0]
        if si1 == 66 and si2 == 67 and slen == 2:
            return struct.unpack_from("<H", buf, p + 4)[0] + 1
        p += 4 + slen
    return None


def _inflate_block(blk):
    xlen = struct.unpack_from("<H", blk, 10)[0]
    return zlib.decompress(blk[12 + xlen:-8], -15)


def is_bgzf(path) -> bool:
    with open(path, "rb") as fh:
        return _bgzf_block_size(fh.read(64), 0) is not None


def _bgzf_pieces(path, pool):
    """Inflated text of a BGZF file, in pieces of whole blocks, blocks inflated in parallel."""
    with open(path, "rb") as fh:
        rest = b""
        while True:
            data = fh.read(READ_BYTES)
            buf = rest + data
            blocks, off = [], 0
            while True:
                size = _bgzf_block_size(buf, off)
                if size is None:
                    if len(buf) - off >= 18:
                        raise ValueError(f"{path}: no BGZF block header where one should start")
                    break
                if off + size > len(buf):
                    break
                blocks.append(memoryview(buf)[off:off + size])
                off += size
            rest = buf[off:]
            if blocks:
                yield b"".join(pool.map(_inflate_block, blocks, chunksize=64))
            if not data:
                if rest:
                    raise ValueError(f"{path}: truncated BGZF file")
                return


def _gzip_pieces(path):
    d = zlib.decompressobj(31)
    with open(path, "rb") as fh:
        while True:
            data = fh.read(READ_BYTES)
            if not data:
                break
            while data:
                yield d.decompress(data)
                if d.eof:                       # concatenated gzip members
                    data = d.unused_data
                    d = zlib.decompressobj(31)
                else:
                    data = b""
        yield d.flush()


def _plain_pieces(path):
    with open(path, "rb") as fh:
        while True:
            data = fh.read(READ_BYTES)
            if not data:
                return
            yield data


def text_chunks(pieces, chunk_bytes=CHUNK_BYTES):
    """Regroup text pieces into chunks of about ``chunk_bytes`` that end with a newline (the remainder is carried to
    the next chunk; a last line without one gets one)."""
    rest = b""
    for p in pieces:
        if not p:
            continue
        buf = rest + p if rest else p
        pos = 0
        while len(buf) - pos >= chunk_bytes:
            cut = buf.rfind(b"\n", pos, pos + chunk_bytes)
            if cut < 0:
                cut = buf.find(b"\n", pos + chunk_bytes)
                if cut < 0:
                    break
            yield buf[pos:cut + 1]
            pos = cut + 1
        rest = buf[pos:]
    if rest:
        yield rest if rest.endswith(b"\n") else rest + b"\n"


def file_pieces(path, pool):
    with open(path, "rb") as fh:
        head = fh.read(2)
    if is_bgzf(path):
        return _bgzf_pieces(path, pool)
    if head == b"\x1f\x8b":
        return _gzip_pieces(path)
    return _plain_pieces(path)


# ---- the tabix index ------------------------------------------------------------------------------------------------
def read_tbi(path):
    """``{contig: ioff}`` of a ``.tbi`` file: the linear index (uint64 virtual offsets of 16 kb windows) per contig,
    names in index order.  Raises ValueError on a malformed index."""
    import gzip
    with gzip.open(path, "rb") as fh:
        raw = fh.read()
    if raw[:4] != b"TBI\x01":
        raise ValueError(f"{path}: not a tabix index")
    n_ref, _fmt, _cs, _cb, _ce, _meta, _skip, l_nm = struct.unpack_from("<8i", raw, 4)
    p = 36
    names = [s.decode() for s in raw[p:p + l_nm].split(b"\0")[:n_ref]]
    p += l_nm
    out = {}
    for name in names:
        (n_bin,) = struct.unpack_from("<i", raw, p)
        p += 4
        for _ in range(n_bin):
            _bin, n_chunk = struct.unpack_from("<Ii", raw, p)
            p += 8 + 16 * n_chunk
        (n_intv,) = struct.unpack_from("<i", raw, p)
        p += 4
        out[name] = np.frombuffer(raw, dtype="<u8", count=n_intv, offset=p).copy()
        p += 8 * n_intv
        if p > len(raw):
            raise ValueError(f"{path}: truncated tabix index")
    return out


class _BlockReader:
    """Random access to the inflated BGZF blocks of a file, each block inflated at most once."""

    def __init__(self, path):
        self.fh = open(path, "rb")
        self.cache = {}

    def block(self, coff):
        got = self.cache.get(coff)
        if got is None:
            self.fh.seek(coff)
            head = self.fh.read(18)
            size = _bgzf_block_size(head, 0)
            if size is None:
                return None
            blk = head + self.fh.read(size - 18)
            got = (_inflate_block(blk), coff + size)
            self.cache[coff] = got
        return got

    def close(self):
        self.fh.close()


def _last_line(buf: bytes):
    """(contig, start) of the last complete line of ``buf``, or None."""
    e = buf.rfind(b"\n")
    if e < 0:
        return None
    s = buf.rfind(b"\n", 0, e) + 1
    f = buf[s:e].split(b"\t", 3)
    if len(f) < 3 or f[0].startswith(b"#"):
        return None
    try:
        return f[0].decode(), int(f[1])
    except ValueError:
        return None


def indexed_text(path, windows, ioff):
    """Text of the records a set of windows needs, read through the linear index: the file's lines from each window's
    first candidate through the first line past the window, overlapping ranges merged, in file order.  ``windows`` =
    [(contig, lo, hi)]; ``ioff`` = ``read_tbi`` of the file.  Returns None (after a warning) when an offset fails its
    check."""
    rank = {c: i for i, c in enumerate(ioff)}
    starts = []
    for c, lo, hi in windows:
        lin = ioff.get(c)
        if lin is None or lo >> LIDX_SHIFT >= len(lin):
            continue                                   # no record of the contig reaches the window
        starts.append((int(lin[lo >> LIDX_SHIFT]), rank[c], hi))
    starts.sort()
    rd = _BlockReader(path)
    try:
        parts, covered = [], -1              # covered: virtual offset just past the text taken so far
        for voff, r, hi in starts:
            voff = max(voff, covered)
            coff, uoff = voff >> 16, voff & 0xFFFF
            got = rd.block(coff)
            if got is None or uoff > len(got[0]) or (uoff and got[0][uoff - 1] != 10):
                warnings.warn(f"{path}.tbi: virtual offset {voff:#x} does not point at a line of {path}; "
                              "reading the whole file instead")
                return None
            segs, coffs, nxt = [got[0][uoff:]], [coff], got[1]
            while True:          # until the last complete line lies past the window (sorted file)
                last = _last_line(b"".join(segs))
                if last is not None and (rank.get(last[0], len(rank)) > r
                                         or (rank.get(last[0]) == r and last[1] >= hi)):
                    break
                more = rd.block(nxt)
                if more is None or not more[0]:
                    break
                segs.append(more[0])
                coffs.append(nxt)
                nxt = more[1]
            joined = b"".join(segs)
            cut = joined.rfind(b"\n") + 1
            if cut == 0:
                continue
            tail, k = len(joined) - cut, len(segs) - 1
            while tail > len(segs[k]):
                tail -= len(segs[k])
                k -= 1
            covered = (coffs[k] << 16) | (len(segs[k]) - tail + (uoff if k == 0 else 0))
            parts.append(joined[:cut])
        return b"".join(parts)
    finally:
        rd.close()


# ---- barcodes ---------------------------------------------------------------------------------------------------------
class BarcodeTable:
    """Device open-addressing table from barcode strings to obs rows (``index_of``: str -> row, duplicates already
    resolved by the caller)."""

    def __init__(self, index_of, device):
        import torch
        names = [k for k in index_of if isinstance(k, str)]
        enc = [k.encode() for k in names]
        off = np.zeros(len(enc) + 1, dtype=np.int64)
        np.cumsum([len(b) for b in enc], out=off[1:])
        self.n = len(enc)
        self.cap = 16
        while self.cap < 2 * self.n:
            self.cap *= 2
        self.bytes = torch.from_numpy(np.frombuffer(b"".join(enc) or b"\0", dtype=np.uint8).copy()).to(device)
        self.off = torch.from_numpy(off).to(device)
        self.val = torch.tensor([index_of[k] for k in names], dtype=torch.int32).to(device) if names else \
            torch.zeros(1, dtype=torch.int32, device=device)
        self.keys = torch.zeros(self.cap, dtype=torch.int64, device=device)
        self.slot = torch.zeros(self.cap, dtype=torch.int32, device=device)
        call("mub_frag_barcode_table", ptr(self.bytes), ptr(self.off), self.n, ptr(self.keys), ptr(self.slot),
             self.cap, stream_ptr())


# ---- parsing --------------------------------------------------------------------------------------------------------
class Records:
    """Parsed records on the device (int32 start, end, score, cell), start-sorted within each contig; ``contigs``
    maps a contig to its record range, in file order; ``lmax`` is the longest fragment."""

    def __init__(self, start, end, score, cell, contigs, lmax):
        self.start, self.end, self.score, self.cell = start, end, score, cell
        self.contigs, self.lmax = contigs, lmax

    @property
    def n(self):
        return int(self.start.numel())


def parse_chunks(chunks, table: BarcodeTable, device, max_records=None, stats=None):
    """Parse text chunks on the device.  Stops once ``max_records`` records are parsed (all of them are returned).
    Raises ValueError for a malformed or unsorted file and NotImplementedError for coordinates beyond int32."""
    import torch
    tile = load().mub_frag_tile_bytes()
    pinned = None
    cols = {k: [] for k in ("start", "end", "score", "cell")}
    contigs, order = {}, []
    n_rec, line_base, lmax = 0, 0, 0
    last_start = None
    s = stream_ptr()
    for text in chunks:
        nb = len(text)
        with phase("fragments.upload"):
            if pinned is None or pinned.numel() < nb:
                torch.cuda.current_stream().synchronize()
                pinned = torch.empty(max(nb, 1), dtype=torch.uint8, pin_memory=True)
            else:
                torch.cuda.current_stream().synchronize()      # the previous chunk's copy has left the buffer
            pinned.numpy()[:nb] = np.frombuffer(text, dtype=np.uint8)
            dev = pinned[:nb].to(device, non_blocking=True)
        with phase("fragments.parse"):
            tiles = (nb + tile - 1) // tile
            tc = torch.empty(tiles + 1, dtype=torch.int64, device=device)
            tc[0] = 0
            call("mub_frag_newline_count", ptr(dev), nb, ptr(tc[1:]), s)
            toff = torch.cumsum(tc, 0)
            n_lines = int(toff[-1])
            nl = torch.empty(max(n_lines, 1), dtype=torch.int64, device=device)
            call("mub_frag_newline_fill", ptr(dev), nb, ptr(toff), ptr(nl), s)
            st = torch.empty(n_lines, dtype=torch.int32, device=device)
            en, sc, ce = torch.empty_like(st), torch.empty_like(st), torch.empty_like(st)
            fl = torch.empty(n_lines, dtype=torch.uint8, device=device)
            status = torch.tensor([_M, _M, _M, 0, 0], dtype=torch.int64, device=device)
            call("mub_frag_parse", ptr(dev), ptr(nl), n_lines, line_base, ptr(table.bytes), ptr(table.off),
                 ptr(table.val), ptr(table.keys) if table.n else None, ptr(table.slot), table.cap, ptr(st), ptr(en),
                 ptr(sc), ptr(ce), ptr(fl), ptr(status), s)
            stat = status.cpu().tolist()
            keep = None
            if stat[4]:
                keep = torch.nonzero((fl & 2) == 0).flatten()
                st, en, sc, ce, fl = st[keep], en[keep], sc[keep], ce[keep], fl[keep]
            n_here = int(st.numel())
            # the last line that matters: the max_records-th record when it falls in this chunk
            limit_line = None
            if max_records is not None and n_rec + n_here >= max_records:
                m = max_records - n_rec
                if m > 0:
                    limit_line = line_base + (int(keep[m - 1]) if keep is not None else m - 1)
                else:
                    limit_line = line_base - 1
            lim = _M - 1 if limit_line is None else limit_line     # an unset status word stays at _M
            if stat[0] <= lim:
                raise ValueError(f"fragments file: line {stat[0] + 1} is not a BED line with 5 tab-separated fields "
                                 "(chrom, start, end, barcode, integer score)")
            if stat[1] <= lim:
                raise NotImplementedError(f"fragments file: line {stat[1] + 1} has a coordinate or score beyond int32")
            if stat[2] <= lim:
                raise ValueError(f"fragments file is not coordinate-sorted (line {stat[2] + 1}); sort it as tabix "
                                 "requires")
            lmax = max(lmax, stat[3])
            # contig runs: names from the host copy of the text
            runs = torch.nonzero(fl & 1).flatten()
            if runs.numel():
                line_at = runs if keep is None else keep[runs]
                starts_of = torch.where(line_at > 0, nl[(line_at - 1).clamp_min(0)] + 1, torch.zeros_like(line_at))
                run_pos = runs.cpu().numpy()
                run_off = starts_of.cpu().numpy()
                run_start = st[runs].cpu().numpy()
                for r, o, s0 in zip(run_pos, run_off, run_start):
                    if limit_line is not None and n_rec + int(r) >= max_records:
                        break
                    e = text.index(b"\t", o)
                    name = text[o:e].decode()
                    g = n_rec + int(r)
                    if order and order[-1] == name:                 # the same contig across a chunk boundary
                        prev = last_start if int(r) == 0 else int(st[r - 1])
                        if prev is not None and s0 < prev:
                            raise ValueError(f"fragments file is not coordinate-sorted (contig {name})")
                        continue
                    if name in contigs:
                        raise ValueError(f"fragments file is not coordinate-sorted: contig {name} appears in two runs")
                    if order:
                        contigs[order[-1]][1] = g
                    order.append(name)
                    contigs[name] = [g, g]
            if n_here:
                last_start = int(st[-1])
            for k, v in zip(("start", "end", "score", "cell"), (st, en, sc, ce)):
                cols[k].append(v)
            n_rec += n_here
            line_base += n_lines
            if stats is not None:
                stats["bytes"] = stats.get("bytes", 0) + nb
            del dev, nl, tc, toff
        if max_records is not None and n_rec >= max_records:
            break
    if order:
        contigs[order[-1]][1] = n_rec
    cat = {k: (torch.cat(v) if v else torch.zeros(0, dtype=torch.int32, device=device)) for k, v in cols.items()}
    return Records(cat["start"], cat["end"], cat["score"], cat["cell"], {k: tuple(v) for k, v in contigs.items()},
                   int(lmax))


def read_records(path, index_of, device, *, max_records=None, chunk_bytes=CHUNK_BYTES, stats=None):
    table = BarcodeTable(index_of, device)
    with ThreadPoolExecutor(threads()) as pool:
        return parse_chunks(text_chunks(file_pieces(path, pool), chunk_bytes), table, device, max_records, stats)


def contigs_of(path):
    """Contigs of a file when its ``.tbi`` can be read, else None."""
    tbi = str(path) + ".tbi"
    if os.path.isfile(tbi) and is_bgzf(path):
        try:
            return read_tbi(tbi)
        except Exception as e:   # noqa: BLE001 -- any unreadable index means a full pass
            warnings.warn(f"{tbi}: unreadable tabix index ({e}); reading the whole file instead")
    return None


# ---- the three computations -------------------------------------------------------------------------------------------
def _query_arrays(R: Records, windows, device):
    import torch
    rl = np.array([R.contigs.get(c, (0, 0))[0] for c, _, _ in windows], dtype=np.int64)
    rh = np.array([R.contigs.get(c, (0, 0))[1] for c, _, _ in windows], dtype=np.int64)
    lo = np.array([w[1] for w in windows], dtype=np.int64)
    hi = np.array([w[2] for w in windows], dtype=np.int64)
    return [torch.from_numpy(a).to(device) for a in (rl, rh, lo, hi)]


def count_matrix(R: Records, windows, n_obs, count_reads, device, batch_entries=1 << 28):
    """cells x features canonical int64 CSR of the fragments overlapping each window (contig, lo, hi)."""
    import scipy.sparse as sp
    import torch
    s = stream_ptr()
    F = len(windows)
    keys, vals = [], []
    with phase("fragments.overlap"):
        q = _query_arrays(R, windows, device)
        counts = torch.zeros(max(F, 1), dtype=torch.int64, device=device)
        call("mub_frag_overlap", ptr(R.start), ptr(R.end), ptr(R.cell), ptr(R.score), ptr(q[0]), ptr(q[1]), ptr(q[2]),
             ptr(q[3]), F, R.lmax, int(bool(count_reads)), 0, ptr(counts), None, None, None, None, s)
        cnt = counts[:F].cpu().numpy()
        # bounded batches of features, each emitting at most batch_entries hits (or one feature)
        f0 = 0
        csum = np.concatenate([[0], np.cumsum(cnt)])
        while f0 < F:
            f1 = int(np.searchsorted(csum, csum[f0] + batch_entries, side="right") - 1)
            f1 = min(max(f1, f0 + 1), F)
            m = int(csum[f1] - csum[f0])
            if m:
                off = torch.from_numpy(csum[f0:f1] - csum[f0]).to(device)
                oc = torch.empty(m, dtype=torch.int32, device=device)
                of = torch.empty(m, dtype=torch.int32, device=device)
                ov = torch.empty(m, dtype=torch.int64, device=device)
                call("mub_frag_overlap", ptr(R.start), ptr(R.end), ptr(R.cell), ptr(R.score), ptr(q[0][f0:f1]),
                     ptr(q[1][f0:f1]), ptr(q[2][f0:f1]), ptr(q[3][f0:f1]), f1 - f0, R.lmax, int(bool(count_reads)),
                     f0, None, ptr(off), ptr(oc), ptr(of), ptr(ov), s)
                keys.append(oc.to(torch.int64) * F + of.to(torch.int64))
                vals.append(ov)
            f0 = f1
    with phase("fragments.reduce"):
        if keys:
            k = torch.cat(keys)
            v = torch.cat(vals)
            k, perm = torch.sort(k)
            v = v[perm]
            uk, inv = torch.unique_consecutive(k, return_inverse=True)
            sums = torch.zeros(uk.numel(), dtype=torch.int64, device=device).index_add_(0, inv, v)
            rows = (uk // F)
            cols = (uk - rows * F).to(torch.int32)
            indptr = torch.zeros(n_obs + 1, dtype=torch.int64, device=device)
            indptr[1:] = torch.cumsum(torch.bincount(rows, minlength=n_obs), 0)
            data, indices, indptr = sums.cpu().numpy(), cols.cpu().numpy(), indptr.cpu().numpy()
        else:
            data, indices, indptr = np.zeros(0, np.int64), np.zeros(0, np.int32), np.zeros(n_obs + 1, np.int64)
    return sp.csr_matrix((data, indices, indptr), shape=(n_obs, F))


def tss_pileup(R: Records, tss, n_obs, up, down, device):
    """Pileup of the fragments around each TSS (contig, Start): (pile int64 device tensor [n][W+1], flank_sum,
    center_sum, center_count) with the flank and centre of ``_calculate_tss_score`` (100 bp, 1001 bp)."""
    import torch
    width = up + down + 1
    need = n_obs * (width + 1) * 8
    free, _ = torch.cuda.mem_get_info(device)
    if need > free:
        raise NotImplementedError(f"tss_enrichment: the {n_obs} x {width + 1} int64 pileup ({need / 2**30:.1f} GiB) "
                                  f"does not fit in the {free / 2**30:.1f} GiB of free device memory")
    windows = [(c, s0 - up, s0 + down) for c, s0 in tss]
    s = stream_ptr()
    with phase("fragments.tss_pileup"):
        diff = torch.zeros((n_obs, width + 1), dtype=torch.int64, device=device)
        if windows:
            q = _query_arrays(R, windows, device)
            call("mub_frag_tss_pileup", ptr(R.start), ptr(R.end), ptr(R.cell), ptr(R.score), ptr(q[0]), ptr(q[1]),
                 ptr(q[2]), ptr(q[3]), len(windows), R.lmax, width, ptr(diff), s)
        cd = (width - 1001) // 2
        c_lo, c_hi = (cd, width - cd) if cd > 0 else (0, 0)
        sums = torch.empty((n_obs, 2), dtype=torch.int64, device=device)
        call("mub_frag_tss_rows", ptr(diff), n_obs, width, 100, c_lo, c_hi, ptr(sums), s)
    return diff, sums, c_hi - c_lo


def tss_scale(diff, n_obs, width, flank_mean, device):
    import torch
    fm = torch.from_numpy(np.ascontiguousarray(flank_mean, dtype=np.float64)).to(device)
    out = torch.empty((n_obs, width), dtype=torch.float64, device=device)
    call("mub_frag_tss_scale", ptr(diff), n_obs, width, ptr(fm), ptr(out), stream_ptr())
    return out


def nucleosome_counts(R: Records, n, n_obs, free_ub, mono_ub, device):
    import torch
    counts = torch.zeros((n_obs, 2), dtype=torch.int32, device=device)
    call("mub_frag_nucleosome", ptr(R.start), ptr(R.end), ptr(R.cell), n, float(free_ub), float(mono_ub), ptr(counts),
         stream_ptr())
    return counts
