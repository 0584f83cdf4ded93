"""The fragments tools on a synthetic 10x-like fragments file, one H100.

    python profiles/bench_fragments.py [fragments=1e8] [cells=10000] [genes=20000] [tss=2000]
    python profiles/bench_fragments.py --cpu [fragments=1e6]     # the reference functions, no GPU

The file (not timed) is written to a temporary directory as BGZF with a ``.tbi`` holding the linear index (no
binning index: the reader does not use it).  Lines have fixed-width zero-padded fields so that the file can be built
with numpy: ``chrNN  start  end  BCnnnnnn-1  score``.  Fragments are spread uniformly over 20 contigs of 150 Mb with a
nucleosomal length mixture.  Each of ``count_fragments_features`` (``genes`` windows of 2-100 kb), ``tss_enrichment``
(``tss`` TSSs, through the index and by a full pass) and ``nucleosome_signal`` (every fragment) runs once as warm-up
and once timed.  Printed per stage: host inflate alone (with its thread count), upload and parse, each kernel (CUDA
events), host assembly and the whole call, and the card's name and power limit.

``--cpu`` runs the unmodified reference functions with the pysam stand-in of oracle/fragments_ref.py on a slice of
``fragments`` records and extrapolates linearly; it excludes pysam's own fetch cost.  Prints one JSON line.
"""
import json
import os
import subprocess
import sys
import tempfile
import time
import warnings
from concurrent.futures import ThreadPoolExecutor

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import fragments_ref as O  # noqa: E402

CONTIG_LEN = 150_000_000
N_CONTIGS = 20
WIDTH = 40          # chrNN \t 9 \t 9 \t BCnnnnnn-1 \t d \n


def args():
    rest = [a for a in sys.argv[1:] if not a.startswith("--")]
    vals = [int(float(a)) for a in rest]
    return vals


def digits(out, col, v, w):
    for k in range(w - 1, -1, -1):
        out[:, col + k] = 48 + v % 10
        v = v // 10


def make_file(tmp, n, n_cells, seed=0):
    """BGZF file + .tbi of n fixed-width fragments; returns (path, per-contig start arrays)."""
    rng = np.random.default_rng(seed)
    per = rng.multinomial(n, np.full(N_CONTIGS, 1.0 / N_CONTIGS))
    path = os.path.join(tmp, "fragments.tsv.gz")
    block = O.BGZF_BLOCK - O.BGZF_BLOCK % WIDTH
    lin = {}
    off = 0
    pool = ThreadPoolExecutor(os.cpu_count() or 8)
    coffs = []
    pos = 0

    def compress(b):
        c = __import__("zlib").compressobj(1, 8, -15)
        payload = c.compress(b) + c.flush()
        import struct
        import zlib
        head = struct.pack("<BBBBIBBHBBHH", 0x1F, 0x8B, 8, 4, 0, 0, 0xFF, 6, 66, 67, 2, 18 + len(payload) + 8 - 1)
        return head + payload + struct.pack("<II", zlib.crc32(b) & 0xFFFFFFFF, len(b))

    contig_records = []
    with open(path, "wb") as fh:
        for ci in range(N_CONTIGS):
            k = int(per[ci])
            s = np.sort(rng.integers(0, CONTIG_LEN - 2000, k))
            ln = np.where(rng.random(k) < 0.55, rng.integers(30, 147, k),
                          np.where(rng.random(k) < 0.8, rng.integers(147, 294, k), rng.integers(294, 1000, k)))
            e = s + ln
            cell = rng.integers(0, int(n_cells * 1.2), k)
            sc = rng.integers(1, 6, k)
            contig_records.append((s, e))
            t = np.empty((k, WIDTH), np.uint8)
            t[:, 0:3] = np.frombuffer(b"chr", np.uint8)
            digits(t, 3, np.full(k, ci + 1), 2)
            t[:, 5] = 9
            digits(t, 6, s, 9)
            t[:, 15] = 9
            digits(t, 16, e, 9)
            t[:, 25] = 9
            t[:, 26:28] = np.frombuffer(b"BC", np.uint8)
            digits(t, 28, cell, 6)
            t[:, 34:36] = np.frombuffer(b"-1", np.uint8)
            t[:, 36] = 9
            t[:, 37] = 48 + sc
            t[:, 38] = 10
            t = t[:, :39]                                  # 39 bytes per line
            raw = t.tobytes()
            # the linear index: the text offset of the first record overlapping each 16 kb window
            first = np.full(e.max() // 16384 + 2, np.iinfo(np.int64).max)
            idx = off + np.arange(k, dtype=np.int64) * 39
            np.minimum.at(first, s >> 14, idx)
            np.minimum.at(first, (e - 1) >> 14, idx)
            lin[f"chr{ci + 1:02d}"] = first
            off += len(raw)
            blocks = [raw[j:j + block] for j in range(0, len(raw), block)]
            for b in pool.map(compress, blocks):
                coffs.append(pos)
                fh.write(b)
                pos += len(b)
        fh.write(O.BGZF_EOF)
    coffs = np.array(coffs, dtype=np.int64)
    # text offsets -> virtual offsets (the text is one stream; blocks are `block` bytes except at contig ends)
    import struct
    blocks_start = []
    u = 0
    for ci in range(N_CONTIGS):
        k = int(per[ci]) * 39
        blocks_start.extend(range(u, u + k, block))
        u += k
    blocks_start = np.array(blocks_start, dtype=np.int64)
    names = list(lin)
    body = [b"TBI\x01", struct.pack("<8i", len(names), O.TBX_UCSC, 1, 2, 3, 35, 0,
                                     sum(len(c) + 1 for c in names)), b"".join(c.encode() + b"\0" for c in names)]
    for c in names:
        f = lin[c]
        prev = np.maximum.accumulate(np.where(f == np.iinfo(np.int64).max, -1, f))
        f = np.where(f == np.iinfo(np.int64).max, np.maximum(prev, 0), f)
        b = np.searchsorted(blocks_start, f, side="right") - 1
        v = (coffs[b].astype(np.uint64) << np.uint64(16)) | (f - blocks_start[b]).astype(np.uint64)
        body += [struct.pack("<i", 0), struct.pack("<i", len(v)), v.astype("<u8").tobytes()]
    rawi = b"".join(body)
    with open(path + ".tbi", "wb") as fh:
        for j in range(0, len(rawi), O.BGZF_BLOCK):
            fh.write(O.bgzf_block(rawi[j:j + O.BGZF_BLOCK]))
        fh.write(O.BGZF_EOF)
    return path, per


def features(n_genes, n_tss, seed=1, contig_len=None):
    import pandas as pd
    rng = np.random.default_rng(seed)
    ch = [f"chr{c:02d}" for c in rng.integers(1, N_CONTIGS + 1, n_genes)]
    st = rng.integers(10_000, (contig_len or CONTIG_LEN) - 200_000, n_genes)
    g = pd.DataFrame({"Chromosome": ch, "Start": st, "End": st + rng.integers(2_000, 100_000, n_genes)})
    return g, g.iloc[:n_tss].copy()


def make_adata(n_cells, path):
    import pandas as pd

    from muon_b200._containers import SimpleAnnData
    obs = pd.DataFrame(index=pd.Index([f"BC{i:06d}-1" for i in range(n_cells)]))
    ad = SimpleAnnData(np.zeros((n_cells, 1), np.float32), obs=obs)
    ad.uns["files"] = {"fragments": path}
    return ad


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip()


def gpu(n, n_cells, n_genes, n_tss):
    import torch

    import muon_b200 as mu
    from muon_b200 import _fragments as F
    from muon_b200 import _lib
    assert torch.cuda.is_available(), "the benchmark needs a GPU"
    out = {"card": card(), "fragments": n, "cells": n_cells, "genes": n_genes, "tss": n_tss}
    with tempfile.TemporaryDirectory() as tmp:
        t0 = time.perf_counter()
        path, _ = make_file(tmp, n, n_cells)
        out["file_gb"] = round(os.path.getsize(path) / 1e9, 3)
        out["make_file_s"] = round(time.perf_counter() - t0, 1)
        genes, tss = features(n_genes, n_tss)
        t0 = time.perf_counter()
        nb = 0
        with ThreadPoolExecutor(F.threads()) as pool:
            for p in F.file_pieces(path, pool):
                nb += len(p)
        dt = time.perf_counter() - t0
        out["inflate"] = {"s": round(dt, 3), "threads": F.threads(), "text_gb": round(nb / 1e9, 3),
                          "text_gb_per_s": round(nb / 1e9 / dt, 3)}
        calls = {
            "count_fragments_features": lambda ad: mu.atac.tl.count_fragments_features(ad, genes, count_reads=False),
            "tss_enrichment_index": lambda ad: mu.atac.tl.tss_enrichment(ad, tss, n_tss=n_tss),
            "tss_enrichment_full_pass": lambda ad: mu.atac.tl.tss_enrichment(ad, tss, n_tss=n_tss, use_index=False),
            "nucleosome_signal": lambda ad: mu.atac.tl.nucleosome_signal(ad, n=n),
        }
        for name, fn in calls.items():
            fn(make_adata(n_cells, path))                     # warm-up
            torch.cuda.synchronize()
            _lib.PHASES = {}
            t0 = time.perf_counter()
            fn(make_adata(n_cells, path))
            torch.cuda.synchronize()
            total = time.perf_counter() - t0
            phases = dict(_lib.PHASES)
            _lib.PHASES = None
            _lib.PROFILE = {}
            fn(make_adata(n_cells, path))
            torch.cuda.synchronize()
            kern = {k: round(sum(a.elapsed_time(b) for a, b in v) / 1e3, 4) for k, v in _lib.PROFILE.items()}
            _lib.PROFILE = None
            rec = {"call_s": round(total, 3), "phases_s": {k: round(v, 3) for k, v in phases.items()},
                   "kernels_s": kern}
            rec["host_other_s"] = round(total - sum(phases.values()), 3)
            out[name] = rec
        out["peak_device_gb"] = round(torch.cuda.max_memory_allocated() / 1e9, 2)
    return out


def cpu(n):
    ref = O.load_reference_fragments()
    os.environ["TQDM_DISABLE"] = "1"
    n_cells, n_genes, n_tss = 10_000, 20_000, 2_000
    full = 100_000_000
    out = {"fragments_slice": n, "scaled_to": full,
           "note": "reference functions with the pysam stand-in, extrapolated linearly; pysam's fetch cost excluded"}
    with tempfile.TemporaryDirectory() as tmp:
        # a slice with the full file's density: contigs n / full as long, genes and TSSs n / full as many
        global CONTIG_LEN
        keep = CONTIG_LEN
        CONTIG_LEN = int(keep * n / full)
        try:
            path, _ = make_file(tmp, n, n_cells)
            genes, _ = features(max(n_genes * n // full, 1), 0, contig_len=CONTIG_LEN)
            tss, _ = features(max(n_tss * n // full, 1), 0, seed=2, contig_len=CONTIG_LEN)
        finally:
            CONTIG_LEN = keep
        for name, fn in (("count_fragments_features", lambda ad: ref.count_fragments_features(ad, genes,
                                                                                              count_reads=False)),
                         ("tss_enrichment", lambda ad: ref.tss_enrichment(ad, tss, n_tss=n_tss)),
                         ("nucleosome_signal", lambda ad: ref.nucleosome_signal(ad, n=n))):
            ad = make_adata(n_cells, path)
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                t0 = time.perf_counter()
                fn(ad)
                dt = time.perf_counter() - t0
            out[name] = {"slice_s": round(dt, 2), "extrapolated_s": round(dt * full / n, 1)}
    return out


if __name__ == "__main__":
    v = args()
    if "--cpu" in sys.argv:
        print(json.dumps(cpu(v[0] if v else 1_000_000)))
    else:
        d = [100_000_000, 10_000, 20_000, 2_000]
        d[:len(v)] = v
        print(json.dumps(gpu(*d)))
