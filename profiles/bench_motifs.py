"""Benchmark of ``mu.atac.tl.get_sequences`` and ``scan_sequences`` on the GPU.

Workload: a seeded synthetic genome (5 contigs, 60-base lines, runs of N, soft-masked stretches), 200 000 peaks of
500 bases, all 746 JASPAR matrices of tests/golden/jaspar_pfm.npz, pvalue 1e-4.  Reports the scan kernels' time from
CUDA events after a warm-up, the column evaluations per second (sum over motifs of windows x length, from shapes)
against the H100 SXM data-sheet FP64 and FP32 rates, the hit count, the wall time of get_sequences and of
scan_sequences split into upload, kernels, download, DataFrame assembly and join, and the card and its power limit.
``--cpu-peaks N`` also times the array restatement of oracle/motif_ref.py (numpy, the stand-in for MOODS in the
tests; MOODS itself is not measured) on the first N peaks.

    python profiles/bench_motifs.py [--peaks 200000] [--width 500] [--cpu-peaks 200]

Writes nothing in the tree: the genome goes to a temporary directory.  Prints one JSON line.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FP64_PEAK, FP32_PEAK = 34e12, 67e12          # H100 SXM data sheet, non-tensor FLOP/s at 700 W


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception:   # noqa: BLE001
        import torch
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def write_genome(path, seed, contig_len=(30_000_000, 25_000_000, 20_000_000, 15_000_000, 12_000_000)):
    rng = np.random.default_rng(seed)
    with open(path, "wb") as fh:
        for i, n in enumerate(contig_len):
            b = rng.choice(np.frombuffer(b"ACGT", np.uint8), n)
            for a in rng.integers(0, n - 5000, n // 200_000):
                b[a:a + int(rng.integers(10, 5000))] = ord("N")
            for a in rng.integers(0, n - 2000, n // 20_000):
                s = slice(a, a + int(rng.integers(50, 2000)))
                b[s] = np.where(b[s] != ord("N"), b[s] | 0x20, b[s])
            fh.write(f">chr{i + 1}\n".encode())
            body = b.tobytes()
            fh.write(b"\n".join(body[k:k + 60] for k in range(0, n, 60)) + b"\n")
    return contig_len


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--peaks", type=int, default=200_000)
    ap.add_argument("--width", type=int, default=500)
    ap.add_argument("--cpu-peaks", type=int, default=0)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()

    import pandas as pd
    import torch

    import muon_b200 as mu
    from muon_b200 import _lib
    from muon_b200._containers import SimpleAnnData
    from muon_b200._motifs import MotifScanner, background_of, log_odds

    assert torch.cuda.is_available(), "bench_motifs needs a GPU"
    z = np.load(os.path.join(ROOT, "tests", "golden", "jaspar_pfm.npz"))
    off = np.concatenate([[0], np.cumsum(z["lengths"])])
    bg = background_of(4)
    mats = [log_odds(z["counts"][:, off[i]:off[i + 1]], bg, 0.0001) for i in range(len(z["names"]))]
    ids = [str(n).rstrip(".pfm") for n in z["names"]]
    meta = pd.DataFrame({"motif_id": z["meta_id"], "tf_gene_name": z["meta_gene"]}).set_index("motif_id")
    out = {"card": card(), "peaks": args.peaks, "width": args.width, "motifs": len(mats)}
    with tempfile.TemporaryDirectory() as tmp:
        fa = os.path.join(tmp, "genome.fa")
        lens = write_genome(fa, args.seed)
        rng = np.random.default_rng(args.seed + 1)
        chrom = rng.integers(0, len(lens), args.peaks)
        start = rng.integers(0, np.array(lens)[chrom] - args.width)
        names = [f"chr{c + 1}:{s}-{s + args.width}" for c, s in zip(chrom, start)]
        ad = SimpleAnnData(np.zeros((1, len(names)), np.float32), var=pd.DataFrame(index=pd.Index(names)))
        t = time.perf_counter()
        seqs = mu.atac.tl.get_sequences(ad, None, fa)
        out["get_sequences_s"] = time.perf_counter() - t

    t = time.perf_counter()
    scanner = MotifScanner(mats, 4, 1e-4)
    out["thresholds_s"] = time.perf_counter() - t
    warm = mu.atac.tl.scan_sequences(seqs[:2000], motif_scanner=scanner, motifs=ids)      # uploads the tables
    del warm
    _lib.PROFILE = {}
    timings = {}
    torch.cuda.synchronize()
    t = time.perf_counter()
    from muon_b200._motifs import scan_sequences
    df = scan_sequences(seqs, scanner, None, ids, meta, 4, 1e-4, 10, timings=timings)
    out["scan_sequences_s"] = time.perf_counter() - t
    torch.cuda.synchronize()
    ev = {k: sum(a.elapsed_time(b) for a, b in v) for k, v in _lib.PROFILE.items()}
    _lib.PROFILE = None
    out["kernel_ms"] = {k: round(v, 3) for k, v in ev.items()}
    out["split_s"] = {k: round(v, 4) for k, v in timings.items()}
    out["hits"] = len(df)
    L = np.array([m.shape[1] for m in mats])
    n = np.array([len(s) for s in seqs])
    evals = int(sum(np.clip(n - l + 1, 0, None).sum() * l for l in L))
    out["column_evaluations"] = evals
    rate = evals / (ev["mub_motif_count"] / 1e3)          # the count pass evaluates every column once
    out["evals_per_s_count_pass"] = rate
    out["share_fp64_peak_count_pass"] = rate / FP64_PEAK       # one float64 add per evaluation
    out["share_fp32_peak_count_pass"] = rate / FP32_PEAK
    out["peak_mem_gib"] = torch.cuda.max_memory_allocated() / 2**30
    if args.cpu_peaks:
        from oracle import motif_ref as O
        tabs = O.tables(mats)
        t = time.perf_counter()
        for s in seqs[:args.cpu_peaks]:
            O.scan_restated(O.codes_of(s), tabs, scanner.thresholds)
        cpu = time.perf_counter() - t
        out["numpy_restatement_s"] = cpu
        out["numpy_restatement_peaks"] = args.cpu_peaks
        out["numpy_restatement_extrapolated_s"] = cpu * len(seqs) / args.cpu_peaks
    print(json.dumps(out))


if __name__ == "__main__":
    main()
