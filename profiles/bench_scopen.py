"""mu.atac.pp.scopen on a synthetic peak matrix, one H100.

    python profiles/bench_scopen.py [cells=20000] [peaks=200000] [density=0.03] [k=30] [--iters 20] [--cpu PEAKS]

The counts are the planted-topic generator's (``_synth.generate_device``), resident on the device and NOT timed.
Phases, each bracketed by device synchronisation:

  * ``pattern``: positives per cell, the pattern fill and the sorted transpose (``Fit.positives`` + ``Fit.build``);
  * ``init``: the fp32 Krylov SVD and the NNDSVD on the host;
  * ``iteration``: ``--iters`` iterations after one warm-up iteration, with the CUDA-event time of every C-ABI call
    split into SpMM, Gram and CD per iteration, and the operand rows the two SpMMs gather (2 nnz k 8 bytes) over the
    SpMM time;
  * ``impute``: clip(W H, 0, 1) for all peaks into one reused device block, without the copy to the host, and the
    same with the copy into a preallocated m x n float64 host array when the host has room for it;
  * ``call``: the whole ``mu.atac.pp.scopen`` with ``max_iter = --iters`` on the first cells x peaks that fit the host
    output (cells fixed, peaks cut).
With ``--cpu PEAKS`` it also times sklearn's coordinate-descent NMF (``_fit_coordinate_descent``, bound +inf) on the
dense X of the first PEAKS peaks on the host CPUs, per iteration.  Prints one JSON line with the card and its power
limit, read in the same run.
"""
import json
import os
import subprocess
import sys
import time
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import muon_b200 as mu  # noqa: E402
from muon_b200 import _lib, _scopen  # noqa: E402
from muon_b200._synth import generate_device  # noqa: E402


def _opt(name, default):
    if name in sys.argv:
        return int(sys.argv[sys.argv.index(name) + 1])
    return default


ITERS = _opt("--iters", 20)
CPU_PEAKS = _opt("--cpu", 0)
args = [a for i, a in enumerate(sys.argv[1:]) if not a.startswith("--") and not sys.argv[i].startswith("--")]
N = int(args[0]) if len(args) > 0 else 20_000
M = int(args[1]) if len(args) > 1 else 200_000
DENSITY = float(args[2]) if len(args) > 2 else 0.03
K = int(args[3]) if len(args) > 3 else 30


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0


def host_free_bytes():
    try:
        for line in open("/proc/meminfo"):
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    except OSError:
        pass
    return 0


def main():
    assert torch.cuda.is_available(), "bench_scopen needs a GPU"
    torch.cuda.set_device(0)
    res = {"card": card(), "cells": N, "peaks": M, "density": DENSITY, "k": K, "iters": ITERS}
    A = generate_device(N, M, DENSITY, seed=3)
    torch.cuda.synchronize()
    fit = _scopen.Fit(A, K)
    counts, t_count = timed(fit.positives)
    s = _scopen.scale_of(counts, 0.0, 0.5)
    _, t_build = timed(lambda: fit.build(s))
    res["nnz"] = fit.nnz
    res["pattern_s"] = t_count + t_build
    (W0, H0), t_init = timed(lambda: _scopen.nndsvd(*fit.svd()))
    res["init_svd_s"] = t_init
    fit.set_factors(W0, H0)
    fit.iterate(1.0, _scopen.UPPER)
    _lib.PROFILE = {}
    _, t_it = timed(lambda: [fit.iterate(1.0, _scopen.UPPER) for _ in range(ITERS)])
    prof, _lib.PROFILE = _lib.PROFILE, None
    torch.cuda.synchronize()
    per = {name: sum(a.elapsed_time(b) for a, b in ev) / ITERS for name, ev in prof.items()}
    res["iteration_ms"] = 1e3 * t_it / ITERS
    res["spmm_ms"] = per.get("mub_scopen_spmm_f64", 0.0)
    res["gram_ms"] = per.get("mub_scopen_gram_f64", 0.0)
    res["cd_ms"] = per.get("mub_scopen_cd_f64", 0.0)
    gathered = 2 * fit.nnz * K * 8
    res["gathered_GB_per_iter"] = gathered / 1e9
    res["spmm_gather_TBps"] = gathered / (res["spmm_ms"] * 1e-3) / 1e12

    rows = max(1, min(M, _scopen.IMPUTE_BLOCK_BYTES // (8 * N)))
    buf = torch.empty(rows * N, dtype=torch.float64, device=fit.dev)

    def impute_device():
        from muon_b200._lib import call, ptr, stream_ptr
        for p0 in range(0, M, rows):
            call("mub_scopen_impute_f64", ptr(fit.W), p0, min(M, p0 + rows), ptr(fit.Ht), N, K, ptr(buf),
                 stream_ptr())
    impute_device()
    _, t_imp = timed(impute_device)
    res["impute_device_s"] = t_imp
    res["impute_device_GBps"] = 8 * M * N / t_imp / 1e9
    del buf
    if host_free_bytes() > 3 * 8 * M * N:
        out = np.empty((M, N))
        _, t_imp_h = timed(lambda: fit.impute(out))
        res["impute_with_copy_s"] = t_imp_h
        del out
    else:
        res["impute_with_copy_s"] = "not measured: host memory"
    del fit, A
    torch.cuda.empty_cache()

    m_call = int(min(M, max(1000, host_free_bytes() // (4 * 8 * N))))
    A = generate_device(N, m_call, DENSITY, seed=3)
    ad = mu.SimpleAnnData(A)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        _, t_call = timed(lambda: mu.atac.pp.scopen(ad, n_components=K, max_iter=ITERS))
    res["call_peaks"] = m_call
    res["call_s"] = t_call
    del ad, A

    if CPU_PEAKS:
        from sklearn.decomposition import _nmf
        Ah = generate_device(N, CPU_PEAKS, DENSITY, seed=3).get()
        P = (Ah > 0).astype(np.float64)
        c = np.asarray(P.sum(axis=1)).ravel()
        Xd = np.ascontiguousarray(P.T.toarray() * _scopen.scale_of(c, 0.0, 0.5)[None, :])
        rng = np.random.default_rng(0)
        W, H = rng.random((CPU_PEAKS, K)), rng.random((K, N))
        t0 = time.perf_counter()
        _nmf._fit_coordinate_descent(Xd, W, H, tol=0.0, max_iter=3, l2_reg_W=1.0, l2_reg_H=1.0)
        res["cpu_dense_peaks"] = CPU_PEAKS
        res["cpu_dense_iteration_s"] = (time.perf_counter() - t0) / 3
        res["cpu_threads"] = len(os.sched_getaffinity(0))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
