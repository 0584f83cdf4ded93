"""mu.tl.mofa with groups on device-resident views: the RNA 500k x 30k (7 %) and ATAC 500k x 200k (3 %) views of
bench.py's MOFA leg, made on the device (generate_device, then tfidf_csr), k=30, 3 groups.

    python profiles/bench_mofa_groups.py [--cells 500000] [--iters 5] [--k 30] [--groups 3] [--host]

3 groups, not 4: mub_mofa_update_z_f32 holds the statistics of every cell class (group x set of views, 2^2 per group
here) in at most 96 KB of shared memory, (K^2 + 2K) * 8 B each: 4 groups at k=30 would need 120 KB and are refused.

Layouts:
  (a) contiguous groups: every (view, group) block is a slice of its view, nothing is copied;
  (b) interleaved groups: every block is gathered (csrc/select.cu), one extra copy of each view (8 B per non-zero).
      That does not fit at 500k cells on an 80 GB card, so (b) runs at the largest cell count that fits, computed
      from the free memory and lowered by 10 % on an out-of-memory error (at most three tries); the count is printed.
For each layout: the marshal time (selection, entry counts, transposed panels and moments: mofa() up to the first
iteration), the selection kernels' CUDA-event time and GB/s against the H100 SXM's 3.35 TB/s data-sheet HBM3 figure,
ms per iteration, torch.cuda.max_memory_allocated(), and the same data fitted as one group.  --host also fits the
host-matrix grouped path of layout (b) when the host has room for it.  The card's name, power limit and SM clock are
read in the same run.  Prints one JSON line per measurement."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import muon_b200 as mu  # noqa: E402
from muon_b200 import _device, _lib, _mofa  # noqa: E402
from muon_b200._synth import generate_device  # noqa: E402

HBM_PEAK = 3.35e12
VIEWS = (("rna", 30_000, 0.07, 2), ("atac", 200_000, 0.03, 1))

ap = argparse.ArgumentParser()
ap.add_argument("--cells", type=int, default=500_000)
ap.add_argument("--iters", type=int, default=5)
ap.add_argument("--k", type=int, default=30)
ap.add_argument("--groups", type=int, default=3)
ap.add_argument("--host", action="store_true")
args = ap.parse_args()


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else None


# ---- instrumentation: wall time of the selections and of MofaDevice.__init__, per-iteration time -------------------
T = {}
sel_bytes = [0]
_orig_select, _orig_init, _orig_step = _device.csr_select, _mofa.MofaDevice.__init__, _mofa.MofaDevice.step


def timed_select(A, rows=None, col_mask=None):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = _orig_select(A, rows, col_mask)
    torch.cuda.synchronize()
    T["select_s"] = T.get("select_s", 0.0) + time.perf_counter() - t0
    if out.data.untyped_storage().data_ptr() != A.data.untyped_storage().data_ptr():
        # no column mask here: the count reads 2 indptr words per row; the fill reads and writes 8 B per entry
        sel_bytes[0] += 16 * out.shape[0] * 2 + 16 * out.nnz
    return out


def timed_init(self, *a, **k):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    _orig_init(self, *a, **k)
    torch.cuda.synchronize()
    T["model_init_s"] = time.perf_counter() - t0
    T["t_init_end"] = time.perf_counter()


def timed_step(self):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    _orig_step(self)
    torch.cuda.synchronize()
    T.setdefault("steps", []).append(time.perf_counter() - t0)


_device.csr_select = timed_select
_mofa.MofaDevice.__init__ = timed_init
_mofa.MofaDevice.step = timed_step


def make_views(n):
    out = {}
    for name, D, dens, seed in VIEWS:
        out[name] = _device.tfidf_csr(generate_device(n, D, dens, seed=seed), inplace_values=True)
    torch.cuda.synchronize()
    return out


def fit(views, groups, label, n):
    T.clear()
    sel_bytes[0] = 0
    obs = [f"c{i}" for i in range(n)]
    md = mu.SimpleMuData({m: mu.SimpleAnnData(X, obs=obs) for m, X in views.items()})
    if groups is not None:
        md.obs["grp"] = groups
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    _lib.PROFILE = {}
    t0 = time.perf_counter()
    mu.tl.mofa(md, use_var=None, likelihoods="gaussian", n_factors=args.k, n_iterations=args.iters,
               convergence_mode="slow", groups_label=None if groups is None else "grp", seed=1)
    torch.cuda.synchronize()
    prof, _lib.PROFILE = _lib.PROFILE, None
    sel_ms = float(sum(a.elapsed_time(b) for name in ("mub_csr_select_count", "mub_csr_select_fill_f32")
                       for a, b in prof.get(name, [])))
    counts_ms = float(sum(a.elapsed_time(b) for a, b in prof.get("mub_tfidf_reduce_tiled_f32", [])))
    steps = T.get("steps", [])
    res = {"layout": label, "cells": n, "groups": 1 if groups is None else len(set(groups.tolist())),
           "k": args.k, "iterations": len(steps),
           "stored_entries": {m: X.nnz for m, X in views.items()},
           "blocks": md.uns["mofa"]["_b200"]["blocks"],
           "marshal_s": T.get("t_init_end", t0) - t0, "selection_wall_s": T.get("select_s", 0.0),
           "model_init_s (panels, moments)": T.get("model_init_s"),
           "select_kernel_ms": sel_ms, "count_pass_ms": counts_ms,
           "select_GBps": sel_bytes[0] / (sel_ms * 1e-3) / 1e9 if sel_ms else None,
           "select_share_of_hbm_peak": sel_bytes[0] / (sel_ms * 1e-3) / HBM_PEAK if sel_ms else None,
           "ms_per_iteration": 1e3 * float(np.mean(steps[1:] if len(steps) > 1 else steps)) if steps else None,
           "ms_per_iteration_all": [1e3 * s for s in steps],
           "max_memory_allocated_GiB": torch.cuda.max_memory_allocated() / 2**30,
           "elbo_last": md.uns["mofa"]["_b200"]["elbo"][-1], "gpu": gpu_info()}
    print(json.dumps(res), flush=True)
    del md
    torch.cuda.empty_cache()
    return res


n, G = args.cells, args.groups
print(json.dumps({"gpu": gpu_info(), "torch": torch.__version__}), flush=True)

# (a) contiguous groups at full size, and the one-group fit of the same data
views = make_views(n)
contiguous = np.repeat(np.array([f"g{g}" for g in range(G)]), -(-n // G))[:n]
fit(views, contiguous, "(a) contiguous groups", n)
fit(views, None, "one group", n)
per_cell = sum(X.nnz for X in views.values()) / n * 8          # bytes of indices + values per cell
del views
torch.cuda.empty_cache()

# (b) interleaved groups: the views, one gathered copy and the transposed panels (8 B per entry each)
free = torch.cuda.mem_get_info()[0]
nb = min(n, int(0.92 * free / (3 * per_cell + 4096)) // 1000 * 1000)
for attempt in range(3):
    try:
        views = make_views(nb)
        interleaved = np.array([f"g{g}" for g in range(G)])[np.arange(nb) % G]
        fit(views, interleaved, "(b) interleaved groups", nb)
        fit(views, None, "one group", nb)
        break
    except torch.cuda.OutOfMemoryError as e:
        print(json.dumps({"layout": "(b) interleaved groups", "cells": nb, "out_of_memory": str(e)[:200]}), flush=True)
        views = None
        _lib.PROFILE = None
        torch.cuda.empty_cache()
        nb = int(nb * 0.9) // 1000 * 1000

if args.host and views is not None:
    need = 6 * sum(X.nnz for X in views.values()) * 8
    avail = os.sysconf("SC_AVPHYS_PAGES") * os.sysconf("SC_PAGE_SIZE")
    if avail < need:
        print(json.dumps({"layout": "(b) host matrices", "skipped": f"needs about {need / 2**30:.0f} GiB of host memory, "
                          f"{avail / 2**30:.0f} GiB available"}), flush=True)
    else:
        host = {m: X.get() for m, X in views.items()}
        del views
        torch.cuda.empty_cache()
        fit(host, interleaved, "(b) host matrices, interleaved groups", nb)
