"""mu.tl.ica on planted non-Gaussian sources, one H100.

    python profiles/bench_ica.py [cells=1000000] [features=50] [--sklearn ROWS]

X is cells x features float32: 10 planted sources (Laplace, uniform, bimodal) in the leading principal subspace and
weak Gaussian noise in the rest, mixed by a random matrix (tests/ica_cases.py::planted), NOT timed.  One warm-up
call, then two timed calls bracketed by device synchronisation:

  * ``full``: default arguments (n_components = features, logcosh, parallel, tol 1e-4, max_iter 200);
  * ``k10``: n_components=10, which converges in a few iterations.

For each: wall time, n_iter, and the summed CUDA-event time of every C-ABI call (moments, project, step, sources);
the step kernel is also reported per iteration, with its float64 rate (4 k^2 n per parallel step) and the bytes of
X1 it reads against the H100 SXM's 3.35 TB/s HBM3 peak.  With ``--sklearn ROWS`` it also times sklearn's FastICA on
the first ROWS cells with the same arguments on the host.  Prints one JSON line with the card and its power limit.
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
import muon_b200 as mu  # noqa: E402
from muon_b200 import _lib  # noqa: E402
from ica_cases import planted  # noqa: E402

args = [a for a in sys.argv[1:] if not a.startswith("--")]
sk_rows = None
if "--sklearn" in sys.argv:
    sk_rows = int(sys.argv[sys.argv.index("--sklearn") + 1])
    args = [a for a in args if a != str(sk_rows)]
N = int(args[0]) if len(args) > 0 else 1_000_000
P = int(args[1]) if len(args) > 1 else 50

X, _ = planted(N, P, 7, np.float32, m=10)


def run(**kw):
    ad = mu.SimpleAnnData(np.zeros((N, 1), dtype=np.float32))
    ad.obsm["X_pca"] = X
    torch.cuda.synchronize()
    _lib.PROFILE = {}
    t0 = time.perf_counter()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        _, info = mu.tl.ica(ad, random_state=0, return_info=True, **kw)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    prof, _lib.PROFILE = _lib.PROFILE, None
    ms = {name: sum(a.elapsed_time(b) for a, b in ev) for name, ev in prof.items()}
    steps = len(prof.get("mub_ica_step_f64", []))
    k = info["components"].shape[0]
    step_ms = ms.get("mub_ica_step_f64", 0.0) / max(steps, 1)
    return {"wall_s": round(wall, 3), "n_iter": info["n_iter"], "k": k,
            "kernel_ms": {n.replace("mub_ica_", ""): round(v, 2) for n, v in ms.items()},
            "step_ms": round(step_ms, 3), "step_gflops": round(4 * k * k * N / step_ms / 1e6, 1),
            "step_x1_tb_s": round(8 * k * N / step_ms / 1e9, 3)}


run(n_components=10)                      # warm-up
out = {"bench": "ica", "cells": N, "features": P, "dtype": "float32", "full": run(), "k10": run(n_components=10)}

if sk_rows:
    from sklearn.decomposition import FastICA
    Xs = X[:sk_rows]
    for name, kw in (("full", {}), ("k10", {"n_components": 10})):
        t0 = time.perf_counter()
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            est = FastICA(random_state=0, **kw)
            est.fit_transform(Xs)
        out[f"sklearn_{name}"] = {"rows": sk_rows, "wall_s": round(time.perf_counter() - t0, 3),
                                  "n_iter": int(est.n_iter_), "host_cpus": os.cpu_count()}

q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                   text=True).stdout.strip().splitlines()
out["gpu"] = q[0] if q else torch.cuda.get_device_name(0)
print(json.dumps(out))
