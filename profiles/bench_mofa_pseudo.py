"""mu.tl.mofa on one bernoulli view kept sparse (csrc/mofa_lowrank.cu): the benchmark generator's 500k x 200k matrix,
binarized on the device, k=30, 5 iterations, one GPU.  Dense pseudo-data of that view would need 1.2 TB.

    python profiles/bench_mofa_pseudo.py [--cells 500000] [--peaks 200000] [--iters 5] [--k 30]

Prints one JSON line: ms per iteration, CUDA-event ms per entry point, the low-rank sweeps' FLOP/s (2 K flops per
element per contraction: zeta = Z W^T is one, g(zeta) C the other) against the 67 TFLOP/s FP32 data-sheet figure of
an H100 SXM, torch.cuda.max_memory_allocated(), and the card's name, power limit and SM clock."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from muon_b200 import _lib  # noqa: E402
from muon_b200._mofa import run_mofa_device  # noqa: E402
from muon_b200._synth import generate_device, make_tables  # noqa: E402

FP32_PEAK = 67e12

ap = argparse.ArgumentParser()
ap.add_argument("--cells", type=int, default=500_000)
ap.add_argument("--peaks", type=int, default=200_000)
ap.add_argument("--density", type=float, default=0.03)
ap.add_argument("--iters", type=int, default=5)
ap.add_argument("--k", type=int, default=30)
args = ap.parse_args()

n, D, K = args.cells, args.peaks, args.k
A = generate_device(n, D, args.density, tables=make_tables(D, args.density, 64, 1), row0=0, n_total=n)
A.data.fill_(1.0)                                         # binarized: a bernoulli view
Z0 = torch.from_numpy(np.random.RandomState(1).normal(size=(n, K)))
torch.cuda.synchronize()

run_mofa_device([A], K, 1, n, Z0, check_convergence=False, likelihoods=["bernoulli"])    # warm-up, builds A^T panels
torch.cuda.synchronize()
torch.cuda.reset_peak_memory_stats()
_lib.PROFILE = {}
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
res = run_mofa_device([A], K, args.iters, n, Z0, check_convergence=False, likelihoods=["bernoulli"])
e1.record()
torch.cuda.synchronize()
prof, _lib.PROFILE = _lib.PROFILE, None
ms = e0.elapsed_time(e1)
kern = {k: float(np.sum([a.elapsed_time(b) for a, b in v])) for k, v in prof.items()}
calls = {k: len(v) for k, v in prof.items()}
# per iteration one column sweep (P: two contractions), one row sweep with B (Q: two) and one without (ln p: one);
# one more column sweep after the last iteration (variance explained)
el = float(n) * D
flops = {"mub_mofa_lowrank_cols_f32": calls.get("mub_mofa_lowrank_cols_f32", 0) * 4 * K * el,
         "mub_mofa_lowrank_rows_f32": (args.iters * 4 + args.iters * 2) * K * el}
rate = {k: f / (kern[k] * 1e-3) for k, f in flops.items() if kern.get(k)}
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip().splitlines()
print(json.dumps({
    "workload": f"mofa, one bernoulli view {n}x{D} ({A.nnz} stored entries), k={K}, {args.iters} iterations",
    "ms_total": ms, "ms_per_iteration": ms / args.iters, "kernel_ms": kern, "kernel_calls": calls,
    "lowrank_TFLOPs": {k: v / 1e12 for k, v in rate.items()},
    "lowrank_share_of_fp32_peak": {k: v / FP32_PEAK for k, v in rate.items()},
    "lowrank_flops_per_iteration": 10 * K * el, "max_memory_allocated_GiB": torch.cuda.max_memory_allocated() / 2**30,
    "elbo": res["elbo"], "gpu": gpu[0] if gpu else None}))
