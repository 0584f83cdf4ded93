"""Exact kNN, tensor-core (wgmma TF32 candidates + fp32 re-rank) vs SIMT kernel.  python profiles/bench_knn.py [n] [d] [k]"""
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from muon_b200 import _device  # noqa: E402

n = int(sys.argv[1]) if len(sys.argv) > 1 else 100_000
d = int(sys.argv[2]) if len(sys.argv) > 2 else 50
k = int(sys.argv[3]) if len(sys.argv) > 3 else 201
g = torch.Generator(device="cuda").manual_seed(0)
X = torch.randn(n, d, generator=g, device="cuda") + 3 * torch.randn(30, d, generator=g, device="cuda")[
    torch.randint(0, 30, (n,), generator=g, device="cuda")]
X = torch.nn.functional.normalize(X).contiguous()
out = {"n": n, "d": d, "k": k}
ref = None
for algo in (["tc"] if os.environ.get("KNN_TC_ONLY") else ["tc", "simt"]):
    idx, dist = _device.knn_l2(X, k, algo=algo)          # warm-up
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    idx, dist = _device.knn_l2(X, k, algo=algo)
    b.record()
    torch.cuda.synchronize()
    out[algo + "_ms"] = a.elapsed_time(b)
    if ref is None:
        ref = idx
    else:
        out["identical"] = bool(torch.equal(ref, idx))
out["pairs_per_s_tc"] = n * n / (out["tc_ms"] * 1e-3)
print(json.dumps(out))
