"""Micro-benchmark of the four SpMM entry points on a slice of the bench matrix: A·B on the CSR arrays
(mub_spmm_csr_*) and Aᵀ·B on the transposed pairs panels (mub_spmm_csrp_*), fp32 and half operand, P = 32, 64, 128.
Every product runs twice on the same arrays: flagged sorted (the fp32 entry points mub_spmm_csr_f32 and
mub_spmm_csrp_f32 then run the tiled kernel, the half-operand ones the row-warp kernel either way) and flagged
unsorted (the row-warp kernel).  CUDA events around `reps` passes after `warmup` passes; the digest of each output
lets two library builds
(MUON_B200_LIB) be compared bit for bit, and the largest relative difference between the two runs is printed.
    python profiles/bench_spmm.py [cells] [peaks] [reps] [P ...]"""
import hashlib
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from muon_b200 import _device  # noqa: E402
from muon_b200._synth import generate_device, make_tables  # noqa: E402

n = int(sys.argv[1]) if len(sys.argv) > 1 else 100_000
d = int(sys.argv[2]) if len(sys.argv) > 2 else 200_000
reps = int(sys.argv[3]) if len(sys.argv) > 3 else 10
widths = [int(p) for p in sys.argv[4:]] or [32, 64, 128]
warmup = 3
A = _device.tfidf_csr(generate_device(n, d, 0.03, tables=make_tables(d, 0.03, 64, 1)))
g = torch.Generator(device="cuda").manual_seed(0)


def schedules(M):
    """(name, matrix) flagged sorted and unsorted, on the same arrays"""
    if isinstance(M, _device.DevicePairs):
        unsorted = _device.DevicePairs(M.indptr, M.pairs, M.shape, sorted_indices=False)
    else:
        unsorted = _device.DeviceCSR(M.indptr, M.indices, M.data, M.shape, sorted_indices=False)
    return (("sorted", M), ("unsorted", unsorted)) if M.sorted_indices else (("unsorted", unsorted),)


def csr_pass(M, B):
    return _device.spmm(M, B, dynamic=False)


def pairs_pass(panels, B):
    out = torch.empty((d, B.shape[1]), dtype=torch.float32, device=B.device)
    for i, (r0, r1, T) in enumerate(panels):
        _device.spmm(T, B[r0:r1], out=out, accumulate=i > 0, dynamic=True)
    return out


print(f"n={n} d={d} nnz={A.nnz} reps={reps} {torch.cuda.get_device_name()}")
for P in widths:
    At = A.transpose_panels(P)
    variants = {"csr": [(s, (lambda B, M=M: csr_pass(M, B))) for s, M in schedules(A)]}
    per_panel = [schedules(T) for _, _, T in At.panels]
    variants["csrp"] = [(per_panel[0][j][0],
                         (lambda B, j=j: pairs_pass([(r0, r1, per_panel[i][j][1])
                                                     for i, (r0, r1, _) in enumerate(At.panels)], B)))
                        for j in range(len(per_panel[0]))]
    for name, rows in (("csr", d), ("csrp", n)):
        B32 = torch.randn((rows, P), generator=g, device="cuda") / 30.0
        for dtype, B in (("f32", B32), ("h16", _device.to_half_scaled(B32))):
            outs = {}
            for sched, run in variants[name]:
                for _ in range(warmup):
                    C = run(B)
                torch.cuda.synchronize()
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
                ev[0].record()
                for _ in range(reps):
                    C = run(B)
                ev[1].record()
                torch.cuda.synchronize()
                ms = ev[0].elapsed_time(ev[1]) / reps
                gb = (8 * A.nnz + B.element_size() * P * (n + d)) / 1e9
                digest = hashlib.sha256(C.cpu().numpy().tobytes()).hexdigest()[:16]
                outs[sched] = C
                print(f"mub_spmm_{name}_{dtype} P={P:3d} {sched:8s}: {ms:8.3f} ms  {gb / ms * 1e3:5.0f} GB/s algorithmic  "
                      f"{ms * 1e9 / A.nnz:5.1f} ps/nnz  digest {digest}")
            if len(outs) == 2:
                diff = ((outs["sorted"] - outs["unsorted"]).abs().max() / outs["unsorted"].abs().max()).item()
                print(f"mub_spmm_{name}_{dtype} P={P:3d} max |sorted - unsorted| / max |unsorted| = {diff:.3g}")
