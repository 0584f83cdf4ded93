"""DSB at CITE-seq scale: ``mu.prot.pp.dsb`` on synthetic protein counts, timed per phase, against the per-cell
rate of the CPU mixture fits.

    python profiles/bench_dsb.py [--cells 1000000] [--proteins 200] [--empty 5000000] [--repeats 3]

Phases (``_lib.phase``: device-synchronised host clock): moments over the empty droplets (with their upload), the
fused per-cell scale+fit (with the cells' upload), the denoising regression and the download of the result; the
whole call is also timed with CUDA events, and what the phases leave out is the host-side droplet selection of
the reference's container branches.  The CPU baseline fits the
reference's two scikit-learn GaussianMixtures (plus their BICs) on 2,000 scaled cells, or, without sklearn,
``oracle.dsb_ref``'s vectorised numpy fits -- the ``cpu_baseline`` field says which.  Prints one JSON line.
"""
import argparse
import json
import os
import sys
import time
import warnings

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def cpu_rate(cells_scaled, random_state=0):
    """Seconds per cell of the reference's per-cell fits (preproc.py:189-198)."""
    try:
        from sklearn.mixture import GaussianMixture
    except ImportError:
        from oracle.dsb_ref import background_means
        t = time.perf_counter()
        background_means(cells_scaled, random_state=random_state)
        return (time.perf_counter() - t) / len(cells_scaled), "oracle.dsb_ref (numpy, float64)"
    tied = GaussianMixture(n_components=2, covariance_type="tied", init_params="random", random_state=random_state)
    full = GaussianMixture(n_components=2, covariance_type="full", init_params="random", random_state=random_state)
    t = time.perf_counter()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for row in cells_scaled:
            x = row[:, None]
            tied.fit(x)
            full.fit(x)
            tied.bic(x) < full.bic(x)
    return (time.perf_counter() - t) / len(cells_scaled), "sklearn GaussianMixture"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cells", type=int, default=1_000_000)
    ap.add_argument("--proteins", type=int, default=200)
    ap.add_argument("--empty", type=int, default=5_000_000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--cpu-sample", type=int, default=2000)
    a = ap.parse_args()

    import torch

    import muon_b200 as mu
    from muon_b200 import _lib
    from oracle.dsb_ref import scale, synth_citeseq

    if not torch.cuda.is_available():
        raise SystemExit("bench_dsb.py needs a GPU")
    t = time.perf_counter()
    cells, empty = synth_citeseq(a.cells, a.empty, a.proteins, seed=0)
    t_gen = time.perf_counter() - t
    E = mu.SimpleAnnData(empty, obs=[f"e{i}" for i in range(a.empty)])
    obs = [f"c{i}" for i in range(a.cells)]

    def once(phases):
        ad = mu.SimpleAnnData(cells, obs=obs)
        _lib.PHASES = phases
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            e0.record()
            mu.prot.pp.dsb(ad, E, random_state=0)
            e1.record()
        torch.cuda.synchronize()
        _lib.PHASES = None
        return e0.elapsed_time(e1) / 1e3

    once({})  # warm-up: module load, allocator, every shape of the timed calls
    walls, phases = [], []
    for _ in range(a.repeats):
        ph = {}
        walls.append(once(ph))
        phases.append(ph)

    idx = np.random.default_rng(1).choice(a.cells, min(a.cpu_sample, a.cells), replace=False)
    per_cell, baseline = cpu_rate(scale(cells[idx], empty[:200_000]))
    props = torch.cuda.get_device_properties(0)
    import subprocess
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"],
                               capture_output=True, text=True, timeout=20).stdout.strip().splitlines()[0]
    except Exception:
        power = "unknown"
    wall = float(np.median(walls))
    print(json.dumps({
        "workload": "dsb", "cells": a.cells, "proteins": a.proteins, "empty_droplets": a.empty,
        "empty_nnz": int(empty.nnz), "gpu": props.name, "power_limit": power,
        "wall_s_median": round(wall, 4), "wall_s_all": [round(w, 4) for w in walls],
        "phases_s_median": {k: round(float(np.median([p.get(k, 0.0) for p in phases])), 4) for k in phases[0]},
        "host_bookkeeping_s_median": round(wall - float(np.median([sum(p.values()) for p in phases])), 4),
        "cells_per_s": round(a.cells / wall, 1),
        "cpu_baseline": baseline, "cpu_s_per_cell": per_cell, "cpu_cells_per_s": round(1 / per_cell, 1),
        "speedup_vs_cpu_fits": round(per_cell * a.cells / wall, 1), "host_generate_s": round(t_gen, 1),
    }))


if __name__ == "__main__":
    main()
