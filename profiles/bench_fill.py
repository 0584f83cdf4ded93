"""Times the transposed row panels of configs[1] alone: TransposedPanels(tfidf(A), 64) on the benchmark generator's
500k x 200k matrix at 3 %, 2 untimed and 3 timed builds, CUDA events per C-ABI call.  ``--no-counts`` builds them
from the same TF-IDF values without the entry counts of the reduce pass, so the panels take the counting pass and the
atomic-cursor fill.  MUON_B200_LIB selects another build of the library (A/B).  Prints one JSON line.

    python profiles/bench_fill.py [--no-counts]
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from muon_b200 import _device, _lib  # noqa: E402
from muon_b200._synth import generate_device, make_tables  # noqa: E402


def main(n=500_000, d=200_000, density=0.03, topics=64, seed=1, counts=True):
    A = generate_device(n, d, density, tables=make_tables(d, density, topics, seed), row0=0, n_total=n)
    X = _device.tfidf_csr(A)
    del A
    if not counts:
        X = X.with_data(X.data)          # same arrays, no entry counts
    for _ in range(2):
        _device.TransposedPanels(X, 64)
    torch.cuda.synchronize()
    runs = []
    for _ in range(3):
        _lib.PROFILE = {}
        t0 = time.perf_counter()
        T = _device.TransposedPanels(X, 64)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        prof, _lib.PROFILE = _lib.PROFILE, None
        ms = {k: round(sum(a.elapsed_time(b) for a, b in v), 2) for k, v in prof.items()}
        calls = {f"{k}_calls": len(v) for k, v in prof.items()}
        runs.append({"wall_ms": round(1e3 * wall, 1), "tiled_fill": T.tiled_fill, "counts_reused": T.counts_reused,
                     "panels": len(T.panels), **ms, **calls})
        del T
    print(json.dumps({"lib": _lib.LIB_PATH, "gpu": torch.cuda.get_device_name(), "counts": counts, "runs": runs}))


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--no-counts", action="store_true", help="panels without the reduce pass's entry counts")
    main(counts=not ap.parse_args().no_counts)
