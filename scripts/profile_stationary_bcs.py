"""Device DBSCAN + cluster statistics (pixie_b200.material_transfer, csrc/cluster.cu) against scikit-learn's DBSCAN on the host,
for the clustering step of handle_stationary_clusters (eps 0.03, min_samples 8) at 100k / 355k (the size of the authors' tree
scene) / 1M stationary particles. The cloud is a thin surface shell of Gaussian centres plus dense clumps (hundreds to
thousands of neighbours per point) and sparse noise, in the simulation frame around (1, 1, 1). Prints one JSON line.

    python scripts/profile_stationary_bcs.py [--sizes 100000,355000,1000000] [--repeats 5] [--no-sklearn]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pixie_b200 import material_transfer as MT  # noqa: E402


def cloud(n, seed=0):
    rng = np.random.default_rng(seed)
    n_shell, n_clump = int(n * 0.8), int(n * 0.18)
    d = rng.standard_normal((n_shell, 3))
    shell = d / np.linalg.norm(d, axis=1, keepdims=True) * np.array([0.35, 0.35, 0.6]) + rng.normal(0, 0.003, size=(n_shell, 3))
    centres = rng.uniform(-0.4, 0.4, size=(max(1, n_clump // 2000), 3))
    clumps = centres[rng.integers(0, len(centres), n_clump)] + rng.normal(0, 0.02, size=(n_clump, 3))
    noise = rng.uniform(-0.7, 0.7, size=(n - n_shell - n_clump, 3))
    return (np.concatenate([shell, clumps, noise]) + 1.0).astype(np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="100000,355000,1000000")
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--no-sklearn", action="store_true")
    a = ap.parse_args()
    dev = "cuda:0"
    out = {"eps": 0.03, "min_samples": 8, "gpu": torch.cuda.get_device_name(0), "host_threads": os.cpu_count(), "runs": []}
    for n in [int(s) for s in a.sizes.split(",")]:
        x = cloud(n)
        xd = torch.from_numpy(x).to(dev)
        labels, index, k = MT._dbscan(xd, 0.03, 8, None, 6)                 # warm-up (module load, allocator)
        times = []
        for _ in range(a.repeats):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            labels, index, k = MT._dbscan(xd, 0.03, 8, None, 6)
            sizes, lo, hi = MT._cluster_stats(xd, index, labels, k)
            times.append(time.perf_counter() - t0)
        r = {"n": n, "clusters": int(k), "noise": int((labels == -1).sum().item()), "device_ms_median": 1e3 * float(np.median(times)),
             "device_ms_min": 1e3 * float(np.min(times))}
        start = torch.cuda.Event(enable_timing=True)
        end = torch.cuda.Event(enable_timing=True)
        start.record()
        MT._dbscan(xd, 0.03, 8, None, 6)
        end.record()
        torch.cuda.synchronize()
        r["dbscan_event_ms"] = start.elapsed_time(end)
        if not a.no_sklearn:
            from sklearn.cluster import DBSCAN
            t0 = time.perf_counter()
            ref = DBSCAN(eps=0.03, min_samples=8, n_jobs=-1).fit_predict(x)
            r["sklearn_s"] = time.perf_counter() - t0
            r["labels_equal"] = bool(np.array_equal(ref, labels.cpu().numpy()))
        out["runs"].append(r)
        print(r, file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
