"""Device particle filling (pixie_b200.particle_filling, csrc/particle_fill.cu) on hollow shell scenes of 300k and 1M Gaussians
in both config shapes the reference uses: n_grid 50 over the metal boundary (fruit / metal / metal_crates / soda_cans) and
n_grid 100 over a 1.2 box. CUDA-event times of the density splat (densify_grids), of classification + fill (fill_grids:
dense counts, interior classification, scans, one host sync for the totals, emission) and of fill_particles end to end
(crop, both steps, concatenation). Prints the card's name and power limit and one JSON line.

    python scripts/profile_filling.py [--sizes 300000,1000000] [--repeats 10]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pixie_b200 import particle_filling as PF  # noqa: E402

CONFIGS = {
    "metal_n50": dict(center=(1.16, 1.0, 1.0), radius=0.22, std=0.004, grid_n=50, boundary=[0.86, 1.46, 0.7, 1.3, 0.7, 1.3],
                      search_exclude_dir=0, ray_cast_dir=1),
    "box1.2_n100": dict(center=(1.0, 1.0, 1.0), radius=0.45, std=0.008, grid_n=100, boundary=[0.4, 1.6, 0.4, 1.6, 0.4, 1.6],
                        search_exclude_dir=2, ray_cast_dir=4),
}


def shell(n, center, radius, std, seed=0):
    """Gaussians on a sphere (radius jittered by 2 %) with random anisotropic covariances of scale `std`."""
    rng = np.random.default_rng(seed)
    v = rng.standard_normal((n, 3))
    pos = np.asarray(center) + radius * (1 + 0.02 * rng.standard_normal((n, 1))) * v / np.linalg.norm(v, axis=1, keepdims=True)
    s = rng.uniform(0.5, 1.5, size=(n, 3)) * std
    Q, _ = np.linalg.qr(rng.standard_normal((n, 3, 3)))
    m = Q @ (s[:, :, None] ** 2 * np.eye(3)) @ Q.transpose(0, 2, 1)
    cov = np.stack([m[:, 0, 0], m[:, 0, 1], m[:, 0, 2], m[:, 1, 1], m[:, 1, 2], m[:, 2, 2]], axis=1)
    return pos.astype(np.float32), rng.uniform(0.3, 1.0, size=(n, 1)).astype(np.float32), cov.astype(np.float32)


def timed(fn, repeats):
    fn()                                                           # warm-up: module load, allocator, cub temp sizes
    ms = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms)), float(np.min(ms))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="300000,1000000")
    ap.add_argument("--repeats", type=int, default=10)
    a = ap.parse_args()
    dev = "cuda:0"
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    out = {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": smi.stdout.strip(), "runs": []}
    print(f"card: {out['gpu']}  (name, power limit: {out['nvidia_smi']})", file=sys.stderr)
    for n in [int(s) for s in a.sizes.split(",")]:
        for name, cfg in CONFIGS.items():
            k = dict(cfg)
            pos, opacity, cov = shell(n, k.pop("center"), k.pop("radius"), k.pop("std"))
            p, o, c = (torch.from_numpy(x).to(dev) for x in (pos, opacity, cov))
            b, g = k["boundary"], k["grid_n"]
            dx = max(b[1] - b[0], b[3] - b[2], b[5] - b[4]) / g
            keep = torch.ones(n, dtype=torch.bool, device=dev)
            for i in range(3):
                keep &= (p[:, i] > b[2 * i]) & (p[:, i] < b[2 * i + 1])
            pc, oc, cc = p[keep] - torch.tensor([b[0], b[2], b[4]], device=dev), o[keep], c[keep]
            count, density = PF.densify_grids(pc, oc, cc, g, dx)
            # thresholds at fixed quantiles of this scene's densities (the configs' absolute values assume trained opacities)
            d = density[density > 0]
            thr = dict(density_thres=float(torch.quantile(d[:1 << 24].float(), 0.9)), search_thres=float(torch.quantile(d[:1 << 24].float(), 0.5)))
            splat = timed(lambda: PF.densify_grids(pc, oc, cc, g, dx), a.repeats)

            def fill():
                cnt = count.clone()
                return PF.fill_grids(cnt, density, dx, 4_000_000, max_particles_per_cell=1, search_exclude_dir=k["search_exclude_dir"],
                                     ray_cast_dir=k["ray_cast_dir"], origin=(b[0], b[2], b[4]), **thr)
            new, n_dense = fill()
            classify_fill = timed(fill, a.repeats)
            total = timed(lambda: PF.fill_particles(p, o, c, g, 4_000_000, 1.0, max_particles_per_cell=1, boundary=b,
                                                    search_exclude_dir=k["search_exclude_dir"], ray_cast_dir=k["ray_cast_dir"], **thr), a.repeats)
            r = {"config": name, "gaussians": n, "in_boundary": int(keep.sum()), "grid_n": g, "n_dense": n_dense,
                 "n_interior": int(new.shape[0]) - n_dense, "splat_ms": splat[0], "classify_fill_ms": classify_fill[0],
                 "fill_particles_ms": total[0], "splat_ms_min": splat[1], "classify_fill_ms_min": classify_fill[1],
                 "fill_particles_ms_min": total[1]}
            out["runs"].append(r)
            print(r, file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
