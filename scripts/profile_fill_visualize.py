"""Device nearest-Gaussian search (pixie_b200.particle_filling.nearest_gaussian / init_filled_particles,
csrc/nearest.cu), the `particle_filling.visualize` step, on two scenes:
  shell_300k   a seeded 300k-Gaussian shell (radius 0.45, 2 % radial jitter) filled at n_grid 100 over [0.4, 1.6]^3; the
               queries are its filled particles
  1M_x_2M      1M Gaussians on the same shell against 2M queries drawn uniformly inside it
CUDA-event medians of: the build (Morton sort and tree, timed as a search with a single query), the search with all
queries, the query phase (their difference) and init_filled_particles end to end (search, the -1 check's host sync, SH
degree 3 gathers). Every device result is checked against the exact oracle on a sample of queries (all of them for the
shell with --oracle, whose CPU time is printed for context). Prints the card's name and power limit and one JSON line.

    python scripts/profile_fill_visualize.py [--repeats 10] [--oracle]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import fill_visualize_ref as R  # noqa: E402
from pixie_b200 import particle_filling as PF  # noqa: E402


def shell(n, seed):
    rng = np.random.default_rng(seed)
    v = rng.standard_normal((n, 3))
    pos = 1.0 + 0.45 * (1 + 0.02 * rng.standard_normal((n, 1))) * v / np.linalg.norm(v, axis=1, keepdims=True)
    s = rng.uniform(0.004, 0.012, (n, 3))
    cov = np.zeros((n, 6))
    cov[:, 0], cov[:, 3], cov[:, 5] = s[:, 0] ** 2, s[:, 1] ** 2, s[:, 2] ** 2
    return pos.astype(np.float32), rng.uniform(0.3, 1.0, (n, 1)).astype(np.float32), cov.astype(np.float32)


def timed(fn, repeats):
    fn()                                                           # warm-up: module load, allocator pool, cub temp sizes
    ms = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms))


def brute_sample(pos, q, got, k, seed=0):
    """The reference's loop on k sampled queries: (float32 d, lowest index) argmin; returns the number of mismatches."""
    idx = np.random.default_rng(seed).choice(len(q), min(k, len(q)), replace=False)
    bad = 0
    for i in idx:
        d = R.nearest_dist_f32(q[i], pos)
        d = np.where(d < np.float32(1e10), d, np.inf)
        bad += int(np.argmin(d) != got[i])
    return bad


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--oracle", action="store_true", help="check every shell query against the CPU oracle and time it")
    a = ap.parse_args()
    dev = "cuda:0"
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    out = {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": smi.stdout.strip(), "runs": []}
    print(f"card: {out['gpu']}  (name, power limit: {out['nvidia_smi']})", file=sys.stderr)

    pos, opacity, cov = shell(300_000, 0)
    p, o, c = (torch.from_numpy(x).to(dev) for x in (pos, opacity, cov))
    b = [0.4, 1.6, 0.4, 1.6, 0.4, 1.6]
    keep = torch.ones(len(pos), dtype=torch.bool, device=dev)
    for i in range(3):
        keep &= (p[:, i] > b[2 * i]) & (p[:, i] < b[2 * i + 1])
    _, density = PF.densify_grids(p[keep] - 0.4, o[keep], c[keep], 100, 0.012)
    d = density[density > 0].float()
    thr = dict(density_thres=float(torch.quantile(d[:1 << 24], 0.9)), search_thres=float(torch.quantile(d[:1 << 24], 0.5)))
    full = PF.fill_particles(p, o, c, 100, 4_000_000, 1.0, boundary=b, search_exclude_dir=2, ray_cast_dir=4, **thr)
    cases = [("shell_300k", pos, full[len(pos):].contiguous())]
    pos1m, _, _ = shell(1_000_000, 1)
    rng = np.random.default_rng(2)
    v = rng.standard_normal((2_000_000, 3))
    q2m = 1.0 + 0.44 * rng.uniform(0, 1, (2_000_000, 1)) ** (1 / 3) * v / np.linalg.norm(v, axis=1, keepdims=True)
    cases.append(("1M_x_2M", pos1m, torch.from_numpy(q2m.astype(np.float32)).to(dev)))

    for name, gpos, q in cases:
        gp = torch.from_numpy(gpos).to(dev)
        n, m = len(gpos), int(q.shape[0])
        shs = torch.randn(n, 16, 3, device=dev)
        op = torch.rand(n, 1, device=dev)
        cv = torch.rand(n, 6, device=dev)
        got = PF.nearest_gaussian(gp, q)
        again = PF.nearest_gaussian(gp, q)
        qh = q.cpu().numpy()
        got_h = got.cpu().numpy()
        r = {"case": name, "gaussians": n, "queries": m, "bit_identical_repeat": bool(torch.equal(got, again)),
             "no_neighbour": int((got < 0).sum())}
        r["brute_mismatches_of_200"] = brute_sample(gpos, qh, got_h, 200)
        build = timed(lambda: PF.nearest_gaussian(gp, q[:1]), a.repeats)
        search = timed(lambda: PF.nearest_gaussian(gp, q), a.repeats)
        r.update(build_ms=build, search_ms=search, query_ms=search - build,
                 init_filled_particles_ms=timed(lambda: PF.init_filled_particles(gp, shs, cv, op, q), a.repeats),
                 pairs_brute_force=float(n) * m)
        if a.oracle and name == "shell_300k":
            t0 = time.perf_counter()
            want = R.nearest_index(gpos, qh)
            r["cpu_oracle_s"] = time.perf_counter() - t0
            r["oracle_mismatches"] = int((want != got_h).sum())
        out["runs"].append(r)
        print(r, file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
