"""Times the device rasterizer (pixie_b200.gs_render) per phase and end to end, against the reference's rasterizer binary
(oracle/_ref/gs_rasterizer, built by oracle/build_gs_rasterizer_ref.py) on the same inputs, alternating the two.

    python scripts/profile_render.py [--reps 20] [--out results.json]

Scenes: 300k and 1M seeded Gaussians (anisotropic covariances, degree-3 SH), at 800x800 and 1920x1080. Per phase: CUDA
events inside one call (preprocess + SH, scan + keys including the host sync for the pair count, sort, ranges, blend);
end to end: CUDA events around whole calls, medians over --reps alternating repetitions. Prints the card's name and power
limit, read in the same run. With --out, also writes the table as JSON to that path.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from pixie_b200 import gs_render as GR  # noqa: E402
from test_gs_render import _ref_module, look_at_camera, ref_render, seeded_scene  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the results as JSON to this path")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "profile_render needs a CUDA device"
    dev = "cuda:0"
    mod = _ref_module()
    info = card()
    print(f"[profile_render] {info}")
    rows = []
    for n in (300_000, 1_000_000):
        for W, H in ((800, 800), (1920, 1080)):
            cam = look_at_camera(W, H, radius=3.0)
            pos, cov, op, shs, _ = seeded_scene(n, seed=n + W, dev=dev, near_cam=cam)
            ours = lambda: GR.rasterize(pos, cov, op, cam, [0, 0, 0], shs=shs, sh_degree=3)  # noqa: E731
            ref = lambda: ref_render(mod, pos, cov, op, cam, [0, 0, 0], shs=shs, deg=3)      # noqa: E731
            for _ in range(3):
                ours(), ref()
            t_ours, t_ref, phases = [], [], []
            for _ in range(args.reps):
                t_ours.append(timed(ours))
                t_ref.append(timed(ref))
                ph = [0.0] * 5
                _, _, pairs = GR._rasterize(pos, cov, op, cam, [0, 0, 0], shs=shs, sh_degree=3, phase_ms=ph)
                phases.append(ph)
            ph = np.median(np.array(phases), axis=0)
            img, _ = ours()
            img_r, _ = ref()
            row = {"n": n, "W": W, "H": H, "pairs": pairs, "ours_ms": float(np.median(t_ours)), "ref_ms": float(np.median(t_ref)),
                   "ours_ms_min": float(np.min(t_ours)), "ref_ms_min": float(np.min(t_ref)),
                   "phases_ms": dict(zip(("preprocess_sh", "scan_keys", "sort", "ranges", "blend"), map(float, ph))),
                   "max_abs_diff": float((img - img_r).abs().max())}
            rows.append(row)
            print(f"[profile_render] n={n} {W}x{H} pairs={pairs}: ours {row['ours_ms']:.3f} ms, reference {row['ref_ms']:.3f} ms; "
                  + ", ".join(f"{k} {v:.3f}" for k, v in row["phases_ms"].items()) + f"; max|diff| {row['max_abs_diff']:.2e}")
            del pos, cov, op, shs
            torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"card": info, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
