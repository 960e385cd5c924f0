"""Profile of dataset-view rendering and scoring (pixie_b200.gs_dataset_render, pixie_b200.gs_metrics) on one GPU.

    python scripts/profile_gs_dataset_render.py [--views 200] [--size 800] [--gaussians 300000]

Builds a seeded Blender dataset (RGBA frames around the object) and checkpoint in a temporary directory, then prints one
JSON line: views/s of the whole command (decode, reads, draws, PNG encodes), the device time per view split into
preprocess, sort (scan + keys + sort + ranges) and blend (CUDA events), host time per view for image reads and PNG
encoding, the metric kernel's time per pair, the same views through the reference rasterizer binary in oracle/_ref/
(when built), and the card's name and power limit.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from pixie_b200 import gs_dataset_render as D  # noqa: E402
from pixie_b200 import gs_metrics as G  # noqa: E402
from pixie_b200 import gs_render as GR  # noqa: E402
from pixie_b200 import scene_files as SF  # noqa: E402
from gs_views_fixtures import reference_rasterizer, ref_render_scale_rot, write_blender, write_checkpoint  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=200)
    ap.add_argument("--size", type=int, default=800)
    ap.add_argument("--gaussians", type=int, default=300000)
    a = ap.parse_args()
    rng = np.random.default_rng(0)
    out = {"card": card(), "views": a.views, "size": a.size, "gaussians": a.gaussians}
    with tempfile.TemporaryDirectory() as tmp:
        src, model = os.path.join(tmp, "src"), os.path.join(tmp, "model")
        write_blender(src, rng, a.views, 0, a.size, a.size, alpha_values=[0, 64, 255])
        write_checkpoint(model, rng, a.gaussians, 16, iteration=30000, extent=0.5)
        with open(os.path.join(model, "cfg_args"), "w") as f:
            f.write(f"Namespace(sh_degree=3, source_path={src!r}, resolution=-1, white_background=False, eval=False)")
        args = D.get_combined_args(["-m", model, "-s", src, "--quiet", "--skip_test"])

        t0 = time.perf_counter()
        train, _ = D.read_scene(args)
        out["host_read_ms_per_view"] = (time.perf_counter() - t0) * 1e3 / a.views
        D.render_sets(args)                                   # warm-up: module loads, allocator, renderer buffers
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        D.render_sets(args)
        torch.cuda.synchronize()
        out["views_per_s"] = a.views / (time.perf_counter() - t0)

        g = SF.decode_checkpoint_ply_scale_rot(SF.checkpoint_path(model), 3, "cuda")
        bg = [0.0, 0.0, 0.0]
        phases = []
        cams = [D.loadCam(-1, info)[0] for info in train[:20]]
        for cam in cams:
            ms = [0.0] * 5
            GR._rasterize_scale_rot(g["pos"], g["scales"], g["rotations"], g["opacity"], cam, bg, g["shs"], 3, phase_ms=ms)
            phases.append(ms)
        p = np.mean(np.array(phases), 0)
        out["device_ms_per_view"] = {"preprocess": p[0], "sort": p[1] + p[2] + p[3], "blend": p[4], "total": float(p.sum())}

        imgs = [GR.rasterize_scale_rot(g["pos"], g["scales"], g["rotations"], g["opacity"], cam, bg, g["shs"], 3)[0] for cam in cams]
        q = [D.quantize(im).cpu().numpy() for im in imgs]
        t0 = time.perf_counter()
        for i, arr in enumerate(q):
            D.save_png(arr, os.path.join(tmp, f"{i}.png"))
        out["host_png_encode_ms_per_image"] = (time.perf_counter() - t0) * 1e3 / len(q)

        da = [torch.from_numpy(x).cuda() for x in q]
        db = [torch.from_numpy(np.ascontiguousarray(x[::-1])).cuda() for x in q]
        for x, y in zip(da, db):
            G.image_metrics(x, y)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        reps = 10
        for _ in range(reps):
            for x, y in zip(da, db):
                G.image_metrics(x, y)
        e1.record()
        e1.synchronize()
        out["metric_kernel_ms_per_pair"] = e0.elapsed_time(e1) / (reps * len(da))

        mod = reference_rasterizer()
        if mod is not None:
            for cam in cams[:3]:
                ref_render_scale_rot(mod, g["pos"], g["scales"], g["rotations"], g["opacity"], cam, bg, g["shs"], 3)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for cam in cams:
                ref_render_scale_rot(mod, g["pos"], g["scales"], g["rotations"], g["opacity"], cam, bg, g["shs"], 3)
            torch.cuda.synchronize()
            out["reference_binary_ms_per_view"] = (time.perf_counter() - t0) * 1e3 / len(cams)
            t0 = time.perf_counter()
            for cam in cams:
                GR.rasterize_scale_rot(g["pos"], g["scales"], g["rotations"], g["opacity"], cam, bg, g["shs"], 3)
            torch.cuda.synchronize()
            out["device_ms_per_view_wall"] = (time.perf_counter() - t0) * 1e3 / len(cams)
        else:
            out["reference_binary_ms_per_view"] = "not built"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
