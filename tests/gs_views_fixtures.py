"""Seeded scenes, datasets and the reference rasterizer binary, shared by the dataset-view tests and
scripts/profile_gs_dataset_render.py. Nothing here needs pytest."""
from __future__ import annotations

import importlib.machinery
import importlib.util
import json
import math
import os
import struct

import numpy as np
import torch
from PIL import Image


def write_checkpoint(model, rng, n, K, iteration=7000, extent=0.6):
    names = ["x", "y", "z", "nx", "ny", "nz", "f_dc_0", "f_dc_1", "f_dc_2"] + [f"f_rest_{i}" for i in range(3 * K - 3)] + \
            ["opacity", "scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3"]
    a = np.zeros(n, dtype=[(nm, "<f4") for nm in names])
    for c in "xyz":
        a[c] = rng.normal(0, extent, n)
    for nm in names:
        if nm.startswith("f_"):
            a[nm] = rng.normal(0, 0.5, n)
        elif nm.startswith("scale"):
            a[nm] = rng.uniform(-6.0, -2.5, n)
        elif nm.startswith("rot"):
            a[nm] = rng.normal(0, 1, n)
    a["opacity"] = rng.normal(0.0, 2.0, n)
    d = os.path.join(model, "point_cloud", f"iteration_{iteration}")
    os.makedirs(d, exist_ok=True)
    head = ["ply", "format binary_little_endian 1.0", f"element vertex {n}"] + [f"property float {nm}" for nm in names] + ["end_header"]
    with open(os.path.join(d, "point_cloud.ply"), "wb") as f:
        f.write(("\n".join(head) + "\n").encode() + a.tobytes())
    return a


def look_at_c2w(pos, target=(0.0, 0.0, 0.0)):
    """A Blender (OpenGL axes) camera-to-world matrix at `pos` looking at `target`, z up."""
    pos = np.asarray(pos, np.float64)
    back = pos - np.asarray(target)
    back /= np.linalg.norm(back)
    right = np.cross([0.0, 0.0, 1.0], back)
    right /= np.linalg.norm(right)
    up = np.cross(back, right)
    m = np.eye(4)
    m[:3, 0], m[:3, 1], m[:3, 2], m[:3, 3] = right, up, back, pos
    return m


def write_blender(src, rng, n_train, n_test, W, H, with_ext=False, alpha_values=None, empty_test_file=False):
    os.makedirs(os.path.join(src, "train"), exist_ok=True)
    os.makedirs(os.path.join(src, "test"), exist_ok=True)
    for split, n in (("train", n_train), ("test", n_test)):
        frames = []
        for i in range(n):
            rgba = rng.integers(0, 256, (H, W, 4), dtype=np.uint8)
            if alpha_values is not None:
                rgba[..., 3] = rng.choice(alpha_values, (H, W))
            Image.fromarray(rgba, "RGBA").save(os.path.join(src, split, f"r_{i}.png"))
            az = 2 * math.pi * (i + 0.5 * (split == "test")) / max(n, 1)
            fp = f"./{split}/r_{i}" + (".png" if with_ext and i % 2 == 0 else "")
            frames.append({"file_path": fp, "transform_matrix": look_at_c2w([4 * math.cos(az), 4 * math.sin(az), 1.5]).tolist()})
        with open(os.path.join(src, f"transforms_{split}.json"), "w") as f:
            json.dump({"camera_angle_x": 0.69, "frames": [] if (empty_test_file and split == "test") else frames}, f)


def write_colmap(src, rng, names, sizes, binary=True, model="PINHOLE", images_dir="images"):
    """sparse/0 with one camera per image (sizes[i] = (W, H)), images written under <src>/<images_dir>."""
    sp = os.path.join(src, "sparse", "0")
    os.makedirs(sp, exist_ok=True)
    os.makedirs(os.path.join(src, images_dir), exist_ok=True)
    cams, imgs = [], []
    for i, (name, (W, H)) in enumerate(zip(names, sizes)):
        q = rng.normal(0, 1, 4)
        q /= np.linalg.norm(q)
        t = np.array([0.0, 0.0, 4.0])             # the world origin 4 units in front of every camera
        params = [0.9 * W, W / 2, H / 2] if model == "SIMPLE_PINHOLE" else [0.9 * W, 0.85 * W, W / 2, H / 2]
        cams.append((i + 1, model, W, H, params))
        imgs.append((i + 1, q, t, i + 1, name))
        Image.fromarray(rng.integers(0, 256, (H, W, 3), dtype=np.uint8)).save(os.path.join(src, images_dir, name))
    if binary:
        with open(os.path.join(sp, "cameras.bin"), "wb") as f:
            f.write(struct.pack("<Q", len(cams)))
            for cid, m, W, H, p in cams:
                f.write(struct.pack("<iiQQ", cid, {"SIMPLE_PINHOLE": 0, "PINHOLE": 1}[m], W, H) + struct.pack("<" + "d" * len(p), *p))
        with open(os.path.join(sp, "images.bin"), "wb") as f:
            f.write(struct.pack("<Q", len(imgs)))
            for iid, q, t, cid, name in imgs:
                f.write(struct.pack("<idddddddi", iid, *q, *t, cid) + name.encode() + b"\x00")
                f.write(struct.pack("<Q", 1) + struct.pack("<ddq", 1.0, 2.0, -1))
    else:
        with open(os.path.join(sp, "cameras.txt"), "w") as f:
            f.write("# camera list\n")
            for cid, m, W, H, p in cams:
                f.write(f"{cid} {m} {W} {H} " + " ".join(repr(float(v)) for v in p) + "\n")
        with open(os.path.join(sp, "images.txt"), "w") as f:
            f.write("# image list\n")
            for iid, q, t, cid, name in imgs:
                f.write(f"{iid} " + " ".join(repr(float(v)) for v in (*q, *t)) + f" {cid} {name}\n1.0 2.0 -1\n")
    return cams, imgs


def tree_snapshot(path):
    out = {}
    for d, _, files in os.walk(path):
        for fn in files:
            p = os.path.join(d, fn)
            out[p] = (os.path.getsize(p), os.path.getmtime(p))
    return out


def reference_rasterizer():
    """The reference's rasterizer extension built by oracle/build_gs_rasterizer_ref.py, or None when it was not built."""
    from oracle import build_gs_rasterizer_ref as B
    path = B.artefact()
    if path is None:
        return None
    loader = importlib.machinery.ExtensionFileLoader(B.NAME, path)
    spec = importlib.util.spec_from_file_location(B.NAME, path, loader=loader)
    mod = importlib.util.module_from_spec(spec)
    loader.exec_module(mod)
    return mod


def ref_render_scale_rot(mod, means, scales, rots, opacity, cam, bg, shs, deg):
    """The reference rasterizer as gaussian_renderer.render calls it with PipelineParams' defaults."""
    dev = means.device
    empty = torch.empty(0, device=dev)
    out = mod.rasterize_gaussians(torch.as_tensor(bg, dtype=torch.float32, device=dev), means, empty, opacity.reshape(-1, 1).contiguous(),
                                  scales, rots, 1.0, empty, cam.world_view_transform.to(dev), cam.full_proj_transform.to(dev),
                                  math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5), cam.image_height, cam.image_width, shs, deg,
                                  cam.camera_center.to(dev), False, False)
    return out[1], out[2]


def seeded_gaussians(n, seed, dev):
    """Means in a ball, log-uniform anisotropic scales (2e-4 .. 0.2), random unit quaternions, opacities in (0.02, 1]."""
    g = torch.Generator().manual_seed(seed)
    pos = torch.randn(n, 3, generator=g) * 0.6
    pos[: n // 20] = torch.randn(n // 20, 3, generator=g) * 8.0
    scales = torch.exp(torch.rand(n, 3, generator=g) * math.log(1e3)) * 2e-4
    rots = torch.nn.functional.normalize(torch.randn(n, 4, generator=g), dim=1)
    opacity = torch.rand(n, 1, generator=g) * 0.98 + 0.02
    shs = torch.randn(n, 16, 3, generator=g) * 0.4
    return [t.to(dev, torch.float32).contiguous() for t in (pos, scales, rots, opacity, shs)]
