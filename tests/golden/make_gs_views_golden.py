"""Generates tests/golden/gs_views_golden.npz by EXECUTING THE REFERENCE'S OWN dataset, camera, argument and metric code
(gaussian-splatting's scene/dataset_readers.py, scene/colmap_loader.py, scene/cameras.py, utils/camera_utils.py,
utils/general_utils.py, utils/graphics_utils.py, arguments/__init__.py, utils/loss_utils.py, utils/image_utils.py) and
torchvision's save_image, on the CPU. PIXIE_REFERENCE names a checkout of the reference:

    PIXIE_REFERENCE=<checkout> python tests/golden/make_gs_views_golden.py

The function sources are pulled out of the reference files with `ast` (as make_render_golden.py does) and exec'd in
namespaces with stand-ins for the imports that cannot run here: `plyfile` (storePly / fetchPly write and read the
training point cloud, which rendering never uses: no-ops), `simple_knn` / `scene.gaussian_model` (BasicPointCloud only
as a type), and CUDA (scene/cameras.py's `.cuda()` calls are removed from its source and data_device is "cpu"). The only
behavioural shim is `Image.fromarray(int8 array, "RGB")`, which current Pillow refuses: it is given the same bytes viewed
as uint8, which is what older Pillow did.

The dataset files are generated from a seed and stored in the npz (key "file/<relative path>", raw bytes), so the tests
rebuild the same tree. Cases:
  blender_<bg>_<eval>_*     readNerfSyntheticInfo: frames with and without ".png", partial alpha (values where 255 times
                            the composite lands just below an integer), white / black background, eval on / off
  colmap_<case>_*           readColmapSceneInfo: PINHOLE binary, SIMPLE_PINHOLE binary, PINHOLE text (the binary files
                            absent), unsorted image names, eval on / off (llffhold 8)
  loadcam_<k>_*             loadCam + Camera: resolution -1 at widths 1600 and 1601, 1 / 2 / 4 / 8, explicit widths,
                            odd sizes; the gt image and the camera's float32 matrices
  args_<k>_*                get_combined_args: a cfg_args text and a command line, the merged namespace as JSON
  png_<k>                   torchvision.utils.save_image bytes of a ground-truth image and of an unclamped render
  metric_<k>_*              loss_utils.ssim / image_utils.psnr of uint8 image pairs read as k / 255 (float32, CPU)
"""
import ast
import collections
import json
import math
import os
import struct
import sys
import tempfile
import types
from argparse import ArgumentParser, Namespace
from pathlib import Path
from typing import NamedTuple

import numpy as np
import torch
import torch.nn.functional as F
import torchvision
from PIL import Image as PILImage
from torch import nn
from torch.autograd import Variable

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ["PIXIE_REFERENCE"]
GS = os.path.join(REF, "third_party", "PhysGaussian", "gaussian-splatting")


def extract(path, names, ns, edit=None):
    src = open(path).read()
    tree = ast.parse(src)
    for node in tree.body:
        nm = None
        if isinstance(node, (ast.FunctionDef, ast.ClassDef)):
            nm = node.name
        elif isinstance(node, ast.Assign) and isinstance(node.targets[0], ast.Name):
            nm = node.targets[0].id
        if nm in names:
            code = ast.get_source_segment(src, node)
            if edit:
                code = edit(code)
            exec(compile(code, path, "exec"), ns)


class _PIL(types.ModuleType):
    """PIL.Image with fromarray(int8, mode) given the bytes as uint8 (the reference's Blender composite)."""

    def __getattr__(self, name):
        return getattr(PILImage, name)

    @staticmethod
    def fromarray(arr, mode=None):
        if mode is not None and arr.dtype == np.int8:
            arr = arr.view(np.uint8)
        return PILImage.fromarray(arr) if mode is None else PILImage.fromarray(arr, mode)


def namespaces():
    g = {"np": np, "torch": torch, "math": math, "NamedTuple": NamedTuple}
    extract(os.path.join(GS, "utils", "graphics_utils.py"), {"getWorld2View2", "getProjectionMatrix", "fov2focal", "focal2fov"}, g)
    col = {"np": np, "collections": collections, "struct": struct}
    extract(os.path.join(GS, "scene", "colmap_loader.py"),
            {"CameraModel", "Camera", "BaseImage", "CAMERA_MODELS", "CAMERA_MODEL_IDS", "CAMERA_MODEL_NAMES", "qvec2rotmat", "Image",
             "read_next_bytes", "read_intrinsics_text", "read_extrinsics_binary", "read_intrinsics_binary", "read_extrinsics_text"}, col)
    rd = {"os": os, "sys": sys, "np": np, "json": json, "Path": Path, "Image": _PIL("PIL.Image"), "NamedTuple": NamedTuple,
          "BasicPointCloud": collections.namedtuple("BasicPointCloud", "points colors normals"), "SH2RGB": lambda x: x,
          "storePly": lambda *a, **k: None, "fetchPly": lambda *a, **k: None,          # plyfile stand-ins: no file is written
          "read_points3D_binary": lambda *a: (None, None, None), "read_points3D_text": lambda *a: (None, None, None)}
    for k in ("read_extrinsics_text", "read_intrinsics_text", "qvec2rotmat", "read_extrinsics_binary", "read_intrinsics_binary"):
        rd[k] = col[k]
    for k in ("getWorld2View2", "focal2fov", "fov2focal"):
        rd[k] = g[k]
    extract(os.path.join(GS, "scene", "dataset_readers.py"),
            {"CameraInfo", "SceneInfo", "getNerfppNorm", "readColmapCameras", "readColmapSceneInfo", "readCamerasFromTransforms",
             "readNerfSyntheticInfo"}, rd)
    cam = {"torch": torch, "nn": nn, "np": np, "getWorld2View2": g["getWorld2View2"], "getProjectionMatrix": g["getProjectionMatrix"]}
    extract(os.path.join(GS, "scene", "cameras.py"), {"Camera"}, cam, edit=lambda s: s.replace(".cuda()", ""))   # CUDA stand-in
    cu = {"torch": torch, "np": np}
    extract(os.path.join(GS, "utils", "general_utils.py"), {"PILtoTorch"}, cu)
    cu.update({"Camera": cam["Camera"], "fov2focal": g["fov2focal"]})
    extract(os.path.join(GS, "utils", "camera_utils.py"), {"WARNED", "loadCam"}, cu)
    ar = {"ArgumentParser": ArgumentParser, "Namespace": Namespace, "sys": sys, "os": os}
    extract(os.path.join(GS, "arguments", "__init__.py"), {"GroupParams", "ParamGroup", "ModelParams", "PipelineParams", "get_combined_args"}, ar)
    me = {"torch": torch, "F": F, "Variable": Variable, "exp": math.exp}
    extract(os.path.join(GS, "utils", "loss_utils.py"), {"gaussian", "create_window", "ssim", "_ssim"}, me)
    extract(os.path.join(GS, "utils", "image_utils.py"), {"psnr"}, me)
    return rd, cu, ar, me


def c2w_looking_at_origin(pos):
    pos = np.asarray(pos, np.float64)
    back = pos / np.linalg.norm(pos)
    right = np.cross([0.0, 0.0, 1.0], back)
    right /= np.linalg.norm(right)
    m = np.eye(4)
    m[:3, 0], m[:3, 1], m[:3, 2], m[:3, 3] = right, np.cross(back, right), back, pos
    return m


def write_blender(src, rng):
    alphas = np.array([0, 1, 37, 77, 127, 128, 200, 254, 255], np.uint8)
    for split, n in (("train", 3), ("test", 2)):
        os.makedirs(os.path.join(src, split), exist_ok=True)
        frames = []
        for i in range(n):
            rgba = rng.integers(0, 256, (9, 17, 4), dtype=np.uint8)
            rgba[..., 3] = rng.choice(alphas, (9, 17))
            rgba[0, :3] = [[255, 255, 255, 128], [10, 200, 3, 77], [254, 1, 128, 37]]
            PILImage.fromarray(rgba, "RGBA").save(os.path.join(src, split, f"r_{i}.png"))
            az = 2 * math.pi * (i + 0.5 * (split == "test")) / n
            fp = f"./{split}/r_{i}" + (".png" if i % 2 == 0 else "")
            frames.append({"file_path": fp, "transform_matrix": c2w_looking_at_origin([4 * math.cos(az), 4 * math.sin(az), 1.5]).tolist()})
        with open(os.path.join(src, f"transforms_{split}.json"), "w") as f:
            json.dump({"camera_angle_x": 0.69, "frames": frames}, f)


def write_colmap(src, rng, model, binary, n=10):
    names = [f"{c}.png" for c in "cajbidhegf"[:n]]
    sp = os.path.join(src, "sparse", "0")
    os.makedirs(sp, exist_ok=True)
    os.makedirs(os.path.join(src, "images"), exist_ok=True)
    cams, imgs = [], []
    for i, name in enumerate(names):
        W, H = 20 + i, 12 + i % 3
        q = rng.normal(0, 1, 4)
        q /= np.linalg.norm(q)
        t = rng.normal(0, 1, 3) + [0.0, 0.0, 4.0]
        p = [rng.uniform(0.7, 1.1) * W, W / 2, H / 2] if model == "SIMPLE_PINHOLE" else \
            [rng.uniform(0.7, 1.1) * W, rng.uniform(0.7, 1.1) * W, W / 2, H / 2]
        cams.append((i + 1, model, W, H, p))
        imgs.append((i + 1, q, t, i + 1, name))
        PILImage.fromarray(rng.integers(0, 256, (H, W, 3), dtype=np.uint8)).save(os.path.join(src, "images", name))
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


def store_tree(out, root, prefix):
    for d, _, files in os.walk(root):
        for fn in sorted(files):
            p = os.path.join(d, fn)
            out[f"file/{prefix}/{os.path.relpath(p, root)}"] = np.frombuffer(open(p, "rb").read(), np.uint8)


def put_cams(out, key, cams):
    out[key + "_R"] = np.array([c.R for c in cams], np.float64).reshape(-1, 3, 3)
    out[key + "_T"] = np.array([c.T for c in cams], np.float64).reshape(-1, 3)
    out[key + "_fov"] = np.array([[c.FovX, c.FovY] for c in cams], np.float64).reshape(-1, 2)
    out[key + "_wh"] = np.array([[c.width, c.height] for c in cams], np.int64).reshape(-1, 2)
    out[key + "_names"] = np.frombuffer(json.dumps([os.path.basename(c.image_path) for c in cams]).encode(), np.uint8)


def main():
    rd, cu, ar, me = namespaces()
    rng = np.random.default_rng(20261019)
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        src = os.path.join(tmp, "blender")
        write_blender(src, rng)
        store_tree(out, src, "blender")
        for white in (False, True):
            for ev in (False, True):
                info = rd["readNerfSyntheticInfo"](src, white, ev)
                key = f"blender_{int(white)}_{int(ev)}"
                put_cams(out, key + "_train", info.train_cameras)
                put_cams(out, key + "_test", info.test_cameras)
                out[key + "_images"] = np.stack([np.array(c.image) for c in info.train_cameras + info.test_cameras])

        for case, model, binary in (("pinhole_bin", "PINHOLE", True), ("simple_bin", "SIMPLE_PINHOLE", True), ("pinhole_txt", "PINHOLE", False)):
            src = os.path.join(tmp, case)
            write_colmap(src, rng, model, binary)
            store_tree(out, src, case)
            for ev in (False, True):
                info = rd["readColmapSceneInfo"](src, None, ev)
                put_cams(out, f"colmap_{case}_{int(ev)}_train", info.train_cameras)
                put_cams(out, f"colmap_{case}_{int(ev)}_test", info.test_cameras)

    # loadCam: (width, height, resolution)
    lc = [(1600, 3, -1), (1601, 6, -1), (3203, 7, -1), (33, 17, 1), (33, 17, 2), (35, 19, 4), (35, 19, 8), (33, 17, 100), (33, 17, 20), (9, 11, 2)]
    out["loadcam_cases"] = np.array(lc, np.int64)
    for k, (W, H, res) in enumerate(lc):
        arr = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        R = np.linalg.qr(rng.normal(size=(3, 3)))[0]
        T = rng.normal(size=3)
        info = rd["CameraInfo"](uid=k, R=R, T=T, FovY=0.5, FovX=0.6, image=PILImage.fromarray(arr), image_path="x.png", image_name="x",
                                width=W, height=H)
        c = cu["loadCam"](types.SimpleNamespace(resolution=res, data_device="cpu"), k, info, 1.0)
        out[f"loadcam_{k}_in"] = arr
        out[f"loadcam_{k}_R"], out[f"loadcam_{k}_T"] = R, T
        out[f"loadcam_{k}_gt"] = c.original_image.numpy()
        out[f"loadcam_{k}_world_view"] = c.world_view_transform.numpy()
        out[f"loadcam_{k}_full_proj"] = c.full_proj_transform.numpy()
        out[f"loadcam_{k}_center"] = c.camera_center.numpy()
        if k == 4:
            with tempfile.TemporaryDirectory() as d:
                torchvision.utils.save_image(c.original_image, os.path.join(d, "gt.png"))
                out["png_gt_in"] = arr
                out["png_gt"] = np.frombuffer(open(os.path.join(d, "gt.png"), "rb").read(), np.uint8)
    img = torch.from_numpy(rng.normal(0.5, 0.4, (3, 13, 21)).astype(np.float32))
    with tempfile.TemporaryDirectory() as d:
        torchvision.utils.save_image(img, os.path.join(d, "r.png"))
        out["png_render_in"] = img.numpy()
        out["png_render"] = np.frombuffer(open(os.path.join(d, "r.png"), "rb").read(), np.uint8)

    # get_combined_args as render.py builds its parser
    cfg = ("Namespace(data_device='cuda', eval=True, images='images', model_path='./out', resolution=2, sh_degree=2, "
           "source_path='/data/scene', white_background=True)")
    cases = [[], ["-r", "4", "-s", "/other", "-i", "imgs"], ["--eval", "-w", "--sh_degree", "1", "--iteration", "500", "--skip_test"],
             ["--resolution", "-1", "--quiet"]]
    out["args_cfg"] = np.frombuffer(cfg.encode(), np.uint8)
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "cfg_args"), "w") as f:
            f.write(cfg)
        merged = []
        for argv in cases:
            parser = ArgumentParser()
            ar["ModelParams"](parser, sentinel=True)
            ar["PipelineParams"](parser)
            parser.add_argument("--iteration", default=-1, type=int)
            parser.add_argument("--skip_train", action="store_true")
            parser.add_argument("--skip_test", action="store_true")
            parser.add_argument("--quiet", action="store_true")
            saved = sys.argv
            sys.argv = ["render.py", "-m", d] + argv
            try:
                a = ar["get_combined_args"](parser)
            finally:
                sys.argv = saved
            v = vars(a)
            v["model_path"] = "<model>"
            merged.append(v)
    out["args_cases"] = np.frombuffer(json.dumps(cases).encode(), np.uint8)
    out["args_merged"] = np.frombuffer(json.dumps(merged).encode(), np.uint8)

    # ssim / psnr: random, noisy and near-flat pairs
    for k, (H, W) in enumerate(((6, 9), (23, 31), (5, 7))):
        a = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        noisy = np.clip(a.astype(np.int64) + rng.integers(-20, 21, a.shape), 0, 255).astype(np.uint8)
        flat = np.full((H, W, 3), 200, np.uint8)
        flat2 = flat.copy()
        flat2[rng.random((H, W)) < 0.05] = 201
        flat2[H // 2, W // 2] = 201
        for j, (x, y) in enumerate(((a, rng.integers(0, 256, (H, W, 3), dtype=np.uint8)), (a, noisy), (flat, flat2))):
            tx = torchvision.transforms.functional.to_tensor(x).unsqueeze(0)
            ty = torchvision.transforms.functional.to_tensor(y).unsqueeze(0)
            out[f"metric_{k}_{j}_a"], out[f"metric_{k}_{j}_b"] = x, y
            out[f"metric_{k}_{j}_ssim"] = np.float32(me["ssim"](tx, ty).item())
            out[f"metric_{k}_{j}_psnr"] = np.float32(me["psnr"](tx, ty).item())
    np.savez_compressed(os.path.join(HERE, "gs_views_golden.npz"), **out)
    print(f"wrote {len(out)} arrays")


if __name__ == "__main__":
    main()
