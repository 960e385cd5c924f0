"""Render a trained 3DGS scene's dataset views from its files: the `gs` step of Pixie's render.py, which runs
gaussian-splatting's `render.py --model_path <gs_output>`.

    python -m pixie_b200.gs_dataset_render -m <model> [-s SOURCE] [-i IMAGES] [-r RES] [-w] [--eval] [--iteration N]
                                           [--skip_train] [--skip_test] [--quiet]

writes <model>/{train,test}/ours_<iter>/{renders,gt}/{idx:05d}.png as the reference does. The host half restates the
reference's readers, in its functions' names and argument meaning:

    get_combined_args(argv)                                arguments/__init__.py:92-112 (cfg_args parsed, not eval'd)
    readCamerasFromTransforms / readNerfSyntheticInfo      scene/dataset_readers.py:179-259 (Blender data)
    readColmapCameras / readColmapSceneInfo                scene/dataset_readers.py:68-177 with colmap_loader.py
    loadCam                                                utils/camera_utils.py:19-52 with PILtoTorch

Deviations, each deliberate:
- cfg_args is parsed with `ast` and must be one `Namespace(...)` call of keyword literals; the reference `eval`s it.
- Nothing is written under the source path: the reference writes a random `points3d.ply` (Blender) or a converted
  `points3D.ply` (COLMAP) there when it is missing, for training; rendering never reads it.
- A 4-pixel-high image is rejected: the reference's alpha-mask test reads the image height (`shape[1] == 4`).
- `--convert_SHs_python`, `--compute_cov3D_python` and `--debug` are rejected, and so is a view loadCam cannot take
  (its mode or target height, see above), all before any device work.

The device half decodes the checkpoint once (scene_files.decode_checkpoint_ply_scale_rot), draws each view with the
rasterizer's scale/rotation entry point (gs_render.rasterize_scale_rot) and quantises the render and the ground truth with
torchvision's save_image expression (mul(255), add_(0.5), clamp_(0, 255), truncation to uint8) as separate float32 ops on
the device. A pool of encoder threads writes the PNGs with PIL as save_image does while the device draws the next views.
"""
from __future__ import annotations

import argparse
import ast
import collections
import concurrent.futures
import json
import math
import os
import struct
import sys
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch
from PIL import Image

from . import gs_render, scene_files


@dataclass
class CameraInfo:
    """scene/dataset_readers.py's CameraInfo: R is stored transposed (the reference's glm convention)."""
    uid: int
    R: np.ndarray
    T: np.ndarray
    FovY: float
    FovX: float
    image: Image.Image
    image_path: str
    image_name: str
    width: int
    height: int


# ------------------------------------------------------------------------------------------------ arguments
_MODEL_DEFAULTS = {"sh_degree": 3, "source_path": "", "model_path": "", "images": "images", "resolution": -1,
                   "white_background": False, "data_device": "cuda", "eval": False}
_REJECTED = ("convert_SHs_python", "compute_cov3D_python", "debug")


def build_parser() -> argparse.ArgumentParser:
    """render.py's parser: ModelParams(sentinel=True) (every default None), PipelineParams and its own flags."""
    p = argparse.ArgumentParser(description="Render a trained Gaussian model's dataset views (gaussian-splatting render.py)")
    p.add_argument("--sh_degree", type=int, default=None)
    p.add_argument("--source_path", "-s", type=str, default=None)
    p.add_argument("--model_path", "-m", type=str, default=None)
    p.add_argument("--images", "-i", type=str, default=None)
    p.add_argument("--resolution", "-r", type=int, default=None)
    p.add_argument("--white_background", "-w", action="store_true", default=None)
    p.add_argument("--data_device", type=str, default=None)
    p.add_argument("--eval", action="store_true", default=None)
    for k in _REJECTED:
        p.add_argument("--" + k, action="store_true", help="not supported (rejected)")
    p.add_argument("--iteration", default=-1, type=int)
    p.add_argument("--skip_train", action="store_true")
    p.add_argument("--skip_test", action="store_true")
    p.add_argument("--quiet", action="store_true")
    return p


def parse_cfg_args(text: str) -> Dict:
    """The keywords of a `Namespace(k=literal, ...)` cfg_args file. Anything else raises ValueError."""
    try:
        tree = ast.parse(text.strip(), mode="eval")
    except SyntaxError as e:
        raise ValueError(f"cfg_args is not a Namespace(...) expression: {e}") from None
    call = tree.body
    if not (isinstance(call, ast.Call) and isinstance(call.func, ast.Name) and call.func.id == "Namespace" and not call.args):
        raise ValueError("cfg_args must hold one Namespace(...) call with keyword arguments only")
    out = {}
    for kw in call.keywords:
        if kw.arg is None:
            raise ValueError("cfg_args: ** arguments are not accepted")
        try:
            out[kw.arg] = ast.literal_eval(kw.value)
        except ValueError:
            raise ValueError(f"cfg_args: {kw.arg} is not a literal") from None
    return out


def get_combined_args(argv: Sequence[str], parser: Optional[argparse.ArgumentParser] = None) -> argparse.Namespace:
    """<model_path>/cfg_args overridden by every command-line value that is not None, as get_combined_args merges them;
    ModelParams' defaults fill what neither gives. Raises on the rejected pipeline options and, as the reference does,
    when cfg_args is missing."""
    parser = parser or build_parser()
    args = parser.parse_args(list(argv))
    for k in _REJECTED:
        if getattr(args, k):
            raise ValueError(f"--{k} is not supported: the device rasterizer evaluates SH colours and covariances itself")
    if args.model_path is None:
        raise ValueError("--model_path / -m is required")
    with open(os.path.join(args.model_path, "cfg_args")) as f:     # a missing file raises, as in the reference
        cfg = parse_cfg_args(f.read())
    merged = dict(_MODEL_DEFAULTS)
    merged.update(cfg)
    for k, v in vars(args).items():
        if v is not None:
            merged[k] = v
    for k in _REJECTED:
        if merged.get(k):
            raise ValueError(f"{k} is not supported: the device rasterizer evaluates SH colours and covariances itself")
    return argparse.Namespace(**merged)


# ------------------------------------------------------------------------------------------------ Blender data
def _composite_trunc(rgba: np.ndarray, white_background: bool) -> np.ndarray:
    """RGBA uint8 composited over the background in float64 and stored as trunc(255 composite). The reference writes
    `Image.fromarray(np.array(arr * 255.0, dtype=np.byte), "RGB")`: the int8 cast wraps and the bytes are read back as
    uint8, which is trunc. (Current Pillow refuses int8 data with a mode, so the reference line itself no longer runs.)"""
    bg = np.array([1, 1, 1]) if white_background else np.array([0, 0, 0])
    norm = rgba / 255.0
    arr = norm[:, :, :3] * norm[:, :, 3:4] + bg * (1 - norm[:, :, 3:4])
    return np.trunc(arr * 255.0).astype(np.uint8)


def readCamerasFromTransforms(path: str, transformsfile: str, white_background: bool, extension: str = ".png") -> List[CameraInfo]:
    cam_infos = []
    with open(os.path.join(path, transformsfile)) as f:
        contents = json.load(f)
    fovx = contents["camera_angle_x"]
    for idx, frame in enumerate(contents["frames"]):
        file_path = frame["file_path"]
        if not file_path.endswith(extension):
            file_path = file_path + extension
        cam_name = os.path.join(path, file_path)
        c2w = np.array(frame["transform_matrix"], dtype=np.float64)
        c2w[:3, 1:3] *= -1
        w2c = np.linalg.inv(c2w)
        R = np.transpose(w2c[:3, :3])
        T = w2c[:3, 3]
        with Image.open(cam_name) as im:
            rgba = np.array(im.convert("RGBA"))
        image = Image.fromarray(_composite_trunc(rgba, white_background), "RGB")
        fovy = gs_render.focal2fov(fov2focal(fovx, image.size[0]), image.size[1])
        cam_infos.append(CameraInfo(idx, R, T, fovy, fovx, image, cam_name, os.path.splitext(os.path.basename(file_path))[0],
                                    image.size[0], image.size[1]))
    return cam_infos


def fov2focal(fov: float, pixels: float) -> float:
    return pixels / (2 * math.tan(fov / 2))


def readNerfSyntheticInfo(path: str, white_background: bool, eval: bool, extension: str = ".png"):
    """(train, test) camera lists; without `eval` the test frames join the training ones."""
    train = readCamerasFromTransforms(path, "transforms_train.json", white_background, extension)
    test = readCamerasFromTransforms(path, "transforms_test.json", white_background, extension)
    if not eval:
        train.extend(test)
        test = []
    return train, test


# ------------------------------------------------------------------------------------------------ COLMAP data
_COLMAP_MODELS = {0: ("SIMPLE_PINHOLE", 3), 1: ("PINHOLE", 4), 2: ("SIMPLE_RADIAL", 4), 3: ("RADIAL", 5), 4: ("OPENCV", 8),
                  5: ("OPENCV_FISHEYE", 8), 6: ("FULL_OPENCV", 12), 7: ("FOV", 5), 8: ("SIMPLE_RADIAL_FISHEYE", 4),
                  9: ("RADIAL_FISHEYE", 5), 10: ("THIN_PRISM_FISHEYE", 12)}


def qvec2rotmat(q) -> np.ndarray:
    return np.array([
        [1 - 2 * q[2] ** 2 - 2 * q[3] ** 2, 2 * q[1] * q[2] - 2 * q[0] * q[3], 2 * q[3] * q[1] + 2 * q[0] * q[2]],
        [2 * q[1] * q[2] + 2 * q[0] * q[3], 1 - 2 * q[1] ** 2 - 2 * q[3] ** 2, 2 * q[2] * q[3] - 2 * q[0] * q[1]],
        [2 * q[3] * q[1] - 2 * q[0] * q[2], 2 * q[2] * q[3] + 2 * q[0] * q[1], 1 - 2 * q[1] ** 2 - 2 * q[2] ** 2]])


def _read(f, n: int, fmt: str):
    data = f.read(n)
    if len(data) != n:
        raise ValueError(f"{f.name}: truncated")
    return struct.unpack("<" + fmt, data)


def read_extrinsics_binary(path: str) -> Dict:
    """{image_id: (qvec, tvec, camera_id, name)} in file order."""
    images = {}
    with open(path, "rb") as f:
        for _ in range(_read(f, 8, "Q")[0]):
            p = _read(f, 64, "idddddddi")
            name = b""
            while True:
                c = f.read(1)
                if not c:
                    raise ValueError(f"{path}: truncated image name")
                if c == b"\x00":
                    break
                name += c
            n2d = _read(f, 8, "Q")[0]
            f.seek(24 * n2d, os.SEEK_CUR)
            images[p[0]] = (np.array(p[1:5]), np.array(p[5:8]), p[8], name.decode("utf-8"))
    return images


def read_intrinsics_binary(path: str) -> Dict:
    """{camera_id: (model name, width, height, params)}."""
    cams = {}
    with open(path, "rb") as f:
        for _ in range(_read(f, 8, "Q")[0]):
            cid, mid, w, h = _read(f, 24, "iiQQ")
            if mid not in _COLMAP_MODELS:
                raise ValueError(f"{path}: unknown camera model id {mid}")
            name, k = _COLMAP_MODELS[mid]
            cams[cid] = (name, w, h, np.array(_read(f, 8 * k, "d" * k)))
    return cams


def read_extrinsics_text(path: str) -> Dict:
    images = {}
    with open(path) as f:
        while True:
            line = f.readline()
            if not line:
                break
            line = line.strip()
            if line and line[0] != "#":
                e = line.split()
                images[int(e[0])] = (np.array(tuple(map(float, e[1:5]))), np.array(tuple(map(float, e[5:8]))), int(e[8]), e[9])
                f.readline()
    return images


def read_intrinsics_text(path: str) -> Dict:
    """As colmap_loader.read_intrinsics_text: only PINHOLE cameras (it asserts so)."""
    cams = {}
    with open(path) as f:
        for line in f:
            line = line.strip()
            if line and line[0] != "#":
                e = line.split()
                if e[1] != "PINHOLE":
                    raise ValueError(f"{path}: the text camera reader supports PINHOLE cameras only, got {e[1]}")
                cams[int(e[0])] = (e[1], int(e[2]), int(e[3]), np.array(tuple(map(float, e[4:]))))
    return cams


def readColmapCameras(cam_extrinsics: Dict, cam_intrinsics: Dict, images_folder: str) -> List[CameraInfo]:
    infos = []
    for qvec, tvec, camera_id, name in cam_extrinsics.values():
        model, width, height, params = cam_intrinsics[camera_id]
        if model == "SIMPLE_PINHOLE":
            FovY, FovX = gs_render.focal2fov(params[0], height), gs_render.focal2fov(params[0], width)
        elif model == "PINHOLE":
            FovY, FovX = gs_render.focal2fov(params[1], height), gs_render.focal2fov(params[0], width)
        else:
            raise ValueError(f"COLMAP camera model {model} not handled: only undistorted datasets (PINHOLE or SIMPLE_PINHOLE)")
        image_path = os.path.join(images_folder, os.path.basename(name))
        image = Image.open(image_path)
        image.load()
        infos.append(CameraInfo(camera_id, np.transpose(qvec2rotmat(qvec)), np.array(tvec), FovY, FovX, image, image_path,
                                os.path.basename(image_path).split(".")[0], width, height))
    return infos


def readColmapSceneInfo(path: str, images: Optional[str], eval: bool, llffhold: int = 8):
    """(train, test) camera lists sorted by image name; with `eval` every llffhold-th goes to test."""
    sparse = os.path.join(path, "sparse/0")
    try:
        extr = read_extrinsics_binary(os.path.join(sparse, "images.bin"))
        intr = read_intrinsics_binary(os.path.join(sparse, "cameras.bin"))
    except (OSError, ValueError, struct.error):
        extr = read_extrinsics_text(os.path.join(sparse, "images.txt"))
        intr = read_intrinsics_text(os.path.join(sparse, "cameras.txt"))
    infos = sorted(readColmapCameras(extr, intr, os.path.join(path, "images" if images is None else images)), key=lambda c: c.image_name)
    if eval:
        return [c for i, c in enumerate(infos) if i % llffhold != 0], [c for i, c in enumerate(infos) if i % llffhold == 0]
    return infos, []


# ------------------------------------------------------------------------------------------------ loadCam
def load_resolution(orig_w: int, orig_h: int, resolution: int, resolution_scale: float = 1.0):
    """loadCam's target (width, height)."""
    if resolution in [1, 2, 4, 8]:
        return round(orig_w / (resolution_scale * resolution)), round(orig_h / (resolution_scale * resolution))
    if resolution == -1:
        global_down = orig_w / 1600 if orig_w > 1600 else 1
    else:
        global_down = orig_w / resolution
    scale = float(global_down) * float(resolution_scale)
    return int(orig_w / scale), int(orig_h / scale)


def _check_loaded(arr_shape, mode: str, path: str) -> None:
    if len(arr_shape) != 3 or arr_shape[2] not in (3, 4):
        raise ValueError(f"{path}: need an RGB or RGBA image, got mode {mode}")
    if arr_shape[0] == 4:
        raise ValueError(f"{path}: a 4-pixel-high image is not supported (the reference reads its height as the channel count "
                         "and would mask it)")


def check_views(views: Sequence[CameraInfo], resolution: int, resolution_scale: float = 1.0) -> None:
    """Raises for the first view loadCam would refuse (mode or target height), so that a run fails before any device work."""
    for info in views:
        W, H = load_resolution(*info.image.size, resolution, resolution_scale)
        channels = {"RGB": 3, "RGBA": 4}.get(info.image.mode, 0)
        _check_loaded((H, W, channels) if channels else (H, W), info.image.mode, info.image_path)


def loadCam(resolution: int, cam_info: CameraInfo, resolution_scale: float = 1.0):
    """(camera, gt uint8 (H, W, 3)): the image resized with PIL as PILtoTorch does, the alpha channel dropped."""
    size = load_resolution(*cam_info.image.size, resolution, resolution_scale)
    arr = np.array(cam_info.image.resize(size))
    _check_loaded(arr.shape, cam_info.image.mode, cam_info.image_path)
    gt = np.ascontiguousarray(arr[:, :, :3])
    cam = gs_render.make_camera(cam_info.R, cam_info.T, cam_info.FovX, cam_info.FovY, gt.shape[1], gt.shape[0])
    return cam, gt


def read_scene(args: argparse.Namespace):
    """Scene's camera lists for the merged arguments: (train, test) CameraInfo lists."""
    src = os.path.abspath(args.source_path)
    if os.path.exists(os.path.join(src, "sparse")):
        return readColmapSceneInfo(src, args.images, args.eval)
    if os.path.exists(os.path.join(src, "transforms_train.json")):
        return readNerfSyntheticInfo(src, args.white_background, args.eval)
    raise ValueError(f"{src}: could not recognize the scene type (no sparse/ and no transforms_train.json)")


# ------------------------------------------------------------------------------------------------ device
def quantize(img: torch.Tensor) -> torch.Tensor:
    """save_image's ndarray: (3, H, W) float -> (H, W, 3) uint8 by mul(255), add_(0.5), clamp_(0, 255), truncation."""
    return img.mul(255).add_(0.5).clamp_(0, 255).permute(1, 2, 0).to(torch.uint8)


def save_png(arr: np.ndarray, path: str) -> None:
    """The file save_image writes for the quantised array."""
    Image.fromarray(arr).save(path)


_ENCODERS = max(1, min(8, os.cpu_count() or 1))


def _write_view(ev, ren: torch.Tensor, gt: torch.Tensor, ren_path: str, gt_path: str) -> None:
    ev.synchronize()
    save_png(ren.numpy(), ren_path)
    save_png(gt.numpy(), gt_path)


def render_set(model_path: str, name: str, iteration: int, views, gaussians: Dict[str, torch.Tensor], sh_degree: int, background,
               resolution: int, quiet: bool = False) -> int:
    """Renders and writes one split; returns the number of views. A pool of encoder threads writes the PNGs (zlib releases
    the GIL) while the device draws the next views; at most two views per encoder are in flight."""
    render_path = os.path.join(model_path, name, f"ours_{iteration}", "renders")
    gts_path = os.path.join(model_path, name, f"ours_{iteration}", "gt")
    os.makedirs(render_path, exist_ok=True)
    os.makedirs(gts_path, exist_ok=True)
    if not views:
        return 0
    dev = gaussians["pos"].device
    pending: "collections.deque" = collections.deque()
    with concurrent.futures.ThreadPoolExecutor(max_workers=_ENCODERS) as pool:
        try:
            for idx, info in enumerate(views):
                cam, gt_np = loadCam(resolution, info)
                img, _ = gs_render.rasterize_scale_rot(gaussians["pos"], gaussians["scales"], gaussians["rotations"], gaussians["opacity"],
                                                       cam, background, gaussians["shs"], sh_degree)
                gt = torch.from_numpy(gt_np).to(dev).permute(2, 0, 1) / 255.0
                ren_h = torch.empty((cam.image_height, cam.image_width, 3), dtype=torch.uint8, pin_memory=True)
                gt_h = torch.empty_like(ren_h, pin_memory=True)
                ren_h.copy_(quantize(img), non_blocking=True)
                gt_h.copy_(quantize(gt), non_blocking=True)
                ev = torch.cuda.Event()
                ev.record()
                pending.append(pool.submit(_write_view, ev, ren_h, gt_h, os.path.join(render_path, f"{idx:05d}.png"),
                                           os.path.join(gts_path, f"{idx:05d}.png")))
                while len(pending) > 2 * _ENCODERS or (pending and pending[0].done()):
                    pending.popleft().result()              # re-raises an encoder's error here
                if not quiet:
                    print(f"\rRendering {name}: {idx + 1}/{len(views)}", end="", file=sys.stderr)
            while pending:
                pending.popleft().result()
        finally:
            for f in pending:
                f.cancel()
    if not quiet:
        print(file=sys.stderr)
    return len(views)


def render_sets(args: argparse.Namespace) -> Dict[str, int]:
    """render.py's render_sets: the latest (or --iteration) checkpoint, decoded once, over both splits."""
    train, test = read_scene(args)
    check_views((train if not args.skip_train else []) + (test if not args.skip_test else []), int(args.resolution))
    folder = os.path.join(args.model_path, "point_cloud")
    iteration = scene_files.search_for_max_iteration(folder) if args.iteration == -1 else int(args.iteration)
    ply = os.path.join(folder, f"iteration_{iteration}", "point_cloud.ply")
    sh_degree = int(args.sh_degree)
    g = scene_files.decode_checkpoint_ply_scale_rot(ply, sh_degree, device="cuda")
    background = [1.0, 1.0, 1.0] if args.white_background else [0.0, 0.0, 0.0]
    out = {}
    with torch.no_grad():
        if not args.skip_train:
            out["train"] = render_set(args.model_path, "train", iteration, train, g, sh_degree, background, int(args.resolution), args.quiet)
        if not args.skip_test:
            out["test"] = render_set(args.model_path, "test", iteration, test, g, sh_degree, background, int(args.resolution), args.quiet)
    return out


def main(argv: Optional[Sequence[str]] = None) -> int:
    args = get_combined_args(sys.argv[1:] if argv is None else argv)
    if not args.quiet:
        print("Rendering " + args.model_path, file=sys.stderr)
    render_sets(args)
    return 0


if __name__ == "__main__":
    sys.exit(main())
