"""Command line of PhysGaussian's gs_simulation.py: simulate (and render / export) one scene from its files.

    python -m pixie_b200.gs_simulation --model_path <trained model> --config <physics config .json> \\
        --point_cloud_path <mapped_preds.ply> --output_path <dir> [--render_img] [--save_ply] [--white_bg] \\
        [--optimization_output_path <dir> [--replay_epoch N]]

writes `<output_path>/frames/{frame:05d}.png` under --render_img and `<output_path>/ply_files/frame_{frame:05d}.ply` under
--render_img --save_ply: the reference exports PLYs only inside its render branch (gs_simulation.py:593-628), and so does
this one. Existing files are overwritten; the output directories are not deleted first (the reference deletes them).
--compile_video, --debug and configs whose particle filling asks for `smooth` are rejected before any device work.
"""
from __future__ import annotations

import argparse
import os
import struct
import zlib
from typing import Optional, Sequence

import numpy as np
import torch

from . import scene_files
from .scene_driver import Scene, SceneBatchDriver, check_supported


def png_pixels(image_hwc: np.ndarray) -> np.ndarray:
    """The 8-bit RGB pixels cv2.imwrite(path, 255 * cvtColor(img, BGR2RGB)) stores for a float32 (H, W, 3) RGB image:
    per channel clamp(rint(255 v), 0, 255) with ties to even (255 v in float32). NaN, and a value whose rounding leaves
    the int32 range (+-Inf included), store 0, as cv2's saturate_cast does after its int32 rounding overflows."""
    r = np.rint(np.float32(255) * np.asarray(image_hwc, dtype=np.float32))
    with np.errstate(invalid="ignore"):
        ok = np.abs(r) < 2.0 ** 31
    return np.where(ok, np.clip(np.where(ok, r, 0), 0, 255), 0).astype(np.uint8)


def write_png(path: str, rgb: np.ndarray) -> None:
    """An (H, W, 3) uint8 image as an 8-bit RGB PNG (zlib, no filtering)."""
    rgb = np.ascontiguousarray(rgb, dtype=np.uint8)
    h, w, c = rgb.shape
    if c != 3:
        raise ValueError("write_png takes (H, W, 3) RGB pixels")

    def chunk(kind: bytes, data: bytes) -> bytes:
        return struct.pack(">I", len(data)) + kind + data + struct.pack(">I", zlib.crc32(kind + data) & 0xFFFFFFFF)

    rows = np.concatenate([np.zeros((h, 1), np.uint8), rgb.reshape(h, w * 3)], axis=1)
    with open(path, "wb") as f:
        f.write(b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 2, 0, 0, 0)) +
                chunk(b"IDAT", zlib.compress(rows.tobytes(), 6)) + chunk(b"IEND", b""))


def parser() -> argparse.ArgumentParser:
    p = argparse.ArgumentParser(prog="python -m pixie_b200.gs_simulation", description=__doc__.split("\n\n")[0])
    p.add_argument("--model_path", type=str, required=True)
    p.add_argument("--output_path", type=str, default=None)
    p.add_argument("--config", type=str, required=True)
    p.add_argument("--save_ply", action="store_true")
    p.add_argument("--render_img", action="store_true")
    p.add_argument("--compile_video", action="store_true")
    p.add_argument("--white_bg", action="store_true")
    p.add_argument("--debug", action="store_true")
    p.add_argument("--point_cloud_path", type=str, required=True, help="material point cloud PLY (mapped_preds.ply)")
    p.add_argument("--optimization_output_path", type=str, default=None, help="directory holding E_field_epoch_XX.ply")
    p.add_argument("--replay_epoch", type=int, default=None, help="E-field epoch to replay; the latest when omitted")
    return p


def main(argv: Optional[Sequence[str]] = None, device="cuda:0") -> int:
    args = parser().parse_args(argv)
    if args.compile_video:
        raise NotImplementedError("--compile_video is not supported: encode the PNGs under <output_path>/frames with a video tool")
    if args.debug:
        raise NotImplementedError("--debug (the semantic point clouds and boundary_conditions.json) is not supported")
    if not os.path.exists(args.model_path):
        raise FileNotFoundError(f"Model path does not exist: {args.model_path}")
    if not os.path.exists(args.config):
        raise FileNotFoundError(f"Scene config does not exist: {args.config}")
    if args.render_img and args.output_path is None:
        raise ValueError("--render_img needs --output_path")
    _, _, _, pp, _ = scene_files.decode_param_json(args.config)
    name = os.path.basename(os.path.normpath(args.model_path))
    check_supported(name, pp)

    save_ply = args.save_ply and args.render_img
    sc = Scene.from_files(name, args.model_path, args.config, white_bg=args.white_bg, save_ply=save_ply, device=device)
    if not args.render_img:
        sc.camera_params = None                       # nothing is rendered
    cloud = scene_files.load_point_cloud(args.point_cloud_path, device)
    if args.optimization_output_path:
        sc.e_field = scene_files.load_optimized_e_field(args.optimization_output_path, args.replay_epoch, device)
    frames_dir = ply_dir = None
    if args.output_path is not None:
        frames_dir, ply_dir = os.path.join(args.output_path, "frames"), os.path.join(args.output_path, "ply_files")
        os.makedirs(frames_dir, exist_ok=True)
        os.makedirs(ply_dir, exist_ok=True)

    def on_image(frame: int, image: torch.Tensor):
        write_png(os.path.join(frames_dir, f"{frame:05d}.png"), png_pixels(image.permute(1, 2, 0).cpu().numpy()))

    driver = SceneBatchDriver.physics_only(device)
    driver.run_physics_simulation(sc, cloud, on_frame=lambda *a: None, on_image=on_image, ply_dir=ply_dir if save_ply else None)
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
