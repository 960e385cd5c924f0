"""Score rendered dataset views on the device: gaussian-splatting's metrics.py without LPIPS.

    python -m pixie_b200.gs_metrics -m <model> [<model> ...]

For each model path, every method directory under <model>/test (sorted; the reference takes os.listdir order) is scored
pair by pair over renders/ and gt/ (sorted file names), and <model>/results.json ({method: {"SSIM", "PSNR"}}) and
<model>/per_view.json ({method: {"SSIM": {name: v}, "PSNR": {name: v}}}) are written with json.dump(..., indent=True) as
the reference writes them. Per-view values and means are float32, as the reference's torch.tensor(...) makes them:
identical images give PSNR Infinity, an empty method directory NaN means. A scene that cannot be scored is reported on
stderr with its cause and the others are still scored; the exit status is then 1 (the reference's bare except exits 0).

LPIPS is not computed: it needs the VGG-16 ImageNet weights and the LPIPS linear-layer weights, which the reference
downloads on first use. Nothing here reaches the network.

    ssim_window()              the normalised float32 11-tap window, built as loss_utils.gaussian builds it
    image_metrics(a, b)        (psnr, ssim) in fp64 of two uint8 (H, W, 3) CUDA images (one kernel launch, pixie_image_metrics)
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import math
import os
import sys
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
from PIL import Image

from . import _lib

_LPIPS_NOTE = ("LPIPS is not computed: it needs the VGG-16 ImageNet weights and the LPIPS linear-layer weights, which the "
               "reference downloads on first use.")


def ssim_window(window_size: int = 11, sigma: float = 1.5) -> torch.Tensor:
    """loss_utils.gaussian: exp(-(x - 5)^2 / (2 sigma^2)) in a float32 tensor, divided by its float32 sum."""
    gauss = torch.tensor([math.exp(-(x - window_size // 2) ** 2 / float(2 * sigma ** 2)) for x in range(window_size)], dtype=torch.float32)
    return gauss / gauss.sum()


_WINDOW = None


def image_metrics(a: torch.Tensor, b: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """(psnr, ssim) as a float64 CUDA tensor of 2, for uint8 (H, W, 3) CUDA images read as k / 255 in float32. Written to
    `out` (2 float64 on the device) when given. Stream-ordered on the current stream; no host sync."""
    global _WINDOW
    if a.dtype != torch.uint8 or b.dtype != torch.uint8:
        raise ValueError("images must be uint8")
    if a.dim() != 3 or a.shape[2] != 3 or a.shape != b.shape:
        raise ValueError(f"images must both be (H, W, 3), got {tuple(a.shape)} and {tuple(b.shape)}")
    if not (a.is_cuda and b.is_cuda) or a.device != b.device:
        raise _lib.PixieError("image_metrics requires CUDA tensors on one device; there is no CPU fallback")
    _lib.require_device()
    if _WINDOW is None:
        _WINDOW = (C.c_float * 11)(*ssim_window().tolist())
    a, b = a.contiguous(), b.contiguous()
    if out is None:
        out = torch.empty(2, dtype=torch.float64, device=a.device)
    _lib.call("pixie_image_metrics", a.device, a, b, int(a.shape[0]), int(a.shape[1]), _WINDOW, out)
    return out


def read_rgb(path: str) -> np.ndarray:
    """to_tensor(Image.open(path))[:3] as uint8 (H, W, 3): RGB, or RGBA with the alpha channel dropped."""
    with Image.open(path) as im:
        arr = np.array(im)
    if arr.ndim != 3 or arr.shape[2] not in (3, 4) or arr.dtype != np.uint8:
        raise ValueError(f"{path}: need an 8-bit RGB or RGBA image, got mode {im.mode}")
    return np.ascontiguousarray(arr[:, :, :3])


def score_method(method_dir: str, device="cuda") -> Tuple[List[str], np.ndarray, np.ndarray]:
    """(names, ssim float32 (N,), psnr float32 (N,)) of renders/ against gt/ in sorted name order."""
    renders, gts = os.path.join(method_dir, "renders"), os.path.join(method_dir, "gt")
    names = sorted(os.listdir(renders))
    res = torch.empty((len(names), 2), dtype=torch.float64, device=device)
    for i, name in enumerate(names):
        a, b = read_rgb(os.path.join(renders, name)), read_rgb(os.path.join(gts, name))
        if a.shape != b.shape:
            raise ValueError(f"{name}: render {a.shape[1]}x{a.shape[0]} and ground truth {b.shape[1]}x{b.shape[0]} differ in size")
        image_metrics(torch.from_numpy(a).to(device), torch.from_numpy(b).to(device), res[i])
    r = res.cpu().numpy()
    return names, r[:, 1].astype(np.float32), r[:, 0].astype(np.float32)


def _mean32(v: np.ndarray) -> float:
    """torch.tensor(values).mean().item() for float32 values: NaN when empty."""
    if v.size == 0:
        return float("nan")
    with np.errstate(invalid="ignore"):
        return float(np.float32(np.mean(v.astype(np.float64))))


def evaluate_scene(scene_dir: str, device="cuda") -> Dict:
    """Scores one model path and writes its results.json and per_view.json; returns the results dict."""
    full, per_view = {}, {}
    test_dir = os.path.join(scene_dir, "test")
    for method in sorted(os.listdir(test_dir)):
        names, ssims, psnrs = score_method(os.path.join(test_dir, method), device)
        full[method] = {"SSIM": _mean32(ssims), "PSNR": _mean32(psnrs)}
        per_view[method] = {"SSIM": {n: float(v) for n, v in zip(names, ssims)}, "PSNR": {n: float(v) for n, v in zip(names, psnrs)}}
        print(f"Method: {method}\n  SSIM : {full[method]['SSIM']:>12.7f}\n  PSNR : {full[method]['PSNR']:>12.7f}\n")
    with open(os.path.join(scene_dir, "results.json"), "w") as fp:
        json.dump(full, fp, indent=True)
    with open(os.path.join(scene_dir, "per_view.json"), "w") as fp:
        json.dump(per_view, fp, indent=True)
    return full


def evaluate(model_paths: Sequence[str], device="cuda") -> int:
    """Scores every model path; returns the number of scenes that could not be scored."""
    failed = 0
    for scene_dir in model_paths:
        print("Scene:", scene_dir)
        try:
            evaluate_scene(scene_dir, device)
        except Exception as e:          # one bad scene does not stop the others
            failed += 1
            print(f"Unable to compute metrics for model {scene_dir}: {type(e).__name__}: {e}", file=sys.stderr)
    return failed


def main(argv: Optional[Sequence[str]] = None) -> int:
    p = argparse.ArgumentParser(description="SSIM and PSNR of rendered test views (gaussian-splatting metrics.py). " + _LPIPS_NOTE)
    p.add_argument("--model_paths", "-m", required=True, nargs="+", type=str, default=[])
    args = p.parse_args(argv)
    return 1 if evaluate(args.model_paths) else 0


if __name__ == "__main__":
    sys.exit(main())
