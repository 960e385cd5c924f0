"""Voxel-grid producer I/O (SURVEY.md 8f-3): feed `clip_features_features.npy` to the U-Net without the reference's
fp16 -> fp32 -> permute -> H2D detour.

The file `voxelize.extract_clip_voxel_grid` writes (pixie/voxel/voxelize.py:86,111) is float16 (D, D, D, C) with X slowest — already
the channels-last layout the convolution kernels read through TMA. The reference dataset (`MaterialVoxelDataset.__getitem__`,
WG/data_utils/my_data.py:160-224) loads it, converts to float32 and permutes to (C, D, H, W) — 805 MB per scene at 64^3 x 768 —
before the H2D copy. Here the file is memory-mapped and copied once into a (reused) pinned buffer; `MaterialFieldPredictor.
predict_packed_host_stream` moves it to the device while the previous scene is still in the networks.
"""
from __future__ import annotations

import os
from typing import Iterable, Iterator, Optional, Sequence, Tuple

import numpy as np
import torch

FEATURE_FILE = "clip_features_features.npy"
MASK_FILE = "clip_features_mask.npy"


def open_feature_grid(path: str) -> np.memmap:
    """Memory-maps a feature grid and checks that it is the (D, D, D, C) float16 array voxelize.py writes."""
    a = np.load(path, mmap_mode="r")
    if a.dtype != np.float16:
        raise TypeError(f"{path}: expected float16 features (voxelize.py:86), got {a.dtype}")
    if a.ndim != 4 or not (a.shape[0] == a.shape[1] == a.shape[2]):
        raise ValueError(f"{path}: expected (D, D, D, C), got {a.shape}")
    return a


def load_feature_grid(path: str, out: Optional[torch.Tensor] = None, pin: Optional[bool] = None) -> torch.Tensor:
    """(1, D, D, D, C) float16 host tensor (pinned when CUDA is available, unless `pin` says otherwise), ready for
    `predict_packed_host[_stream]`. `out` re-uses a buffer of the right shape."""
    a = open_feature_grid(path)
    shape = (1,) + tuple(a.shape)
    if out is None:
        out = torch.empty(shape, dtype=torch.float16)
        if pin if pin is not None else torch.cuda.is_available():
            out = out.pin_memory()
    elif tuple(out.shape) != shape or out.dtype != torch.float16:
        raise ValueError(f"out must be float16 {shape}, got {out.dtype} {tuple(out.shape)}")
    np.copyto(out.numpy()[0], a)          # one pass over the mapped file, no fp32 intermediate
    return out


def load_mask(path: str) -> torch.Tensor:
    """clip_features_mask.npy as float32 (D, D, D), as `_load_clip_features_mask` returns it (my_data.py:147-153)."""
    if not os.path.exists(path):
        raise FileNotFoundError(f"clip_features_mask.npy not found at {path}. Please run voxelization first.")
    return torch.from_numpy(np.load(path).astype(np.float32))


def load_grid_metadata(npz_path: str) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """(min_bounds, max_bounds, grid_shape) of clip_features.npz, as map_pred_to_coords.py:146-150 reads them: the
    bounds a Scene needs to place its predicted material field."""
    with np.load(npz_path) as metadata:
        return metadata["min_bounds"], metadata["max_bounds"], metadata["grid_shape"]


class SceneGrid:
    """One scene of `scene_stream`: `.dir`, the pinned `.tensor`, and `.h2d_done` — the CUDA event after which the pinned
    buffer may be rewritten (set by the consumer, e.g. MaterialFieldPredictor.predict_packed_host_stream)."""
    __slots__ = ("dir", "tensor", "h2d_done")

    def __init__(self, d: str, tensor: torch.Tensor):
        self.dir, self.tensor, self.h2d_done = d, tensor, None

    def __iter__(self):              # unpacks as (scene_dir, grid)
        return iter((self.dir, self.tensor))


def scene_stream(scene_dirs: Sequence[str], n_buffers: int = 3) -> Iterator[SceneGrid]:
    """Yields a SceneGrid for every scene, cycling through `n_buffers` pinned host buffers. Before a buffer is rewritten the
    generator waits for the `h2d_done` event of the scene that used it last, so a consumer that copies asynchronously only has
    to record that event (it must have finished with a scene's buffer by other means if it leaves `h2d_done` unset). Meant to
    be consumed lazily — `predict_packed_host_stream(scene_stream(dirs))` — so that at most `n_buffers` scenes are in flight."""
    bufs = [None] * n_buffers
    last = [None] * n_buffers
    for i, d in enumerate(scene_dirs):
        path = os.path.join(d, FEATURE_FILE)
        slot = i % n_buffers
        if last[slot] is not None and last[slot].h2d_done is not None:
            last[slot].h2d_done.synchronize()               # the device has read the previous content of this buffer
        try:
            bufs[slot] = load_feature_grid(path, out=bufs[slot])
        except ValueError:
            bufs[slot] = load_feature_grid(path)           # grid shape changed between scenes
        last[slot] = SceneGrid(d, bufs[slot])
        yield last[slot]
