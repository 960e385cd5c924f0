"""Rendering of simulated frames on the device: scene cameras, spherical-harmonic colours and a tile-based Gaussian
rasterizer (gs_simulation.py:573-631 with `--render_img`; the reference calls Inria's diff-gaussian-rasterization).

    rasterize(means3D, cov3D, opacity, camera, bg, shs=None, sh_degree=0, colors=None) -> (image (3, H, W), radii (N,))
    rasterize_scale_rot(means3D, scales, rotations, opacity, camera, bg, shs, sh_degree)  the same frame from scales and
                                                                           rotations, as render.py's views are drawn
    get_camera_view(cameras, default_camera_index, ...)                    utils/camera_view_utils.py:164-268
    get_center_view_worldspace_and_observant_coordinate(...)               utils/transformation_utils.py:143-166
    decode_camera_params(sim_params)                                       utils/decode_param.py:212-270

The camera arithmetic runs in float64 numpy and is cast to float32 where the reference casts (getWorld2View2 returns
float32, the projection matrix is a float32 tensor); the view centre is computed in float64 where the reference
computes it in float32. Colours from `shs` are evaluated toward the camera centre inside the rasterizer's preprocess
kernel as convert_SH (utils/render_utils.py:113-130) does: +0.5, clamped at 0. The image is RGB, float32, unclamped.
The forward pass only; no CPU fallback. Work runs on the current stream of the tensors' device. One renderer per
device serves every call: a frame waits on the device for the previous one, whatever stream either is drawn on, and
calls from several host threads take turns.
"""
from __future__ import annotations

import ctypes as C
import json
import math
import os
import threading
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from . import _lib

ZNEAR, ZFAR = 0.01, 100.0


@dataclass
class Camera:
    """What the rasterizer reads from the reference's `scene.cameras.Camera`: float32 CPU tensors, matrices stored
    transposed (row-vector convention) as the reference stores them."""
    image_width: int
    image_height: int
    FoVx: float
    FoVy: float
    world_view_transform: torch.Tensor   # (4, 4)
    projection_matrix: torch.Tensor      # (4, 4)
    full_proj_transform: torch.Tensor    # (4, 4) = world_view_transform @ projection_matrix
    camera_center: torch.Tensor          # (3,)


# ------------------------------------------------------------------------------------------------ camera
def focal2fov(focal: float, pixels: float) -> float:
    return 2 * math.atan(pixels / (2 * focal))


def get_world2view2(R: np.ndarray, t: np.ndarray) -> np.ndarray:
    """getWorld2View2 with translate 0 and scale 1: [R^T | t] as float32 (the inverse-of-inverse round trip in float64)."""
    Rt = np.zeros((4, 4))
    Rt[:3, :3] = np.asarray(R, dtype=np.float64).T
    Rt[:3, 3] = t
    Rt[3, 3] = 1.0
    C2W = np.linalg.inv(Rt)
    return np.float32(np.linalg.inv(C2W))


def get_projection_matrix(znear: float, zfar: float, fovX: float, fovY: float) -> np.ndarray:
    """getProjectionMatrix: the symmetric perspective matrix (z to [0, 1]), float32."""
    top = math.tan(fovY / 2) * znear
    right = math.tan(fovX / 2) * znear
    P = np.zeros((4, 4), dtype=np.float32)
    P[0, 0] = 2.0 * znear / (right + right)
    P[1, 1] = 2.0 * znear / (top + top)
    P[3, 2] = 1.0
    P[2, 2] = zfar / (zfar - znear)
    P[2, 3] = -(zfar * znear) / (zfar - znear)
    return P


def make_camera(R: np.ndarray, T: np.ndarray, FoVx: float, FoVy: float, width: int, height: int) -> Camera:
    """scene.cameras.Camera with znear 0.01, zfar 100, trans 0, scale 1."""
    wv = torch.from_numpy(get_world2view2(R, T)).t().contiguous()
    proj = torch.from_numpy(get_projection_matrix(ZNEAR, ZFAR, FoVx, FoVy)).t().contiguous()
    full = wv @ proj
    center = torch.linalg.inv(wv)[3, :3].contiguous()
    return Camera(int(width), int(height), float(FoVx), float(FoVy), wv, proj, full, center)


def _rodrigues_rotation(axis: np.ndarray, angle_deg: float) -> np.ndarray:
    axis = axis / np.linalg.norm(axis)
    a = np.deg2rad(angle_deg)
    c, s = np.cos(a), np.sin(a)
    t = 1 - c
    x, y, z = axis
    return np.array([[t * x * x + c, t * x * y - s * z, t * x * z + s * y],
                     [t * x * y + s * z, t * y * y + c, t * y * z - s * x],
                     [t * x * z - s * y, t * y * z + s * x, t * z * z + c]])


def _camera_rotation(camera_to_object: np.ndarray, object_vertical_downward: np.ndarray) -> np.ndarray:
    """Columns: right, down (the vertical projected off the viewing axis), forward."""
    f = camera_to_object / np.linalg.norm(camera_to_object)
    down = object_vertical_downward - np.dot(object_vertical_downward, f) * f
    down = down / np.linalg.norm(down)
    return np.column_stack((np.cross(down, f), down, f))


def _local_coord(vertical: np.ndarray):
    vertical = vertical / np.linalg.norm(vertical)
    h1 = np.array([1, 1, 1])
    if np.abs(np.dot(h1, vertical)) < 0.01:
        h1 = np.array([0.72, 0.37, -0.67])
    h1 = h1 - np.dot(h1, vertical) * vertical
    h1 = h1 / np.linalg.norm(h1)
    return vertical, h1, np.cross(h1, vertical)


def orbit_camera_pose(azimuth, elevation, radius, roll, view_center, observant_coordinates):
    """get_camera_position_and_rotation: position on the sphere around `view_center` (degrees; azimuth 0 along the first
    observant axis) and the camera rotation looking at the centre, rolled about the viewing axis."""
    az, el = azimuth / 180.0 * np.pi, elevation / 180.0 * np.pi
    canonical = np.array([np.cos(az) * np.cos(el), np.sin(az) * np.cos(el), np.sin(el)]) * radius
    position = view_center + observant_coordinates @ canonical
    R_base = _camera_rotation(view_center - position, -observant_coordinates[:, 2])
    R = _rodrigues_rotation(R_base[:, 2], 0.0 if roll is None else roll) @ R_base
    return position, R


def get_center_view_worldspace_and_observant_coordinate(mpm_space_viewpoint_center, mpm_space_vertical_upward_axis,
                                                        rotation_matrices, scale_origin, original_mean_pos):
    """The view centre and the (h1, h2, vertical) basis in the Gaussians' frame. Like the reference, the shift to the
    simulation box is undone with z_shift 0, whatever the scene's z_shift_value."""
    rots = [np.asarray(torch.as_tensor(R).detach().cpu(), dtype=np.float64) for R in rotation_matrices]
    scale = float(torch.as_tensor(scale_origin).detach().cpu())
    mean = np.asarray(torch.as_tensor(original_mean_pos).detach().cpu(), dtype=np.float64).reshape(3)

    def undo(p):
        p = mean + (np.asarray(p, dtype=np.float64).reshape(3) - 1.0) / scale
        for R in reversed(rots):
            p = p @ R
        return p

    center = np.asarray(mpm_space_viewpoint_center, dtype=np.float64).reshape(3)
    up = np.asarray(mpm_space_vertical_upward_axis, dtype=np.float64).reshape(3)
    c_world = undo(center)
    vertical, h1, h2 = _local_coord(undo(up + center) - c_world)
    return c_world, np.column_stack((h1, h2, vertical))


def load_cameras(cameras: Union[str, Sequence[Dict]]) -> List[Dict]:
    """The cameras.json list, from the list itself, the file, or the model directory holding it."""
    if isinstance(cameras, (str, os.PathLike)):
        path = os.path.join(cameras, "cameras.json") if os.path.isdir(cameras) else cameras
        with open(path) as f:
            cameras = json.load(f)
    cams = list(cameras)
    if not cams:
        raise ValueError("the camera list is empty")
    return cams


def get_camera_view(cameras: Union[str, Sequence[Dict]], default_camera_index: int = 0, center_view_world_space=None,
                    observant_coordinates=None, show_hint: bool = False, init_azimuthm=None, init_elevation=None, init_radius=None,
                    init_roll=None, move_camera: bool = False, current_frame: int = 0, delta_a=0, delta_e=0, delta_r=0,
                    delta_roll=0) -> Camera:
    """camera_view_utils.get_camera_view: camera `default_camera_index` of the list, or at -1 the orbit camera
    (init_* + current_frame * delta_* when move_camera) with the first camera's image size and focal lengths."""
    return make_camera(*camera_pose(cameras, default_camera_index, center_view_world_space, observant_coordinates, show_hint,
                                    init_azimuthm, init_elevation, init_radius, init_roll, move_camera, current_frame, delta_a,
                                    delta_e, delta_r, delta_roll))


def camera_pose(cameras, default_camera_index=0, center_view_world_space=None, observant_coordinates=None, show_hint=False,
                init_azimuthm=None, init_elevation=None, init_radius=None, init_roll=None, move_camera=False, current_frame=0,
                delta_a=0, delta_e=0, delta_r=0, delta_roll=0):
    """The float64 (R, T, FoVx, FoVy, width, height) get_camera_view hands to the reference's Camera."""
    if show_hint:
        raise ValueError("show_hint prints the default camera's orbit coordinates and exits the reference program; "
                         "it is not a rendering mode. Set init_azimuthm / init_elevation / init_radius instead")
    cams = load_cameras(cameras)
    idx = int(default_camera_index)
    if idx >= len(cams):
        raise ValueError(f"default_camera_index {idx} is out of range for {len(cams)} cameras")
    if idx > -1:
        raw = cams[idx]
        rotation, position = raw["rotation"], raw["position"]
    else:
        raw = cams[0]
        if init_azimuthm is None or init_elevation is None or init_radius is None:
            raise ValueError("default_camera_index -1 needs init_azimuthm, init_elevation and init_radius")
        if center_view_world_space is None or observant_coordinates is None:
            raise ValueError("default_camera_index -1 needs center_view_world_space and observant_coordinates")
        roll = 0.0 if init_roll is None else init_roll
        a, e, r = init_azimuthm, init_elevation, init_radius
        if move_camera:
            if delta_a is None or delta_e is None or delta_r is None or delta_roll is None:
                raise ValueError("move_camera needs delta_a, delta_e and delta_r")
            a, e, r, roll = a + current_frame * delta_a, e + current_frame * delta_e, r + current_frame * delta_r, \
                roll + current_frame * delta_roll
        position, rotation = orbit_camera_pose(a, e, r, roll, np.asarray(center_view_world_space, dtype=np.float64),
                                               np.asarray(observant_coordinates, dtype=np.float64))
    tmp = np.zeros((4, 4))
    tmp[:3, :3] = np.asarray(rotation, dtype=np.float64)
    tmp[:3, 3] = np.asarray(position, dtype=np.float64)
    tmp[3, 3] = 1
    C2W = np.linalg.inv(tmp)
    width, height = int(raw["width"]), int(raw["height"])
    return C2W[:3, :3].transpose(), C2W[:3, 3], focal2fov(raw["fx"], width), focal2fov(raw["fy"], height), width, height


_CAMERA_DEFAULTS = {"mpm_space_viewpoint_center": [1.0, 1.0, 1.0], "mpm_space_vertical_upward_axis": [0, 0, 1],
                    "default_camera_index": 0, "show_hint": False, "init_azimuthm": None, "init_elevation": None,
                    "init_radius": None, "delta_a": None, "delta_e": None, "delta_r": None, "move_camera": False,
                    "init_roll": 0.0, "delta_roll": 0.0}


def decode_camera_params(sim_params: Dict) -> Dict:
    """The camera block of decode_param_json (decode_param.py:212-270): its keys with the reference's defaults. Raises
    on show_hint, which exits the reference program instead of rendering."""
    if not isinstance(sim_params, dict):
        raise TypeError(f"camera parameters must be a dict, got {type(sim_params).__name__}")
    p = {k: sim_params.get(k, d) for k, d in _CAMERA_DEFAULTS.items()}
    if p["show_hint"]:
        raise ValueError("show_hint prints the default camera's orbit coordinates and exits the reference program; "
                         "it is not a rendering mode. Set init_azimuthm / init_elevation / init_radius instead")
    for k in ("mpm_space_viewpoint_center", "mpm_space_vertical_upward_axis"):
        if np.asarray(p[k]).shape != (3,):
            raise ValueError(f"{k} must hold 3 numbers, got {p[k]!r}")
    if int(p["default_camera_index"]) < 0 and None in (p["init_azimuthm"], p["init_elevation"], p["init_radius"]):
        raise ValueError("default_camera_index -1 (the orbit camera) needs init_azimuthm, init_elevation and init_radius")
    if p["move_camera"] and None in (p["delta_a"], p["delta_e"], p["delta_r"]):
        raise ValueError("move_camera needs delta_a, delta_e and delta_r")
    return p


# ------------------------------------------------------------------------------------------------ rasterizer
_RENDERERS: Dict[int, "_Renderer"] = {}
_RENDERERS_LOCK = threading.Lock()


class _Renderer:
    """One device's renderer handle; its buffers grow to the largest frame seen and are reused. Its host-side state
    (capacities, the pinned pair-count word) is guarded by `lock`."""

    def __init__(self, device: torch.device):
        lib = _lib.require_device()
        h = C.c_void_p()
        with torch.cuda.device(device):
            _lib.check(lib.pixie_gs_renderer_create(C.byref(h)))
        self.h, self.lib = h, lib
        self.lock = threading.Lock()

    def __del__(self):
        if getattr(self, "h", None) and self.h.value:
            self.lib.pixie_gs_renderer_destroy(self.h)


def _renderer(device: torch.device) -> _Renderer:
    idx = device.index if device.index is not None else torch.cuda.current_device()
    with _RENDERERS_LOCK:
        if idx not in _RENDERERS:
            _RENDERERS[idx] = _Renderer(torch.device("cuda", idx))
        return _RENDERERS[idx]


def _f32(values, n: int, name: str):
    v = torch.as_tensor(values, dtype=torch.float32).detach().cpu().reshape(-1)
    if v.numel() != n:
        raise ValueError(f"{name} must hold {n} values, got {v.numel()}")
    return (C.c_float * n)(*v.tolist())


def _rasterize(means3D, cov3D, opacity, camera: Camera, bg, shs=None, sh_degree: int = 0, colors=None,
               phase_ms: Optional[list] = None) -> Tuple[torch.Tensor, torch.Tensor, int]:
    if means3D.dim() != 2 or means3D.shape[1] != 3:
        raise ValueError(f"means3D must be (N, 3), got {tuple(means3D.shape)}")
    n = means3D.shape[0]
    if tuple(cov3D.shape) != (n, 6):
        raise ValueError(f"cov3D must be (N, 6) = ({n}, 6), got {tuple(cov3D.shape)}")
    if not (tuple(opacity.shape) == (n,) or tuple(opacity.shape) == (n, 1)):
        raise ValueError(f"opacity must be (N,) or (N, 1) for N = {n}, got {tuple(opacity.shape)}")
    if (shs is None) == (colors is None):
        raise ValueError("give exactly one of shs and colors")
    if shs is not None:
        if int(sh_degree) not in (0, 1, 2, 3):
            raise ValueError(f"sh_degree must be 0..3, got {sh_degree}")
        if shs.dim() != 3 or shs.shape[0] != n or shs.shape[2] != 3 or shs.shape[1] < (int(sh_degree) + 1) ** 2:
            raise ValueError(f"shs must be (N, K, 3) with K >= (sh_degree + 1)^2 = {(int(sh_degree) + 1) ** 2}, got {tuple(shs.shape)}")
    elif tuple(colors.shape) != (n, 3):
        raise ValueError(f"colors must be (N, 3) = ({n}, 3), got {tuple(colors.shape)}")
    W, H = int(camera.image_width), int(camera.image_height)
    if W < 1 or H < 1:
        raise ValueError(f"camera image size must be positive, got {W} x {H}")
    tensors = [means3D, cov3D, opacity, shs if shs is not None else colors]
    if not all(t.is_cuda for t in tensors):
        raise _lib.PixieError("rasterize requires CUDA tensors; there is no CPU fallback")
    dev = means3D.device
    if any(t.device != dev for t in tensors):
        raise ValueError("means3D, cov3D, opacity and shs / colors must be on one device")
    if any(t.dtype != torch.float32 for t in tensors):
        raise ValueError("means3D, cov3D, opacity and shs / colors must be float32")
    m, c, o = means3D.detach().contiguous(), cov3D.detach().contiguous(), opacity.detach().reshape(-1).contiguous()
    s = shs.detach().contiguous() if shs is not None else None
    col = colors.detach().contiguous() if colors is not None else None
    view = _f32(camera.world_view_transform, 16, "world_view_transform")
    proj = _f32(camera.full_proj_transform, 16, "full_proj_transform")
    campos = _f32(camera.camera_center, 3, "camera_center")
    bgc = _f32(bg, 3, "bg")
    r = _renderer(dev)
    n_rendered = C.c_int(0)
    ms = (C.c_float * 5)() if phase_ms is not None else None
    with torch.cuda.device(dev), r.lock:
        image = torch.empty((3, H, W), dtype=torch.float32, device=dev)
        radii = torch.empty((n,), dtype=torch.int32, device=dev)
        _lib.check(r.lib.pixie_gs_render(
            r.h, C.c_void_p(m.data_ptr()), C.c_void_p(c.data_ptr()), C.c_void_p(o.data_ptr()),
            C.c_void_p(s.data_ptr() if s is not None else None), int(s.shape[1]) if s is not None else 0, int(sh_degree),
            C.c_void_p(col.data_ptr() if col is not None else None), n, view, proj, campos,
            math.tan(camera.FoVx * 0.5), math.tan(camera.FoVy * 0.5), W, H, bgc, C.c_void_p(image.data_ptr()),
            C.c_void_p(radii.data_ptr()), C.byref(n_rendered), ms, C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
    if phase_ms is not None:
        phase_ms[:] = list(ms)
    return image, radii, n_rendered.value


def rasterize(means3D: torch.Tensor, cov3D: torch.Tensor, opacity: torch.Tensor, camera: Camera, bg,
              shs: Optional[torch.Tensor] = None, sh_degree: int = 0, colors: Optional[torch.Tensor] = None
              ) -> Tuple[torch.Tensor, torch.Tensor]:
    """One frame: (image (3, H, W) float32 RGB, unclamped; radii (N,) int32, 0 where culled). means3D (N, 3), cov3D (N, 6)
    upper-triangular (xx, xy, xz, yy, yz, zz), opacity (N,) or (N, 1), all float32 CUDA tensors; colours from shs
    (N, (D+1)^2 or more, 3) at degree sh_degree <= 3 toward the camera centre, or from colors (N, 3) as given; bg: 3 values."""
    image, radii, _ = _rasterize(means3D, cov3D, opacity, camera, bg, shs, sh_degree, colors)
    return image, radii


def _rasterize_scale_rot(means3D, scales, rotations, opacity, camera: Camera, bg, shs, sh_degree: int,
                         phase_ms: Optional[list] = None) -> Tuple[torch.Tensor, torch.Tensor, int]:
    if means3D.dim() != 2 or means3D.shape[1] != 3:
        raise ValueError(f"means3D must be (N, 3), got {tuple(means3D.shape)}")
    n = means3D.shape[0]
    if tuple(scales.shape) != (n, 3):
        raise ValueError(f"scales must be (N, 3) = ({n}, 3), got {tuple(scales.shape)}")
    if tuple(rotations.shape) != (n, 4):
        raise ValueError(f"rotations must be (N, 4) = ({n}, 4), got {tuple(rotations.shape)}")
    if not (tuple(opacity.shape) == (n,) or tuple(opacity.shape) == (n, 1)):
        raise ValueError(f"opacity must be (N,) or (N, 1) for N = {n}, got {tuple(opacity.shape)}")
    if int(sh_degree) not in (0, 1, 2, 3):
        raise ValueError(f"sh_degree must be 0..3, got {sh_degree}")
    if shs.dim() != 3 or shs.shape[0] != n or shs.shape[2] != 3 or shs.shape[1] < (int(sh_degree) + 1) ** 2:
        raise ValueError(f"shs must be (N, K, 3) with K >= (sh_degree + 1)^2 = {(int(sh_degree) + 1) ** 2}, got {tuple(shs.shape)}")
    W, H = int(camera.image_width), int(camera.image_height)
    if W < 1 or H < 1:
        raise ValueError(f"camera image size must be positive, got {W} x {H}")
    tensors = [means3D, scales, rotations, opacity, shs]
    if not all(t.is_cuda for t in tensors):
        raise _lib.PixieError("rasterize_scale_rot requires CUDA tensors; there is no CPU fallback")
    dev = means3D.device
    if any(t.device != dev for t in tensors):
        raise ValueError("means3D, scales, rotations, opacity and shs must be on one device")
    if any(t.dtype != torch.float32 for t in tensors):
        raise ValueError("means3D, scales, rotations, opacity and shs must be float32")
    m, sc, rot, s = (t.detach().contiguous() for t in (means3D, scales, rotations, shs))
    o = opacity.detach().reshape(-1).contiguous()
    view = _f32(camera.world_view_transform, 16, "world_view_transform")
    proj = _f32(camera.full_proj_transform, 16, "full_proj_transform")
    campos = _f32(camera.camera_center, 3, "camera_center")
    bgc = _f32(bg, 3, "bg")
    r = _renderer(dev)
    n_rendered = C.c_int(0)
    ms = (C.c_float * 5)() if phase_ms is not None else None
    with torch.cuda.device(dev), r.lock:
        image = torch.empty((3, H, W), dtype=torch.float32, device=dev)
        radii = torch.empty((n,), dtype=torch.int32, device=dev)
        _lib.check(r.lib.pixie_gs_render_scale_rot(
            r.h, C.c_void_p(m.data_ptr()), C.c_void_p(sc.data_ptr()), C.c_void_p(rot.data_ptr()), C.c_void_p(o.data_ptr()),
            C.c_void_p(s.data_ptr()), int(s.shape[1]), int(sh_degree), n, view, proj, campos,
            math.tan(camera.FoVx * 0.5), math.tan(camera.FoVy * 0.5), W, H, bgc, C.c_void_p(image.data_ptr()),
            C.c_void_p(radii.data_ptr()), C.byref(n_rendered), ms, C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
    if phase_ms is not None:
        phase_ms[:] = list(ms)
    return image, radii, n_rendered.value


def rasterize_scale_rot(means3D: torch.Tensor, scales: torch.Tensor, rotations: torch.Tensor, opacity: torch.Tensor, camera: Camera,
                        bg, shs: torch.Tensor, sh_degree: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """One frame as gaussian_renderer.render draws it with PipelineParams' defaults (gaussian-splatting's render.py):
    (image (3, H, W) float32 RGB, unclamped; radii (N,) int32). The covariance is built in the rasterizer's preprocess from
    scales (N, 3) and rotations (N, 4) (unit quaternions w x y z) as forward.cu's computeCov3D builds it at scale_modifier
    1; colours from shs (N, (D+1)^2 or more, 3) at degree sh_degree as its computeColorFromSH evaluates them. All float32
    CUDA tensors; opacity (N,) or (N, 1); bg: 3 values."""
    image, radii, _ = _rasterize_scale_rot(means3D, scales, rotations, opacity, camera, bg, shs, sh_degree)
    return image, radii
