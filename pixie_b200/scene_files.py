"""Start a scene from the files a user has: the trained Gaussian model directory, the physics config JSON and the material
point cloud (the front of gs_simulation.py, :108-251 and :355-437, :491-531), without the reference's GaussianModel,
plyfile, Warp or its compiled rasterizer.

- `read_ply` parses a binary little-endian PLY's header and returns its first element (the reference reads
  `elements[0]`) as a numpy structured view. ascii, big-endian and list properties raise `ValueError` (plyfile would read
  them; none of the files these loaders read is written that way).
- `load_checkpoint` / `load_gaussians` decode `point_cloud/iteration_*/point_cloud.ply` on the device: the vertex table is
  read straight into a pinned buffer, copied once, and `pixie_gaussian_checkpoint_decode` produces pos, shs, opacity and
  the covariance, optionally keeping only the rows above the opacity threshold. `decode_checkpoint_ply_scale_rot` decodes
  the same table to the activated scales and normalised rotations instead, for render.py's views. The Gaussian columns must be float32
  (a stated deviation: plyfile would convert other types).
- `decode_param_json`, `generate_rotation_matrices`, `load_point_cloud`, `load_e_field_from_ply` and
  `find_e_field_epoch` restate utils/decode_param.py, utils/transformation_utils.py and gs_simulation.py.
"""
from __future__ import annotations

import ctypes as C
import json
import os
import re
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib, gs_render, particle_filling

_PLY_TYPES = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "i2", "int16": "i2", "ushort": "u2", "uint16": "u2",
              "int": "i4", "int32": "i4", "uint": "u4", "uint32": "u4", "float": "f4", "float32": "f4", "double": "f8", "float64": "f8"}


class PlyElement:
    """The first element of a PLY file: its name, row count, numpy row dtype (little-endian, packed) and where its rows
    start in the file."""

    def __init__(self, path: str, name: str, count: int, dtype: np.dtype, data_offset: int):
        self.path, self.name, self.count, self.dtype, self.data_offset = path, name, count, dtype, data_offset

    @property
    def names(self) -> List[str]:
        return list(self.dtype.names)

    def read(self) -> np.ndarray:
        """The rows as a structured array."""
        return np.fromfile(self.path, dtype=self.dtype, count=self.count, offset=self.data_offset)


def read_ply(path: str) -> PlyElement:
    """Parses the header of a binary little-endian PLY and describes its first element."""
    with open(path, "rb") as f:
        if f.readline().rstrip(b"\r\n") != b"ply":
            raise ValueError(f"{path}: not a PLY file")
        fmt, elements = None, []
        while True:
            line = f.readline()
            if not line:
                raise ValueError(f"{path}: the PLY header has no end_header")
            words = line.decode("ascii", "replace").split()
            if not words or words[0] in ("comment", "obj_info"):
                continue
            if words[0] == "end_header":
                break
            if words[0] == "format":
                fmt = words[1] if len(words) > 1 else None
            elif words[0] == "element":
                if len(words) != 3:
                    raise ValueError(f"{path}: bad element line {line!r}")
                elements.append((words[1], int(words[2]), []))
            elif words[0] == "property":
                if not elements:
                    raise ValueError(f"{path}: property before any element")
                if len(words) >= 2 and words[1] == "list":
                    raise ValueError(f"{path}: list properties are not supported")
                if len(words) != 3 or words[1] not in _PLY_TYPES:
                    raise ValueError(f"{path}: bad property line {line!r}")
                elements[-1][2].append((words[2], "<" + _PLY_TYPES[words[1]]))
            else:
                raise ValueError(f"{path}: unknown header line {line!r}")
        data_offset = f.tell()
    if fmt != "binary_little_endian":
        raise ValueError(f"{path}: only binary_little_endian PLY files are supported, this one is {fmt}")
    if not elements:
        raise ValueError(f"{path}: the PLY file has no element")
    name, count, props = elements[0]
    if len({p for p, _ in props}) != len(props):
        raise ValueError(f"{path}: duplicate property names")
    dtype = np.dtype(props)
    need = data_offset + count * dtype.itemsize
    if os.path.getsize(path) < need:
        raise ValueError(f"{path}: the file ends before its {count} {name} rows")
    return PlyElement(path, name, count, dtype, data_offset)


def _numeric_sorted(names, prefix):
    return sorted([n for n in names if n.startswith(prefix)], key=lambda x: int(x.split("_")[-1]))


def _checkpoint_columns(el: PlyElement, K: int) -> List[int]:
    """Byte offsets of x y z, f_dc_0..2, f_rest_* (numeric order), opacity, scale_*, rot* as load_ply picks them."""
    names = el.names
    rest = _numeric_sorted(names, "f_rest_")
    if len(rest) != 3 * K - 3:                     # load_ply's assert
        raise AssertionError(f"{el.path}: {len(rest)} f_rest_* properties, SH degree {int(round(K ** 0.5)) - 1} needs {3 * K - 3}")
    scale, rot = _numeric_sorted(names, "scale_"), _numeric_sorted(names, "rot")
    if len(scale) != 3 or len(rot) != 4:
        raise ValueError(f"{el.path}: a Gaussian checkpoint has 3 scale_* and 4 rot_* properties, this one {len(scale)} and {len(rot)}")
    cols = ["x", "y", "z", "f_dc_0", "f_dc_1", "f_dc_2"] + rest + ["opacity"] + scale + rot
    out = []
    for c in cols:
        if c not in el.dtype.fields:
            raise ValueError(f"{el.path}: the checkpoint has no {c!r} property")
        dt, off = el.dtype.fields[c][:2]
        if dt != np.dtype("<f4"):
            raise ValueError(f"{el.path}: property {c!r} is {dt}, the decoder reads float32 Gaussian properties only")
        out.append(off)
    return out


def _checkpoint_layout(path: str, sh_degree: int) -> Tuple[PlyElement, int, List[int]]:
    """The checkpoint's vertex element, K and column offsets; raises on a bad degree or file before any device work."""
    K = (int(sh_degree) + 1) ** 2
    if K not in (1, 4, 9, 16):
        raise ValueError(f"sh_degree must be 0..3, got {sh_degree}")
    el = read_ply(path)
    return el, K, _checkpoint_columns(el, K)


def _checkpoint_table(el: PlyElement, dev: torch.device) -> torch.Tensor:
    """The vertex rows, read straight into a pinned buffer and copied to `dev` once."""
    nbytes = el.count * el.dtype.itemsize
    host = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
    with open(el.path, "rb") as f:
        f.seek(el.data_offset)
        if nbytes and f.readinto(memoryview(host.numpy())) != nbytes:
            raise ValueError(f"{el.path}: short read")
    return host.to(dev, non_blocking=True)


def decode_checkpoint_ply(path: str, sh_degree: int = 3, opacity_threshold: Optional[float] = None, device="cuda:0") -> Dict[str, torch.Tensor]:
    """pos (M, 3), shs (M, K, 3), opacity (M, 1) and cov (M, 6) of a Gaussian checkpoint PLY, decoded on the device; with
    `opacity_threshold`, only the rows whose opacity is > float32(threshold), in file order (gs_simulation.py:405)."""
    el, K, cols = _checkpoint_layout(path, sh_degree)
    _lib.require_device()
    dev = torch.device(device)
    n, stride = el.count, el.dtype.itemsize
    pos = torch.empty((n, 3), dtype=torch.float32, device=dev)
    shs = torch.empty((n, K, 3), dtype=torch.float32, device=dev)
    opacity = torch.empty((n, 1), dtype=torch.float32, device=dev)
    cov = torch.empty((n, 6), dtype=torch.float32, device=dev)
    table = _checkpoint_table(el, dev)
    thr = 0.0 if opacity_threshold is None else float(np.float32(opacity_threshold))
    m = C.c_longlong(0)
    _lib.call("pixie_gaussian_checkpoint_decode", dev, table, n, stride, (C.c_int * len(cols))(*cols), K, int(opacity_threshold is not None),
              thr, pos, shs, opacity, cov, C.byref(m))
    table.record_stream(torch.cuda.current_stream(dev))
    M = m.value
    return {"pos": pos[:M], "shs": shs[:M], "opacity": opacity[:M], "cov": cov[:M]}


def decode_checkpoint_ply_scale_rot(path: str, sh_degree: int = 3, device="cuda:0") -> Dict[str, torch.Tensor]:
    """pos (N, 3), shs (N, K, 3), opacity (N, 1), scales (N, 3) and rotations (N, 4) of a Gaussian checkpoint PLY, decoded on
    the device as GaussianModel.load_ply then get_xyz, get_features, get_opacity (sigmoid), get_scaling (exp) and
    get_rotation (F.normalize, w x y z as stored) give them: what gaussian-splatting's render.py rasterizes. No opacity
    filter; the same pinned read and single host-to-device copy as decode_checkpoint_ply."""
    el, K, cols = _checkpoint_layout(path, sh_degree)
    _lib.require_device()
    dev = torch.device(device)
    n, stride = el.count, el.dtype.itemsize
    table = _checkpoint_table(el, dev)
    out = {"pos": torch.empty((n, 3), dtype=torch.float32, device=dev), "shs": torch.empty((n, K, 3), dtype=torch.float32, device=dev),
           "opacity": torch.empty((n, 1), dtype=torch.float32, device=dev), "scales": torch.empty((n, 3), dtype=torch.float32, device=dev),
           "rotations": torch.empty((n, 4), dtype=torch.float32, device=dev)}
    _lib.call("pixie_gaussian_checkpoint_decode_scale_rot", dev, table, n, stride, (C.c_int * len(cols))(*cols), K,
              *(out[k] for k in ("pos", "shs", "opacity", "scales", "rotations")))
    table.record_stream(torch.cuda.current_stream(dev))
    return out


def search_for_max_iteration(folder: str) -> int:
    """searchForMaxIteration (gaussian-splatting/utils/system_utils.py:26-28): the largest int(name.split("_")[-1]) over the
    folder's entries; an entry without a numeric suffix raises ValueError as it does there."""
    return max(int(name.split("_")[-1]) for name in os.listdir(folder))


def checkpoint_path(model_path: str, iteration: int = -1) -> str:
    """<model_path>/point_cloud/iteration_<it>/point_cloud.ply, the latest iteration when `iteration` is -1."""
    folder = os.path.join(model_path, "point_cloud")
    if iteration == -1:
        iteration = search_for_max_iteration(folder)
    return os.path.join(folder, f"iteration_{iteration}", "point_cloud.ply")


class GaussianCheckpoint:
    """What gs_simulation.py reads of a loaded GaussianModel: get_xyz, get_features, get_opacity, get_covariance() and the
    SH degrees."""

    def __init__(self, decoded: Dict[str, torch.Tensor], sh_degree: int):
        self._d = decoded
        self.active_sh_degree = self.max_sh_degree = int(sh_degree)

    @property
    def get_xyz(self) -> torch.Tensor:
        return self._d["pos"]

    @property
    def get_features(self) -> torch.Tensor:
        return self._d["shs"]

    @property
    def get_opacity(self) -> torch.Tensor:
        return self._d["opacity"]

    def get_covariance(self, scaling_modifier=1) -> torch.Tensor:
        if scaling_modifier != 1:
            raise ValueError("the decoded covariance is for scaling_modifier 1, as gs_simulation.py uses it")
        return self._d["cov"]


def load_checkpoint(model_path: str, sh_degree: int = 3, iteration: int = -1, device="cuda:0") -> GaussianCheckpoint:
    """gs_simulation.load_checkpoint (:215-227): the model's latest (or `iteration`'s) checkpoint, decoded on the device."""
    return GaussianCheckpoint(decode_checkpoint_ply(checkpoint_path(model_path, iteration), sh_degree, None, device), sh_degree)


def _params(d: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    return {"pos": d["pos"], "screen_points": torch.zeros_like(d["pos"]), "shs": d["shs"], "opacity": d["opacity"], "cov3D_precomp": d["cov"]}


def load_params_from_gs(gaussians: GaussianCheckpoint, threshold: Optional[float] = None) -> Dict[str, torch.Tensor]:
    """render_utils.load_params_from_gs with compute_cov3D_python (pos, screen_points, shs, opacity, cov3D_precomp); with
    `threshold`, the rows gs_simulation.py:405 keeps."""
    p = _params(gaussians._d)
    if threshold is None:
        return p
    mask = p["opacity"][:, 0] > threshold
    return {k: v[mask] for k, v in p.items()}


def load_gaussians(model_path: str, opacity_threshold: float, sh_degree: int = 3, iteration: int = -1, device="cuda:0") -> Dict[str, torch.Tensor]:
    """load_checkpoint + load_params_from_gs + the opacity filter of gs_simulation.py:403-410 in one decode on the device."""
    return _params(decode_checkpoint_ply(checkpoint_path(model_path, iteration), sh_degree, opacity_threshold, device))


# ------------------------------------------------------------------------------------------------ physics config
_ABSENT = object()
# decode_param.py:7-74: (key, default) in the order the reference inserts them; _ABSENT keys are copied only when present
_MATERIAL_KEYS = (("material", "jelly"), ("grid_lim", 2.0), ("n_grid", 50), ("nu", 0.4), ("E", 1e5), ("yield_stress", _ABSENT),
                  ("hardening", _ABSENT), ("xi", _ABSENT), ("friction_angle", _ABSENT), ("plastic_viscosity", _ABSENT), ("g", 9.8),
                  ("density", 200.0), ("rpic_damping", _ABSENT), ("pic_damping", _ABSENT), ("softening", _ABSENT),
                  ("opacity_threshold", _ABSENT), ("grid_v_damping_scale", _ABSENT))
_TIME_KEYS = (("substep_dt", 1e-4), ("frame_dt", 1e-2), ("frame_num", 100))
_PREPROCESSING_KEYS = (("nn_distance_threshold", 0.1), ("to_original_coord", True), ("z_shift_value", 0.0),
                       ("only_handle_largest_cluster", True), ("k_smoothing_neighbors", 10), ("out_of_bound_check_freq", 10),
                       ("fix_ground", True), ("opacity_threshold", 0.02), ("rotation_degree", []), ("rotation_axis", []),
                       ("sim_area", None))


def _take(src: Dict, keys) -> Dict:
    out = {}
    for k, d in keys:
        if k in src:
            out[k] = src[k]
        elif d is not _ABSENT:
            out[k] = list(d) if isinstance(d, list) else d
    return out


def decode_param_json(path: str) -> Tuple[Dict, object, Dict, Dict, Dict]:
    """utils/decode_param.decode_param_json: (material_params, bc_params, time_params, preprocessing_params,
    camera_params) with the reference's defaults, key order and errors. The camera block goes through
    gs_render.decode_camera_params, which also rejects show_hint and incomplete orbit / move_camera settings."""
    with open(path) as f:
        sim = json.load(f)
    material = _take(sim, _MATERIAL_KEYS)
    if "nu" in sim and (material["nu"] > 0.5 or material["nu"] < 0.0):
        raise ValueError("Poisson's ratio should be less than 0.5")
    if "additional_material_params" in sim:
        extra = sim["additional_material_params"]
        for p in extra:
            for k in ("point", "size", "E", "nu"):
                if k not in p:
                    raise TypeError(f"{k} is not defined")
            p.setdefault("density", material["density"])
        material["additional_material_params"] = extra
    bc = sim.get("boundary_conditions", {})
    time = _take(sim, _TIME_KEYS)
    pre = _take(sim, _PREPROCESSING_KEYS)
    pf = sim.get("particle_filling")
    pre["particle_filling"] = None if pf is None else particle_filling.decode_filling_params(pf, material)
    camera = gs_render.decode_camera_params(sim)
    return material, bc, time, pre, camera


def generate_rotation_matrices(degrees: Sequence, axes: Sequence[int], device="cuda:0") -> List[torch.Tensor]:
    """utils/transformation_utils.generate_rotation_matrices(torch.tensor(degrees), axes): float32 3x3 rotations computed
    on the CPU as the reference computes them (theta = degree / 180.0 * 3.1415926, an integer degree list staying int64
    until that division), then moved to `device`."""
    deg = torch.tensor(degrees)
    if len(deg) != len(axes):
        raise AssertionError(f"{len(deg)} rotation degrees but {len(axes)} rotation axes")
    out = []
    for d, axis in zip(deg, axes):
        theta = d / 180.0 * 3.1415926
        c, s = torch.cos(theta), torch.sin(theta)
        one, zero = torch.ones_like(c), torch.zeros_like(c)
        if axis == 0:
            rows = ((one, zero, zero), (zero, c, -s), (zero, s, c))
        elif axis == 1:
            rows = ((c, zero, s), (zero, one, zero), (-s, zero, c))
        elif axis == 2:
            rows = ((c, -s, zero), (s, c, zero), (zero, zero, one))
        else:
            raise ValueError("Invalid axis selection")
        out.append(torch.stack([torch.stack(r) for r in rows]).to(torch.float32).to(device))
    return out


# ------------------------------------------------------------------------------------------------ material cloud, E field
def _column(rows: np.ndarray, name: str, path: str) -> np.ndarray:
    if name not in rows.dtype.names:
        raise ValueError(f"{path}: no {name!r} property")
    return rows[name]


def load_point_cloud(ply_path: str, device="cuda:0") -> Dict[str, torch.Tensor]:
    """The material point cloud of gs_simulation.load_point_cloud (:108-202) as extract_material_points returns it: pos,
    density, E, nu, conf (float32; conf is ones when the file has none), material_id and part_labels (int32; part_labels
    from `part_label` when present, else material_id), on `device`."""
    rows = read_ply(ply_path).read()
    f32 = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(device)          # noqa: E731
    i32 = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)).to(device)            # noqa: E731
    pos = np.column_stack([_column(rows, c, ply_path) for c in "xyz"])
    mat = _column(rows, "material_id", ply_path)
    names = rows.dtype.names
    return {"pos": f32(pos), "density": f32(_column(rows, "density", ply_path)), "E": f32(_column(rows, "E", ply_path)),
            "nu": f32(_column(rows, "nu", ply_path)), "material_id": i32(mat),
            "part_labels": i32(rows["part_label"] if "part_label" in names else mat),
            "conf": f32(rows["conf"] if "conf" in names else np.ones(len(rows), dtype=np.float32))}


def load_e_field_from_ply(ply_file_path: str, device="cuda:0") -> torch.Tensor:
    """gs_simulation.load_e_field_from_ply (:246-250): the vertex `E` column as float32 on `device`."""
    rows = read_ply(ply_file_path).read()
    return torch.from_numpy(np.ascontiguousarray(_column(rows, "E", ply_file_path), dtype=np.float32)).to(device)


_E_FIELD = re.compile(r"E_field_epoch_(\d+)\.ply")


def find_e_field_epoch(optimization_output_path: str, replay_epoch: Optional[int] = None) -> str:
    """The E-field file of gs_simulation.py:508-526: E_field_epoch_{epoch:02d}.ply, the latest epoch when
    `replay_epoch` is None."""
    if replay_epoch is None:
        try:
            names = os.listdir(optimization_output_path)
        except FileNotFoundError:
            raise FileNotFoundError(f"Optimization output path not found: {optimization_output_path}") from None
        epochs = [int(m.group(1)) for m in map(_E_FIELD.match, names) if m]
        if not epochs:
            raise FileNotFoundError(f"No E_field_epoch_*.ply files found in {optimization_output_path}")
        replay_epoch = max(epochs)
    return os.path.join(optimization_output_path, f"E_field_epoch_{replay_epoch:02d}.ply")


def load_optimized_e_field(optimization_output_path: str, replay_epoch: Optional[int] = None, device="cuda:0") -> torch.Tensor:
    """The replayed Young's moduli, load_e_field_from_ply(...) * 1e7 (gs_simulation.py:527)."""
    return load_e_field_from_ply(find_e_field_epoch(optimization_output_path, replay_epoch), device) * 1e7
