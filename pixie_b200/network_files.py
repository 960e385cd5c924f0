"""The file side of the material networks: what the reference's neural mode reads and writes around the U-Net forward, so
that a user goes from checkpoints and labelled grids to predictions, metrics and the material point cloud without the
reference's Hydra config, WG tree, plyfile or model classes.

- `load_network_checkpoint`, `load_normalization_ranges`: training_utils.load_checkpoint's state-dict extraction and the
  p1 / p99 keys of normalization_ranges.yaml.
- `MaterialVoxelDataset`, `load_test_dataset`: the file discovery of WG/data_utils/my_data.py:29-132 and the test split of
  inference_combined.py:48-78.
- `material_metrics`, `batch_metrics`, `InferenceMetrics`, `generate_metrics_report`, `save_predictions`: process_batch
  (inference_combined.py:108-217) and pixie/metrics.py:105-416. The per-voxel work is one device pass
  (csrc/material_metrics.cu); the float32 scalar arithmetic after it is replayed on the host with torch as the reference
  writes it.
- `write_material_point_cloud`, `map_pred_to_ply`, `transform_nerf_to_world`: pixie/voxel/map_pred_to_coords.py:77-283 on
  top of `material_transfer.extract_material_points`, writing the bytes plyfile writes.
"""
from __future__ import annotations

import ctypes as C
import json
import logging
import math
import os
from collections import defaultdict
from pathlib import Path
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib, scene_files, voxel_io

log = logging.getLogger("pixie_b200.network_files")


# --------------------------------------------------------------------------------------------------- checkpoints, ranges
def load_network_checkpoint(path: Optional[str]):
    """The state dict of a `.pth` checkpoint, unwrapped as training_utils.load_checkpoint does (`model_state_dict`, then
    `state_dict`, then the object itself), loaded on the CPU with weights_only=True. A missing file returns None: the
    reference then silently evaluates an untrained network, so this logs an error."""
    if not path or not os.path.isfile(path):
        log.error("checkpoint %r does not exist; the reference would evaluate an untrained network", path)
        return None
    ckpt = torch.load(path, map_location="cpu", weights_only=True)
    if isinstance(ckpt, dict):
        for key in ("model_state_dict", "state_dict"):
            if key in ckpt:
                return ckpt[key]
    return ckpt


def load_normalization_ranges(path: str) -> Dict[str, float]:
    """normalization_ranges.yaml -> the `ranges` dict extract_material_points takes (training_utils.py:21-47)."""
    import yaml
    if not os.path.exists(path):
        raise FileNotFoundError(f"Normalization ranges file not found at {path}.")
    with open(path) as f:
        r = yaml.safe_load(f)
    return {"density_min": r["density_p1"], "density_max": r["density_p99"], "E_min": r["E_p1"], "E_max": r["E_p99"],
            "nu_min": r["nu_p1"], "nu_max": r["nu_p99"]}


def _load_json(path):
    with open(path) as f:
        return json.load(f)


def _save_json(data, path):
    with open(path, "w") as f:
        json.dump(data, f, indent=2)


# -------------------------------------------------------------------------------------------------------- dataset, split
class MaterialVoxelDataset:
    """The labelled scenes under `render_outputs_dir`, discovered as MaterialVoxelDataset._collect_files does (my_data.py:
    61-132, feature_type "clip", no class filter): `os.listdir` order; objects named in `problematic_objects` (a JSON list,
    normalization_stats_dir/problematic_objects.json) are skipped, and so are objects without features or labels, with
    material ids outside [0, num_material_classes) or with shapes other than (D, D, D, C_mat) / (D, D, D, C_feat)."""

    def __init__(self, render_outputs_dir: str, sample_id: int = 0, grid_size: int = 64, feature_channels: int = 768,
                 in_material_channels: int = 4, num_material_classes: int = 8, background_id: int = 7,
                 problematic_objects: Optional[str] = None, enforce_mask_consistency: bool = True):
        self.root, self.sample_id, self.D = render_outputs_dir, sample_id, grid_size
        self.C_feat, self.C_mat, self.n_classes = feature_channels, in_material_channels, num_material_classes
        self.background_id, self.enforce_mask_consistency = background_id, enforce_mask_consistency
        self.problematic_objects = set()
        if problematic_objects and os.path.exists(problematic_objects):
            self.problematic_objects = set(_load_json(problematic_objects))
            log.warning(f"Loaded {len(self.problematic_objects)} problematic objects to skip")
        self.data_files, self.feature_files, self.mask_files, self.obj_ids = self._collect_files()
        log.info(f"[DATASET] Loaded {len(self.data_files)} data files.")

    def _collect_files(self):
        data_files, feat_files, mask_files, obj_ids = [], [], [], []
        D = self.D
        for obj_id in os.listdir(self.root):
            if obj_id in self.problematic_objects:
                log.warning(f"Skipping {obj_id} because it is in the problematic objects list")
                continue
            feat_fp = f"{self.root}/{obj_id}/clip_features_features.npy"
            mat_fp = f"{self.root}/{obj_id}/sample_{self.sample_id}/material_grid.npy"
            mask_fp = f"{self.root}/{obj_id}/clip_features_mask.npy"
            if not os.path.exists(feat_fp):
                log.warning(f"Skipping {obj_id} because {feat_fp} does not exist")
                continue
            if not os.path.exists(mat_fp):
                log.warning(f"Skipping {obj_id} because {mat_fp} does not exist")
                continue
            try:
                mat_chn = np.load(mat_fp, mmap_mode="r")[..., -1]
                max_id, min_id = mat_chn.max(), mat_chn.min()
                if not (0 <= min_id < self.n_classes) or max_id >= self.n_classes:
                    log.warning(f"[Data warning] Skipping {obj_id}: material_id outside valid range Your range: (min {min_id}, max {max_id}). "
                                f"Valid range: (0, {self.n_classes - 1})")
                    continue
            except Exception as e:                                                      # noqa: BLE001
                log.warning(f"[Data warning] Could not validate material_id for {obj_id}: {e}. Skipping.")
                continue
            mat_shape = np.load(mat_fp, mmap_mode="r").shape
            feat_shape = np.load(feat_fp, mmap_mode="r").shape
            if len(feat_shape) == 3:
                feat_shape = (D, D, D, 1)
            if not (mat_shape == (D, D, D, self.C_mat) and feat_shape == (D, D, D, self.C_feat)):
                log.warning(f"[Data warning] Skipping {obj_id}: mat_shape: {mat_shape} != ({D, D, D, self.C_mat}) or feat_shape: "
                            f"{feat_shape} != ({D, D, D, self.C_feat})")
                continue
            data_files.append(mat_fp)
            feat_files.append(feat_fp)
            mask_files.append(mask_fp)
            obj_ids.append(obj_id)
        return data_files, feat_files, mask_files, obj_ids

    def __len__(self):
        return len(self.data_files)

    def info(self, idx: int) -> Dict[str, str]:
        """The `info` dict save_predictions stores (sample_id as the string it writes)."""
        return {"obj_id": self.obj_ids[idx], "sample_id": str(self.sample_id), "data_path": self.data_files[idx],
                "feature_path": self.feature_files[idx], "mask_path": self.mask_files[idx]}

    def load_labels(self, idx: int) -> Tuple[np.ndarray, np.ndarray]:
        """(raw material grid (D, D, D, C_mat) float32, mask (D, D, D) float32), with __getitem__'s mask-consistency assert."""
        mat = np.load(self.data_files[idx]).astype(np.float32)
        mask = voxel_io.load_mask(self.mask_files[idx]).numpy()
        if self.enforce_mask_consistency:
            expected = (mat[..., -1] != self.background_id).astype(np.float32)
            assert np.array_equal(mask, expected), \
                f"Mask inconsistency for {self.obj_ids[idx]}: clip_features_mask.npy doesn't match material_id-based mask"
        return mat, mask


def load_test_dataset(dataset: MaterialVoxelDataset, obj_id: Optional[str] = None, use_saved_test_split: bool = False,
                      seg_checkpoint: Optional[str] = None, train_size: float = 0.9) -> List[int]:
    """Dataset indices to evaluate, in the reference's order (inference_combined.py:48-78): the objects named `obj_id`;
    else the objects of test_set.json next to the seg checkpoint; else the test part of random_split with
    torch.Generator().manual_seed(42). Raises ValueError when `obj_id` matches nothing (the reference exits)."""
    if obj_id:
        idx = [i for i, o in enumerate(dataset.obj_ids) if o == obj_id]
        if not idx:
            raise ValueError(f"No data found for object ID: {obj_id}")
        return idx
    if use_saved_test_split:
        fp = os.path.join(os.path.dirname(seg_checkpoint or ""), "test_set.json")
        assert os.path.isfile(fp), f"Test split file not found: {fp}"
        saved = set(_load_json(fp))
        idx = [i for i, o in enumerate(dataset.obj_ids) if o in saved]
        if idx:
            return idx
    n = len(dataset)
    n_train = int(train_size * n)
    _, test = torch.utils.data.random_split(range(n), [n_train, n - n_train], generator=torch.Generator().manual_seed(42))
    return list(test.indices)


# ------------------------------------------------------------------------------------------------------------- metrics
def material_metrics(mat: torch.Tensor, mask: Optional[torch.Tensor], seg_logits: torch.Tensor, cont_pred: torch.Tensor,
                     ranges: Dict[str, float], background_id: int = 7, gt_out: Optional[torch.Tensor] = None):
    """One device pass over a batch (csrc/material_metrics.cu). mat: (N, D, D, D, C_mat) raw material grids, mask:
    (N, D, D, D) or None (then mask = id != background_id, compute_accuracy's other branch), seg_logits (N, K, D, D, D),
    cont_pred (N, 3, D, D, D), all float32 on one CUDA device. Returns (gt (N, 4, D, D, D) device, counts (N, 2) int64
    numpy = (total, correct), sums (N, 4) float64 numpy = (sum (cont - gt)^2 mask per channel, sum mask))."""
    _lib.require_device()
    _lib.require_cuda("material_metrics", seg_logits)
    dev = seg_logits.device
    n, K = int(seg_logits.shape[0]), int(seg_logits.shape[1])
    spatial = tuple(seg_logits.shape[2:])
    if mat.dim() != 5 or tuple(mat.shape[:4]) != (n,) + spatial or tuple(cont_pred.shape) != (n, 3) + spatial or \
            (mask is not None and tuple(mask.shape) != (n,) + spatial):
        raise ValueError(f"shape mismatch: mat {tuple(mat.shape)}, mask {None if mask is None else tuple(mask.shape)}, "
                         f"seg {tuple(seg_logits.shape)}, cont {tuple(cont_pred.shape)}")
    V = int(np.prod(spatial))
    f = lambda t: t.detach().to(dev, torch.float32).contiguous()                        # noqa: E731
    mat_, seg_, cont_ = f(mat), f(seg_logits), f(cont_pred)
    mask_ = None if mask is None else f(mask)
    gt = gt_out if gt_out is not None else torch.empty((n, 4) + spatial, dtype=torch.float32, device=dev)
    counts = torch.empty((n, 2), dtype=torch.int64, device=dev)
    sums = torch.empty((n, 4), dtype=torch.float64, device=dev)
    r = ranges
    rng = (C.c_double * 6)(r["density_min"], r["density_max"], r["E_min"], r["E_max"], r["nu_min"], r["nu_max"])
    _lib.call("pixie_material_metrics", dev, mat_, int(mat.shape[-1]), mask_, seg_, K, cont_, n, V, rng, int(background_id), gt, counts,
              sums)
    return gt, counts.cpu().numpy(), sums.cpu().numpy()


def _accuracy(total: int, correct: int) -> float:
    """compute_accuracy's last lines: 0.0 when total == 0, else correct.float() / total.float() in float32."""
    if total == 0:
        return 0.0
    return (torch.tensor(correct, dtype=torch.int64).float() / torch.tensor(total, dtype=torch.int64).float()).item()


def batch_metrics(counts: np.ndarray, sums: np.ndarray) -> Tuple[Tuple[float, ...], List[Dict[str, float]]]:
    """The float32 arithmetic of process_batch (:129-159) on the per-sample counts and sums of `material_metrics`:
    masked_mean's num / (den.clamp(min=1) + 1e-8), the batch means over samples (and channels) and the per-sample dicts.
    Returns ((seg_acc, cont_mse, density_mse, youngs_mse, poisson_mse), [sample_metrics, ...])."""
    counts = np.asarray(counts, dtype=np.int64).reshape(-1, 2)
    sums = np.asarray(sums, dtype=np.float64).reshape(-1, 4)
    num = torch.from_numpy(sums[:, :3].astype(np.float32))
    den = torch.from_numpy(sums[:, 3:4].astype(np.float32))
    mse = num / (den.clamp(min=1) + 1e-8)                                                # (N, 3) float32
    total, correct = (int(v) for v in counts.sum(0))
    batch = (_accuracy(total, correct), mse.mean().item(), mse[:, 0:1].mean().item(), mse[:, 1:2].mean().item(),
             mse[:, 2:3].mean().item())
    samples = []
    for i in range(counts.shape[0]):
        m = {"seg_acc": _accuracy(int(counts[i, 0]), int(counts[i, 1])), "density_mse": mse[i:i + 1, 0:1].mean().item(),
             "youngs_mse": mse[i:i + 1, 1:2].mean().item(), "poisson_mse": mse[i:i + 1, 2:3].mean().item()}
        m["cont_mse"] = (m["density_mse"] + m["youngs_mse"] + m["poisson_mse"]) / 3.0
        samples.append(m)
    return batch, samples


class InferenceMetrics:
    """pixie/metrics.py:105-153: batch-level lists, per-object lists of sample metrics and the evaluated object ids."""

    def __init__(self):
        self.seg_accuracies, self.cont_mse_values, self.density_mse_values = [], [], []
        self.youngs_mse_values, self.poisson_mse_values = [], []
        self.obj_metrics: Dict[str, Dict[str, list]] = {}
        self.local_obj_ids: List[str] = []

    def add_batch_metrics(self, seg_acc, cont_mse, density_mse, youngs_mse, poisson_mse):
        self.seg_accuracies.append(seg_acc)
        self.cont_mse_values.append(cont_mse)
        self.density_mse_values.append(density_mse)
        self.youngs_mse_values.append(youngs_mse)
        self.poisson_mse_values.append(poisson_mse)

    def add_sample_metrics(self, obj_id, metrics_dict):
        if obj_id not in self.obj_metrics:
            self.obj_metrics[obj_id] = defaultdict(list)
        for key, value in metrics_dict.items():
            self.obj_metrics[obj_id][key].append(value)

    def gather_all_metrics(self, rank: int = 0, world_size: int = 1):
        """Seven lists with one entry per rank, on rank 0 (gather_object over the default group when world_size > 1)."""
        lists = [self.seg_accuracies, self.cont_mse_values, self.density_mse_values, self.youngs_mse_values, self.poisson_mse_values,
                 self.local_obj_ids, self.obj_metrics]
        if world_size == 1:
            return [[m] for m in lists]
        import torch.distributed as dist
        gathered = []
        for m in lists:
            out = [None] * world_size
            dist.gather_object(m, out if rank == 0 else None, dst=0)
            gathered.append(out)
        return gathered


def generate_metrics_report(all_metrics, output_dir: str, seg_checkpoint_path, cont_checkpoint_path, dispersion: str = "sem") -> Dict:
    """pixie/metrics.py:156-223, 333-411: per-object averages, global means, the SE (dispersion "sem") or STD dispersions and
    the 90 % interval of the accuracy; writes metrics.json and evaluated_obj_ids.json and returns the metrics dict. The
    per-class table (generate_class_table) needs Objaverse class metadata and is not written."""
    all_seg_acc, all_cont, all_dens, all_young, all_pois, all_obj_ids, all_obj_metrics = all_metrics
    merged: Dict[str, Dict[str, list]] = {}
    for obj_dict in all_obj_metrics:
        if obj_dict is None:
            continue
        for oid, metrics in obj_dict.items():
            if oid not in merged:
                merged[oid] = defaultdict(list)
            for key, values in metrics.items():
                merged[oid][key].extend(values)
    obj_avgs = {oid: {k: sum(v) / len(v) if v else 0.0 for k, v in m.items()} for oid, m in merged.items()}
    names = ["seg_acc", "cont_mse", "density_mse", "youngs_mse", "poisson_mse"]
    global_avgs = {}
    for name in names:
        values = [a[name] for a in obj_avgs.values() if name in a]
        global_avgs[name] = np.mean(values) if values else 0.0
    use_sem = dispersion.lower() in {"sem", "stderr"}

    def calc(values):
        if not values or len(values) <= 1:
            return 0.0
        return np.std(values, ddof=1) / math.sqrt(len(values)) if use_sem else np.std(values, ddof=0)

    seg_se = calc([a["seg_acc"] for a in obj_avgs.values()])
    z = 1.645
    lo, hi = global_avgs["seg_acc"] - z * seg_se, global_avgs["seg_acc"] + z * seg_se
    label = "SE" if use_sem else "STD"
    print("\nInference complete!")
    print(f"  Average Segmentation Accuracy: {global_avgs['seg_acc']:.4f}")
    print(f"    90% CI: [{lo:.4f}, {hi:.4f}] (± {z * seg_se:.4f})")
    print(f"  Average Continuous MSE: {global_avgs['cont_mse']:.6f} ({label} {calc([a['cont_mse'] for a in obj_avgs.values()]):.6f})")
    for metric, text in (("density_mse", "Density"), ("youngs_mse", "Young's"), ("poisson_mse", "Poisson")):
        print(f"    • {text} MSE: {global_avgs[metric]:.6f} ({label} {calc([a[metric] for a in obj_avgs.values()]):.6f})")

    disp = {}
    for metric in ("cont_mse", "density_mse", "youngs_mse", "poisson_mse"):
        values = [a[metric] for a in obj_avgs.values()]
        if len(values) > 1:
            disp[metric] = float(np.std(values, ddof=1) / math.sqrt(len(values))) if label == "SE" else float(np.std(values, ddof=0))
        else:
            disp[metric] = 0.0
    data = {
        "checkpoints": {"segmentation": seg_checkpoint_path, "continuous": cont_checkpoint_path},
        "summary": {
            "total_objects": len(obj_avgs),
            "dispersion_type": label,
            "segmentation_accuracy": {"mean": float(global_avgs["seg_acc"]),
                                      "confidence_interval_90": {"low": float(lo), "high": float(hi), "margin": float(z * seg_se)}},
            "continuous_metrics": {
                "overall": {"mean": float(global_avgs["cont_mse"]), "dispersion": disp["cont_mse"]},
                "density": {"mean": float(global_avgs["density_mse"]), "dispersion": disp["density_mse"]},
                "youngs_modulus": {"mean": float(global_avgs["youngs_mse"]), "dispersion": disp["youngs_mse"]},
                "poisson_ratio": {"mean": float(global_avgs["poisson_mse"]), "dispersion": disp["poisson_mse"]},
            },
        },
        "per_object_metrics": obj_avgs,
        "per_object_raw_data": {
            oid: {"segmentation_accuracy": {"values": m["seg_acc"], "mean": sum(m["seg_acc"]) / len(m["seg_acc"]) if m["seg_acc"] else 0.0},
                  "continuous_mse": {"values": m["cont_mse"], "mean": sum(m["cont_mse"]) / len(m["cont_mse"]) if m["cont_mse"] else 0.0}}
            for oid, m in merged.items()},
    }
    _save_json(data, os.path.join(output_dir, "metrics.json"))
    flat_ids = [i for part in all_obj_ids if part for i in part]
    _save_json(sorted(set(flat_ids)), os.path.join(output_dir, "evaluated_obj_ids.json"))
    return data


def save_predictions(output_dir: str, info: Dict[str, str], pred: np.ndarray, gt: np.ndarray, mask: np.ndarray) -> None:
    """save_predictions (inference_combined.py:173-217): <output_dir>/<obj_id>/sample_<id>_{pred,gt,mask,info}.npy, with
    pred the packed (3 + K, D, D, D) prediction, gt the normalised (4, D, D, D) ground truth and info the pickled dict."""
    sample_id = str(info["sample_id"])
    obj_dir = os.path.join(output_dir, info["obj_id"])
    os.makedirs(obj_dir, exist_ok=True)
    np.save(os.path.join(obj_dir, f"sample_{sample_id}_pred.npy"), pred)
    np.save(os.path.join(obj_dir, f"sample_{sample_id}_gt.npy"), gt)
    np.save(os.path.join(obj_dir, f"sample_{sample_id}_mask.npy"), mask)
    info_to_save = {"obj_id": info["obj_id"], "sample_id": sample_id, "data_path": info["data_path"],
                    "feature_path": info["feature_path"], "mask_path": info["mask_path"]}
    np.save(os.path.join(obj_dir, f"sample_{sample_id}_info.npy"), info_to_save)


# ----------------------------------------------------------------------------------------------------- material cloud PLY
#: the vertex table of map_pred_to_ply (map_pred_to_coords.py:222-231), in its property order
CLOUD_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("red", "u1"), ("green", "u1"), ("blue", "u1"), ("alpha", "u1"),
                        ("part_label", "<i4"), ("density", "<f4"), ("E", "<f4"), ("nu", "<f4"), ("material_id", "<i4"), ("conf", "<f4")])
# plyfile's names for numpy types (its _data_type_reverse)
_PLY_NAMES = {"i1": "char", "u1": "uchar", "i2": "short", "u2": "ushort", "i4": "int", "u4": "uint", "f4": "float", "f8": "double"}


def ply_header(dtype: np.dtype, count: int) -> bytes:
    """The header PlyData([PlyElement.describe(rows, 'vertex')], text=False).write puts before a binary vertex table."""
    lines = ["ply", "format binary_little_endian 1.0", f"element vertex {count}"]
    lines += [f"property {_PLY_NAMES[dtype[n].str[1:]]} {n}" for n in dtype.names]
    return ("\n".join(lines + ["end_header"]) + "\n").encode("ascii")


def _write_rows(path: str, rows: np.ndarray) -> None:
    rows = np.ascontiguousarray(rows.astype(rows.dtype.newbyteorder("<"), copy=False))
    with open(path, "wb") as f:
        f.write(ply_header(rows.dtype, len(rows)))
        f.write(rows.tobytes())


def material_cloud_table(field: Dict[str, torch.Tensor]) -> np.ndarray:
    """extract_material_points' dict as map_pred_to_ply's structured vertex table (white, opaque)."""
    pos = field["pos"].cpu().numpy()
    t = np.zeros(len(pos), dtype=CLOUD_DTYPE)
    t["x"], t["y"], t["z"] = pos[:, 0], pos[:, 1], pos[:, 2]
    for c in ("red", "green", "blue", "alpha"):
        t[c] = 255
    t["part_label"] = field["part_labels"].cpu().numpy()
    for k in ("density", "E", "nu", "material_id", "conf"):
        t[k] = field[k].cpu().numpy()
    return t


def write_material_point_cloud(path: str, table) -> None:
    """Writes a material point cloud (map_pred_to_ply's vertex table, or extract_material_points' dict) as plyfile does."""
    _write_rows(path, material_cloud_table(table) if isinstance(table, dict) else np.asarray(table, dtype=CLOUD_DTYPE))


def transform_nerf_to_world(ply_path: str, dataparser_path: str, world_output_path: str) -> None:
    """map_pred_to_coords.py:77-121: the PLY's x y z from the NeRF training frame to the world frame of
    dataparser_transforms.json, x_world = (T^-1 [x / scale, 1])[:3], every other column copied. Host float32 numpy, the
    reference's own expressions: float32 T, float32 np.linalg.inv, x / float32(scale), and the float32 matmul of numpy
    (its BLAS sgemm decides the order of the 4-term sums, as in the reference)."""
    rows = scene_files.read_ply(ply_path).read()
    with open(dataparser_path) as f:
        dp = json.load(f)
    scale = float(dp["scale"])
    T = np.eye(4, dtype=np.float32)
    T[:3, :] = np.asarray(dp["transform"], dtype=np.float32)
    T_inv = np.linalg.inv(T)
    coords = np.vstack((rows["x"], rows["y"], rows["z"])).T.astype(np.float32) / scale
    coords_h = np.concatenate([coords, np.ones((coords.shape[0], 1), dtype=np.float32)], axis=1)
    world = (T_inv @ coords_h.T).T[:, :3]
    out = rows.copy()
    out["x"], out["y"], out["z"] = world[:, 0], world[:, 1], world[:, 2]
    _write_rows(world_output_path, out)


def map_pred_to_ply(pred_path: str, mask_path: str, grid_feature_path: str, output_path: str, obj_id: Optional[str] = None,
                    world_output_path: Optional[str] = None, dataparser_path: Optional[str] = None,
                    ranges: Optional[Dict[str, float]] = None, device="cuda:0") -> Dict[str, torch.Tensor]:
    """map_pred_to_coords.py:128-283: sample_<id>_pred.npy + mask + clip_features.npz bounds -> mapped_preds.ply (and the
    world-frame copy when `world_output_path` is given; dataparser_transforms.json next to the grid file by default).
    The unscaling and the vertex table run on the device (extract_material_points), which is returned."""
    from .material_transfer import extract_material_points
    min_bounds, max_bounds, grid_shape = voxel_io.load_grid_metadata(grid_feature_path)
    pred = np.load(pred_path)
    mask = np.load(mask_path)
    assert mask.shape == (64, 64, 64), f"mask.shape: {mask.shape}. Expected (64, 64, 64)"
    if not np.array_equal(pred.shape[1:4], grid_shape):
        raise ValueError(f"Prediction spatial dimensions {pred.shape[1:4]} do not match grid shape {grid_shape}")
    if not np.array_equal(mask.shape, grid_shape):
        raise ValueError(f"Mask shape {mask.shape} does not match grid shape {grid_shape}")
    field = extract_material_points(torch.from_numpy(np.ascontiguousarray(pred, dtype=np.float32)).to(device),
                                    torch.from_numpy(np.ascontiguousarray(mask, dtype=np.float32)).to(device), min_bounds, max_bounds, ranges)
    write_material_point_cloud(output_path, field)
    log.info(f"Saved PLY file to {output_path} from {pred_path}")
    if world_output_path is not None:
        if dataparser_path is None:
            dataparser_path = Path(grid_feature_path).parent / "dataparser_transforms.json"
            if not dataparser_path.exists():
                raise FileNotFoundError(f"Could not find dataparser_transforms.json at {dataparser_path}. "
                                        "Please provide the path using --dataparser_path argument.")
        transform_nerf_to_world(output_path, str(dataparser_path), world_output_path)
    return field
