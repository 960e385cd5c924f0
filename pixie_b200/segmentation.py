"""VLM-mode part segmentation (pixie/voxel/segmentation.py): every occupied voxel of a CLIP feature grid goes to the part
query it resembles most, optionally smoothed by a k-nearest-neighbour label vote, and the parts' materials are written as
`segmented_rgb.ply`, `segmented_semantics.ply` (the `--point_cloud_path` of gs_simulation in VLM mode) and
`material_grid.npy` (the labels MaterialVoxelDataset evaluates against).

The similarities, labels and scores come from `pixie_part_similarity`, which reads the fp16 grid once on the device with no
fp32 copy; the vote from `pixie_knn_label_vote` and the RGB lookup from `pixie_nearest_vertex`, both exact searches on the
device. The query embeddings are an input: `--query_embeddings` (P, C), or the user's f3rm CLIP when it is installed.

    python -m pixie_b200.segmentation --grid_feature_path .../clip_features.npz --occupancy_path .../occupancy.ply \\
        --output_dir out --material_dict_path chosen_vlm_results.json [--query_embeddings q.npy] [--use_spatial_smoothing true]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from . import _lib
from .network_files import _write_rows
from .scene_files import read_ply
from .voxel_io import load_feature_grid

MAX_PARTS = 64
# matplotlib's tab10 colormap (RGBA, float64)
TAB10 = [tuple(int(h[i:i + 2], 16) / 255 for i in (1, 3, 5)) + (1.0,) for h in
         ("#1f77b4", "#ff7f0e", "#2ca02c", "#d62728", "#9467bd", "#8c564b", "#e377c2", "#7f7f7f", "#bcbd22", "#17becf")]
SEGMENTED_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("red", "u1"), ("green", "u1"), ("blue", "u1"), ("alpha", "u1"),
                            ("part_label", "<i4"), ("density", "<f4"), ("E", "<f4"), ("nu", "<f4"), ("material_id", "<i4")])


def _ptr(t: Optional[torch.Tensor]):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _stream(device) -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def str2bool(v):
    """pixie/utils.py:69-77."""
    if isinstance(v, bool):
        return v
    if v.lower() in ("yes", "true", "True", "t", "y", "1"):
        return True
    elif v.lower() in ("no", "false", "False", "f", "n", "0"):
        return False
    else:
        raise argparse.ArgumentTypeError("Boolean value expected.")


# ------------------------------------------------------------------------------------------------ device operations
def normalize_queries(query_embs, device) -> torch.Tensor:
    """run_clip's query rows (:109-110): `.float()`, then divided by their norm, on `device`."""
    q = torch.as_tensor(query_embs).to(device).float()
    return q / q.norm(dim=-1, keepdim=True)


def part_similarity(features: torch.Tensor, unit_queries: torch.Tensor, softmax_temperature: float = 0.1,
                    mask: Optional[torch.Tensor] = None, n_occupied: Optional[int] = None, with_probs: bool = True):
    """(similarities (N, P) fp32, labels (N,) int64, scores (N,) fp32, probabilities (N, P) fp32 or None) for the rows of the
    float16 `features` (..., C) selected by the boolean `mask` (over the leading dims, C order; every row without one).
    `unit_queries` (P, C) fp32 are normalize_queries' rows. `n_occupied` is mask's count when the caller has it."""
    lib = _lib.require_device()
    if not features.is_cuda or features.dtype != torch.float16:
        raise _lib.PixieError("part_similarity needs float16 CUDA features; there is no CPU fallback")
    C_ = features.shape[-1]
    if unit_queries.ndim != 2 or unit_queries.shape[1] != C_:
        raise ValueError(f"query embeddings must be (P, {C_}), got {tuple(unit_queries.shape)}")
    P = unit_queries.shape[0]
    if not 1 <= P <= MAX_PARTS:
        raise ValueError(f"part_similarity supports 1 to {MAX_PARTS} part queries, got {P}")
    dev = features.device
    f = features.contiguous().reshape(-1, C_)
    q = unit_queries.to(dev, torch.float32).contiguous()
    m8 = None
    if mask is not None:
        m8 = mask.to(dev).reshape(-1).to(torch.uint8).contiguous()
        if m8.numel() != f.shape[0]:
            raise ValueError(f"mask has {m8.numel()} entries for {f.shape[0]} feature rows")
        n = int(m8.count_nonzero()) if n_occupied is None else int(n_occupied)
    else:
        n = f.shape[0]
    sims = torch.empty((n, P), dtype=torch.float32, device=dev)
    probs = torch.empty((n, P), dtype=torch.float32, device=dev) if with_probs else None
    labels = torch.empty(n, dtype=torch.int64, device=dev)
    scores = torch.empty(n, dtype=torch.float32, device=dev)
    # torch divides by a Python scalar as a multiplication by its fp32 reciprocal
    inv_t = float(np.float32(1.0) / np.float32(softmax_temperature))
    with torch.cuda.device(dev):
        _lib.check(lib.pixie_part_similarity(_ptr(f), _ptr(m8), f.shape[0], C_, n, _ptr(q), P, inv_t, _ptr(sims), _ptr(labels),
                                             _ptr(scores), _ptr(probs), _stream(dev)))
    return sims, labels, scores, probs


def knn_label_vote(coords: torch.Tensor, labels: torch.Tensor, k: int = 200) -> torch.Tensor:
    """For each point, the smallest of the most frequent labels among its k nearest points (itself included; fp64
    distances, ties at the k-th distance to the lowest index), int64 on the device of `coords`."""
    n = coords.shape[0]
    if not 1 <= k <= n:
        raise ValueError(f"Expected n_neighbors <= n_samples_fit, but n_neighbors = {k}, n_samples_fit = {n}, n_samples = {n}"
                         if k > n else f"k must be >= 1, got {k}")
    lib = _lib.require_device()
    dev = coords.device if coords.is_cuda else torch.device("cuda", torch.cuda.current_device())
    pos = coords.to(dev, torch.float32).contiguous()
    if not bool(torch.isfinite(pos).all()):
        raise ValueError("knn_label_vote needs finite coordinates")
    lab = labels.to(dev, torch.int64).contiguous()
    out = torch.empty(n, dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        _lib.check(lib.pixie_knn_label_vote(_ptr(pos), n, _ptr(lab), int(k), _ptr(out), _stream(dev)))
    return out


def nearest_vertex(vertices: np.ndarray, queries: torch.Tensor) -> torch.Tensor:
    """Index (int64, host) of the nearest float64 vertex of each float32 query by the fp64 distance, ties to the lowest."""
    lib = _lib.require_device()
    dev = queries.device if queries.is_cuda else torch.device("cuda", torch.cuda.current_device())
    v = torch.from_numpy(np.ascontiguousarray(vertices, dtype=np.float64)).to(dev)
    q = queries.to(dev, torch.float32).contiguous()
    idx = torch.empty(q.shape[0], dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(lib.pixie_nearest_vertex(_ptr(v), v.shape[0], _ptr(q), q.shape[0], _ptr(idx), _stream(dev)))
    return idx.cpu().to(torch.int64)


# ------------------------------------------------------------------------------------------------ the reference's API
def _mask_path(grid_feature_path: str) -> str:
    p = grid_feature_path.replace(".npz", "_mask.npy")
    assert os.path.exists(p), f"Mask not found at {p}. Please run voxelization first."
    return p


def _grid_coords(min_bounds, max_bounds, grid_shape, device) -> torch.Tensor:
    """The (D, H, W, 3) voxel coordinates of get_initial_voxel_grid_from_saved (:70-74): float32 linspace per axis, ij."""
    x, y, z = (torch.linspace(min_bounds[i], max_bounds[i], int(grid_shape[i]), device=device) for i in range(3))
    return torch.stack(torch.meshgrid(x, y, z, indexing="ij"), dim=-1)


def _load_grid(grid_feature_path: str, device):
    with np.load(grid_feature_path) as metadata:
        min_bounds, max_bounds, grid_shape = metadata["min_bounds"], metadata["max_bounds"], metadata["grid_shape"]
    feats = load_feature_grid(grid_feature_path.replace(".npz", "_features.npy"))[0].to(device, non_blocking=True)
    mask_np = np.load(_mask_path(grid_feature_path)).astype(bool)
    coords = _grid_coords(min_bounds, max_bounds, grid_shape, device)[torch.from_numpy(mask_np).to(device)]
    metrics = {"initial": np.prod(grid_shape), "masked_voxels": int(mask_np.sum())}
    return feats, mask_np, coords, metrics


def get_initial_voxel_grid_from_saved(grid_feature_path: str, occupancy_path: str = None, device: str = "cuda"):
    """(features of the occupied voxels (N, C) float16, their coordinates (N, 3) float32, metrics) as :18-88 returns them.
    The grid crosses to the device once, from a pinned host copy of the file."""
    feats, mask_np, coords, metrics = _load_grid(grid_feature_path, device)
    linear_mask = torch.from_numpy(mask_np.reshape(-1)).to(device)
    return feats.reshape(-1, feats.shape[-1])[linear_mask], coords, metrics


def load_occupancy_grid(occupancy_path: str, device: str = "cuda") -> torch.Tensor:
    """The occupancy PLY's vertices as float32 (N, 3) (:91-94)."""
    rows = read_ply(occupancy_path).read()
    pts = np.column_stack([rows[c].astype(np.float64) for c in "xyz"])
    return torch.tensor(pts, dtype=torch.float32, device=device)


def encode_queries(queries: Sequence[str], device="cuda") -> torch.Tensor:
    """CLIP text embeddings of the part queries from the user's f3rm (:100-109), `.float()`, not yet normalised."""
    try:
        from f3rm.features.clip import clip
        from f3rm.features.clip_extract import CLIPArgs
    except ImportError as e:
        raise RuntimeError("encoding the part queries needs f3rm's CLIP, which is not installed; pass the (P, C) text embeddings "
                           "of the material dict's keys with --query_embeddings (query_embs= in Python)") from e
    clip_model, _ = clip.load(CLIPArgs.model_name, device=device)
    with torch.no_grad():
        return clip_model.encode_text(clip.tokenize(list(queries)).to(device)).float()


def run_clip(queries, features_filtered, softmax_temperature, device="cuda", query_embs=None):
    """(probabilities, similarities) (N, P) fp32 as :98-122 returns them, for the float16 features (N, C) of the occupied
    voxels. `query_embs` (P, C) replaces the CLIP text encoder; without it the queries are encoded with f3rm."""
    q = normalize_queries(encode_queries(queries, device) if query_embs is None else query_embs, features_filtered.device)
    sims, _, _, probs = part_similarity(features_filtered, q, softmax_temperature)
    return probs, sims


def clip_part_segmentation(grid_feature_path: str, part_queries: List[str], occupancy_path: str = None, device: str = "cuda",
                           softmax_temperature: float = 0.1, query_embs=None):
    """(coordinates (N, 3) float32, labels (N,) int64, scores (N,) fp32, metrics) as :125-183 returns them. The kernel reads
    the occupied voxels straight from the full grid."""
    if query_embs is None:
        query_embs = encode_queries(part_queries, device)
    feats, mask_np, coords, metrics = _load_grid(grid_feature_path, device)
    q = normalize_queries(query_embs, feats.device)
    _, labels, scores, _ = part_similarity(feats, q, softmax_temperature, mask=torch.from_numpy(mask_np),
                                           n_occupied=metrics["masked_voxels"], with_probs=False)
    metrics["num_parts"] = len(part_queries)
    counts = torch.bincount(labels, minlength=len(part_queries)).cpu().tolist() if labels.numel() else [0] * len(part_queries)
    for i, query in enumerate(part_queries):
        metrics[f"part_{i}_{query}"] = counts[i]
    return coords, labels, scores, metrics


def local_post_process_segmentation(coords: torch.Tensor, part_labels: torch.Tensor, k: int = 200) -> torch.Tensor:
    """:190-226: each label becomes the mode (smallest on a tie) of the original labels of its k nearest voxels."""
    return knn_label_vote(coords, part_labels, k).to(part_labels.device)


def _occupancy_colors(rows: np.ndarray, path: str) -> np.ndarray:
    """The vertex colours as trimesh gives them: RGBA uint8, alpha 255 when the file has none."""
    names = rows.dtype.names
    if not all(c in names for c in ("red", "green", "blue")):
        raise ValueError(f"{path}: the occupancy PLY has no red/green/blue vertex colours")
    cols = [rows[c] for c in ("red", "green", "blue")] + [rows["alpha"] if "alpha" in names else np.full(len(rows), 255, np.uint8)]
    if any(c.dtype != np.uint8 for c in cols):
        raise ValueError(f"{path}: expected uchar vertex colours")
    return np.column_stack(cols)


def _part_properties(part_labels_np, part_queries, material_props):
    """Per-voxel density, E, nu (float32) and material_id (int32) from the parts' materials (:323-338)."""
    n = len(part_labels_np)
    density, E, nu = np.zeros(n, np.float32), np.zeros(n, np.float32), np.zeros(n, np.float32)
    material_id = np.zeros(n, np.int32)
    for i in range(part_labels_np.max() + 1):
        mask = part_labels_np == i
        if not np.any(mask):
            continue
        part_name = part_queries[i]
        assert part_name in material_props, f"part_name `{part_name}` not found in material_props. Material props: {material_props}"
        props = material_props[part_name]
        density[mask] = props.get("density", 200)
        E[mask] = props.get("E", 2e6)
        nu[mask] = props.get("nu", 0.4)
        material_id[mask] = props.get("material_id", 0)
    return density, E, nu, material_id


def segmented_point_cloud(coords: torch.Tensor, part_labels: torch.Tensor, part_queries: List[str],
                          material_props: Dict[str, Dict[str, float]], device="cuda:0") -> Dict[str, torch.Tensor]:
    """The material point cloud that scene_files.load_point_cloud reads from segmented_semantics.ply (pos, density, E, nu,
    material_id, part_labels, conf = 1), built in memory for SceneBatchDriver.run_physics_simulation."""
    labels_np = part_labels.cpu().numpy()
    density, E, nu, material_id = _part_properties(labels_np, part_queries, material_props)
    f32 = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(device)          # noqa: E731
    i32 = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)).to(device)            # noqa: E731
    return {"pos": coords.to(device, torch.float32), "density": f32(density), "E": f32(E), "nu": f32(nu),
            "material_id": i32(material_id), "part_labels": i32(labels_np.astype(np.int32)),
            "conf": torch.ones(len(labels_np), dtype=torch.float32, device=device)}


def save_segmented_point_cloud(coords: torch.Tensor, part_labels: torch.Tensor, output_dir: str, cmap_name: str = "tab10",
                               original_pc_path: str = None, part_queries: List[str] = None,
                               material_props: Dict[str, Dict[str, float]] = None, grid_feature_path: str = None,
                               background_id: int = 7):
    """:231-471: segmented_rgb.ply, segmented_semantics.ply and, with grid_feature_path, material_grid.npy and its four
    channel grids, in output_dir. The RGB colours come from the nearest occupancy vertex, found on the device."""
    if cmap_name != "tab10":
        raise ValueError(f"only the tab10 colormap is built in, got {cmap_name!r}")
    os.makedirs(output_dir, exist_ok=True)
    coords_np = coords.cpu().numpy()
    part_labels_np = part_labels.cpu().numpy()
    assert len(part_labels_np) == len(coords_np), (
        f"part_labels_np and coords_np must have the same length. len(part_labels_np): {len(part_labels_np)}, len(coords_np): "
        f"{len(coords_np)}. Mismatch is likely due to new voxelization and cached part_labels_np. Try re-running with overwrite=True "
        "to recompute part_labels")
    n = coords_np.shape[0]
    rgb_colors = np.zeros((n, 4), dtype=np.float32)
    semantic_colors = np.zeros((n, 4), dtype=np.float32)
    if original_pc_path:
        rows = read_ply(original_pc_path).read()
        original_vertices = np.column_stack([rows[c].astype(np.float64) for c in "xyz"])
        original_colors = _occupancy_colors(rows, original_pc_path)
        if original_colors.max() > 1.0:
            original_colors = original_colors / 255.0
        indices = nearest_vertex(original_vertices, coords).numpy()
        rgb_colors[:, :3] = original_colors[indices, :3]
        rgb_colors[:, 3] = 1.0
    else:
        rgb_colors[:, :3] = 1.0
        rgb_colors[:, 3] = 1.0
    for i in range(part_labels_np.max() + 1):
        mask = part_labels_np == i
        if np.any(mask):
            semantic_colors[mask] = np.array(TAB10[i % len(TAB10)])
    density, E, nu, material_id = _part_properties(part_labels_np, part_queries, material_props)

    for path, colors in (("segmented_rgb.ply", rgb_colors), ("segmented_semantics.ply", semantic_colors)):
        c8 = (colors * 255).astype(np.uint8)
        t = np.zeros(n, dtype=SEGMENTED_DTYPE)
        t["x"], t["y"], t["z"] = coords_np[:, 0], coords_np[:, 1], coords_np[:, 2]
        t["red"], t["green"], t["blue"], t["alpha"] = c8[:, 0], c8[:, 1], c8[:, 2], c8[:, 3]
        t["part_label"] = part_labels_np
        t["density"], t["E"], t["nu"], t["material_id"] = density, E, nu, material_id
        _write_rows(os.path.join(output_dir, path), t)

    if grid_feature_path is not None:
        with np.load(grid_feature_path) as metadata:
            grid_shape = metadata["grid_shape"]
        material_grid = np.zeros((*grid_shape, 4), dtype=np.float32)
        material_grid[..., 3] = background_id
        mask = np.load(_mask_path(grid_feature_path)).astype(bool)
        flat_idx = np.flatnonzero(mask.ravel(order="C"))
        assert len(flat_idx) == len(coords_np), (
            f"Mask/coords length mismatch: mask has {len(flat_idx)} true voxels, coords has {len(coords_np)} points. "
            "Ensure coords come from mask.")
        material_grid_flat = material_grid.reshape(-1, 4)
        material_grid_flat[flat_idx, 0] = density
        material_grid_flat[flat_idx, 1] = E
        material_grid_flat[flat_idx, 2] = nu
        material_grid_flat[flat_idx, 3] = material_id
        np.save(os.path.join(output_dir, "material_grid.npy"), material_grid)
        for i, name in enumerate(("density_grid.npy", "E_grid.npy", "nu_grid.npy", "material_id_grid.npy")):
            np.save(os.path.join(output_dir, name), material_grid[..., i])


# ------------------------------------------------------------------------------------------------ command line
def parse_args(argv=None):
    parser = argparse.ArgumentParser(prog="python -m pixie_b200.segmentation", description=__doc__.split("\n\n")[0])
    parser.add_argument("--grid_feature_path", type=str, required=True)
    parser.add_argument("--occupancy_path", type=str, required=True)
    parser.add_argument("--output_dir", type=str, required=True)
    parser.add_argument("--material_dict_path", type=str, required=True,
                        help="Path to JSON file mapping part queries to material properties")
    parser.add_argument("--use_spatial_smoothing", type=str2bool, default=False)
    parser.add_argument("--overwrite", type=str2bool, default=False)
    parser.add_argument("--background_id", type=int, default=7, help="Material ID for background voxels")
    parser.add_argument("--query_embeddings", type=str, default=None,
                        help=".npy (P, C) CLIP text embeddings of the material dict's keys, in key order (default: encode "
                             "them with f3rm's CLIP)")
    return parser.parse_args(argv)


def load_material_dict(path: str):
    """(material props, part queries in key order) of chosen_vlm_results.json (unwrapping "material_dict")."""
    assert os.path.exists(path), f"material_dict_path {path} does not exist"
    with open(path) as f:
        material_props = json.load(f)
    if "material_dict" in material_props:
        material_props = material_props["material_dict"]
    return material_props, list(material_props.keys())


def main(argv=None):
    args = parse_args(argv)
    material_props, part_queries = load_material_dict(args.material_dict_path)
    if not part_queries:
        raise ValueError(f"{args.material_dict_path}: the material dict has no parts")
    for q in part_queries:
        if not isinstance(material_props[q], dict):
            raise ValueError(f"{args.material_dict_path}: part {q!r} maps to {material_props[q]!r}, not a property dict")
    labels_output_path = os.path.join(args.output_dir, "part_labels.npy")
    recompute = args.overwrite or not os.path.exists(labels_output_path)
    query_embs = None
    if recompute:
        if len(part_queries) > MAX_PARTS:
            raise ValueError(f"{len(part_queries)} parts; at most {MAX_PARTS} are supported")
        if args.query_embeddings is not None:
            query_embs = np.load(args.query_embeddings)
            if query_embs.ndim != 2 or query_embs.shape[0] != len(part_queries):
                raise ValueError(f"{args.query_embeddings}: expected ({len(part_queries)}, C) embeddings, one row per key of "
                                 f"{args.material_dict_path}, got {query_embs.shape}")
        with np.load(args.grid_feature_path) as metadata:
            grid_shape = tuple(int(s) for s in metadata["grid_shape"])
        feat_shape = np.load(args.grid_feature_path.replace(".npz", "_features.npy"), mmap_mode="r").shape
        if query_embs is not None and feat_shape[-1] != query_embs.shape[1]:
            raise ValueError(f"the features have C = {feat_shape[-1]}, the query embeddings {query_embs.shape[1]}")
        if tuple(feat_shape[:-1]) != grid_shape:
            raise ValueError(f"the features are {feat_shape}, the grid_shape is {grid_shape}")
    else:
        cached = np.load(labels_output_path)
        if cached.size and (cached.min() < 0 or cached.max() >= len(part_queries)):
            raise ValueError(f"{labels_output_path} has labels outside [0, {len(part_queries)}): the material dict has no part "
                             "for them; rerun with --overwrite true")
    if recompute:
        os.makedirs(args.output_dir, exist_ok=True)
        coords_filtered, part_labels, _, _ = clip_part_segmentation(args.grid_feature_path, part_queries, args.occupancy_path,
                                                                    query_embs=query_embs)
        if args.use_spatial_smoothing:
            part_labels = local_post_process_segmentation(coords_filtered, part_labels)
        np.save(labels_output_path, part_labels.cpu().numpy())
    else:
        part_labels = torch.from_numpy(cached)
        coords_filtered = load_occupancy_grid(args.occupancy_path)
    save_segmented_point_cloud(coords_filtered, part_labels, args.output_dir, original_pc_path=args.occupancy_path,
                               part_queries=part_queries, material_props=material_props, grid_feature_path=args.grid_feature_path,
                               background_id=args.background_id)


if __name__ == "__main__":
    main()
