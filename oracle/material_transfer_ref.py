"""ORACLE (test infrastructure, not product code): CPU restatement of the reference's material-field -> particle
transfer, following the reference line by line with numpy / scikit-learn as the reference does.

  unscale_prediction            pixie/voxel/map_pred_to_coords.py:41-75
  vertex_table                  pixie/voxel/map_pred_to_coords.py:198-245   (what map_pred_to_ply writes into the PLY)
  MaterialProperties, perform_knn_smoothing
                                third_party/PhysGaussian/material_field.py:26-86, 228-293
  apply_additional_params       third_party/PhysGaussian/mpm_solver_warp/mpm_utils.py:591-610 via material_field.py:343-363

PINNED BY THE REFERENCE'S OWN FUNCTIONS: the reference modules import hydra / plyfile / warp / taichi (absent here) and cannot be
imported whole, but tests/golden/make_transfer_golden.py pulls the function sources out of the reference files with `ast` and
executes them (real numpy / scikit-learn / torch); tests/test_transfer_golden.py holds every function below to the resulting
fixture tests/golden/transfer_golden.npz BIT-EXACTLY (that is how the DEFAULT_VALUES['E'] = 5000.0 slip of round 1 was caught).
Only tests/ may import this file.
"""
from __future__ import annotations

import numpy as np

DEFAULT_VALUES = {"density": 1000.0, "E": 5000.0, "nu": 0.3, "part_label": 0, "material_id": "stationary"}   # material_field.py:16-23
STATIONARY_ID = 6                                                                                       # mpm_solver_warp.py:10-26


def _from_unit(c: np.ndarray, lo: float, hi: float) -> np.ndarray:
    """[-1, 1] -> [lo, hi]; float32 array arithmetic with Python-float bounds, evaluated in the reference's order
    ((c + 1) * (hi - lo) / 2 + lo, map_pred_to_coords.py:62-71)."""
    return (c + 1.0) * (hi - lo) / 2.0 + lo


def unscale_prediction(pred_tensor: np.ndarray, r: dict) -> np.ndarray:
    """map_pred_to_coords.py:41-75: channels 0/1 are log10(density), log10(E), channel 2 is nu; the class channels pass through."""
    out = pred_tensor.copy().astype(np.float32)
    unit = np.clip(pred_tensor[:3], -1.0, 1.0)                 # the network output is not strictly bounded
    out[0] = 10 ** _from_unit(unit[0], r["density_min"], r["density_max"])
    out[1] = 10 ** _from_unit(unit[1], r["E_min"], r["E_max"])
    out[2] = _from_unit(unit[2], r["nu_min"], r["nu_max"])
    return out


def vertex_table(scaled_pred: np.ndarray, mask: np.ndarray, min_bounds, max_bounds, r: dict) -> dict:
    """The vertex records map_pred_to_ply writes (:198-245), as arrays: occupied voxels in C order, voxel centres from
    np.linspace over the bounds (meshgrid 'ij'), id = argmax of the class channels, conf = their maximum. A (1, 64, 64, 64)
    class block holds the ids themselves (get_mat_id), truncated by the 'i4' fields, with conf = 1."""
    field = unscale_prediction(scaled_pred, r)
    classes = field[3:]
    ids = classes[0] if classes.shape == (1, 64, 64, 64) else np.argmax(classes, axis=0)  # get_mat_id :122-126
    axes = [np.linspace(min_bounds[d], max_bounds[d], mask.shape[d]) for d in range(3)]
    centres = np.stack(np.meshgrid(*axes, indexing="ij"), axis=-1)
    keep = mask > 0
    conf = np.max(classes, axis=0)[keep] if classes.shape[0] > 1 else np.ones(int(keep.sum()), dtype=np.float32)
    f32 = lambda a: a[keep].astype(np.float32)                                          # PLY fields are 'f4' / 'i4' (:222-231)
    return {"pos": centres[keep].astype(np.float32), "density": f32(field[0]), "E": f32(field[1]), "nu": f32(field[2]),
            "material_id": ids[keep].astype(np.int32), "part_labels": ids[keep].astype(np.int32), "conf": conf.astype(np.float32)}


_CATEGORICAL = ("material_id", "part_labels")
_ORDER = ("part_labels", "density", "E", "nu", "material_id", "conf")                     # MaterialProperties.properties order (:29-36)


def _fallback_values(props: dict, n: int) -> dict:
    """get_defaults (:38-50): 'stationary' for the material, 0 for the part label, the mean of everything else."""
    out = {}
    for name in _ORDER:
        v = props[name]
        if name == "material_id":
            fill = STATIONARY_ID
        elif name == "part_labels":
            fill = DEFAULT_VALUES["part_label"]
        else:
            fill = np.mean(v) if len(v) > 0 else DEFAULT_VALUES.get(name, 0.0)
        out[name] = np.full(n, fill, dtype=v.dtype if hasattr(v, "dtype") else np.float32)
    return out


def _first_most_frequent(values) -> int:
    """Counter(values).most_common(1)[0][0]: highest count, ties resolved by first appearance."""
    seen = list(dict.fromkeys(values.tolist()))
    counts = [int(np.sum(values == s)) for s in seen]
    return seen[int(np.argmax(counts))]                        # argmax returns the first maximum


def _from_neighbours(props: dict, idx: np.ndarray, dist: np.ndarray, weighted: bool) -> dict:
    """assign_from_neighbors (:52-86) for one particle: idx / dist = its k neighbours in ascending distance."""
    w = 1.0 / (dist + 1e-8)
    w = w / np.sum(w)
    out = {}
    for name in _ORDER:
        v = props[name][idx]
        if name in _CATEGORICAL:
            if weighted:
                labels, inverse = np.unique(v, return_inverse=True)
                out[name] = labels[np.argmax(np.bincount(inverse, weights=w))]
            else:
                out[name] = _first_most_frequent(v)
        else:
            out[name] = np.dot(w, v) if weighted else np.mean(v)
    return out


def perform_knn_smoothing(query_positions: np.ndarray, params: dict, k_smoothing_neighbors=10, nn_distance_threshold=0.1,
                          weighted_assignment=False):
    """material_field.py:228-293 with scikit-learn's NearestNeighbors, as the reference."""
    from sklearn.neighbors import NearestNeighbors
    n = len(query_positions)
    props = {"part_labels": params["part_labels"], "density": params["density"], "E": params["E"], "nu": params["nu"],
             "material_id": params["material_id"], "conf": params["conf"]}
    if len(props["part_labels"]) == n:                          # :236-238
        return tuple(props[name] for name in _ORDER)
    dist, idx = NearestNeighbors(n_neighbors=k_smoothing_neighbors, algorithm="auto").fit(params["pos"]).kneighbors(query_positions)
    far = dist[:, 0] > nn_distance_threshold
    assert int(np.sum(far)) <= 0.1 * n                          # :271
    result = _fallback_values(props, n)
    for i in np.flatnonzero(~far):
        for name, value in _from_neighbours(props, idx[i], dist[i], weighted_assignment).items():
            result[name][i] = value
    return tuple(result[name] for name in _ORDER)


def apply_additional_params(x: np.ndarray, densities, E_values, nu_values, material_ids, size=0.001):
    """One box per particle, applied in order (material_field.py:347-358 + mpm_utils.py:591-610): returns the per-particle
    (E, nu, density, material) after all launches. float32 comparisons like the Warp kernel."""
    x = x.astype(np.float32)
    n = len(x)
    E = np.zeros(n, np.float32); nu = np.zeros(n, np.float32); d = np.zeros(n, np.float32); m = np.zeros(n, np.int32)
    s = np.float32(size)
    for i in range(n):
        inside = np.all((x > x[i] - s) & (x < x[i] + s), axis=1)
        E[inside] = np.float32(E_values[i]); nu[inside] = np.float32(nu_values[i]); d[inside] = np.float32(densities[i]); m[inside] = int(material_ids[i])
    return E, nu, d, m
