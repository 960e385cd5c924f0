"""fp64 restatement of the VLM part segmentation (pixie/voxel/segmentation.py), the oracle of pixie_b200.segmentation.

  similarities      run_clip (:98-122) in fp64: unit feature rows against unit query rows, softmax(sims / T), and the
                    labels / scores of clip_part_segmentation (:162-168). torch tensors in, so that a 64^3 grid can be
                    held to it on the device; numpy arrays are accepted too.
  vote_reference    local_post_process_segmentation (:190-226) as the reference runs it: scikit-learn's KDTree and
                    scipy's mode (its tie choice at the k-th distance is scikit-learn's).
  vote_exact        the same vote with the k nearest chosen by (fp64 squared distance, index), brute force.
  kth_distance_gap  per point, whether the k-th and (k+1)-th fp64 distances differ (there the two votes agree).
  knn_table         the K nearest of every point with their d2, one brute-force pass; vote_of and gap_of give the vote and
                    the gap for every k <= K (K - 1 for the gap) from it.
  nearest_exact     the nearest finite float64 vertex of float32 queries by fp64 squared distance, ties to the lowest index.
  save_files        save_segmented_point_cloud (:231-471) in numpy, with scipy's cKDTree for the colours.
"""
from __future__ import annotations

import os

import numpy as np
import torch

TAB10 = ("#1f77b4", "#ff7f0e", "#2ca02c", "#d62728", "#9467bd", "#8c564b", "#e377c2", "#7f7f7f", "#bcbd22", "#17becf")


def similarities(features, query_embs, temperature: float = 0.1):
    """(sims (N, P), probs (N, P), labels (N,), scores (N,)) in fp64 for the float16 feature rows (N, C) and the raw query
    embeddings (P, C). A zero or NaN row gives NaN similarities and probabilities, label 0 (numpy / torch put a NaN first)."""
    f = torch.as_tensor(features).double()
    q = torch.as_tensor(query_embs).to(f.device).double()
    f = f / f.norm(dim=-1, keepdim=True)
    q = q / q.norm(dim=-1, keepdim=True)
    sims = f @ q.T
    probs = torch.softmax(sims / temperature, dim=1)
    labels = torch.argmax(probs, dim=1)
    scores = torch.gather(probs, 1, labels[:, None])[:, 0]
    return sims, probs, labels, scores


def _mode(rows: np.ndarray) -> np.ndarray:
    """Per row, the most frequent value, the smallest on a count tie (scipy.stats.mode's choice)."""
    out = np.empty(len(rows), np.int64)
    for r, row in enumerate(rows):
        vals, counts = np.unique(row, return_counts=True)
        out[r] = vals[np.argmax(counts)]
    return out


def vote_reference(coords: np.ndarray, labels: np.ndarray, k: int = 200) -> np.ndarray:
    from scipy.stats import mode
    from sklearn.neighbors import KDTree
    c = np.asarray(coords)
    _, idx = KDTree(c).query(c, k=k)
    return np.asarray(mode(np.asarray(labels)[idx], axis=1, keepdims=False).mode, np.int64)


def _d2(q: np.ndarray, p: np.ndarray) -> np.ndarray:
    """(len(q), len(p)) fp64 squared distances (dx*dx + dy*dy) + dz*dz, one rounding per operation."""
    q, p = q.astype(np.float64), p.astype(np.float64)
    d = [q[:, None, a] - p[None, :, a] for a in range(3)]
    return (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]


def knn_table(coords: np.ndarray, kmax: int, chunk: int = 512):
    """((N, K) indices, (N, K) fp64 squared distances) of the K = min(kmax, N) nearest points of every point by (fp64 squared
    distance, index). The k nearest for any k <= K are the first k columns, so one table serves many k."""
    c = np.asarray(coords, np.float32)
    K = min(kmax, len(c))
    idx, dist = np.empty((len(c), K), np.int64), np.empty((len(c), K), np.float64)
    for s in range(0, len(c), chunk):
        d2 = _d2(c[s:s + chunk], c)
        o = np.argsort(d2, axis=1, kind="stable")[:, :K]
        idx[s:s + chunk], dist[s:s + chunk] = o, np.take_along_axis(d2, o, axis=1)
    return idx, dist


def knn_exact(coords: np.ndarray, k: int, chunk: int = 512) -> np.ndarray:
    """(N, k) indices of the k nearest points by (fp64 squared distance, index)."""
    return knn_table(coords, k, chunk)[0]


def vote_of(labels: np.ndarray, idx: np.ndarray) -> np.ndarray:
    """The vote over the (N, k) neighbour indices idx: per row the most frequent label, the smallest on a count tie."""
    return _mode(np.asarray(labels, np.int64)[idx])


def vote_exact(coords: np.ndarray, labels: np.ndarray, k: int = 200) -> np.ndarray:
    return vote_of(labels, knn_exact(coords, k))


def gap_of(dist: np.ndarray, k: int) -> np.ndarray:
    """kth_distance_gap from knn_table's distances with at least k + 1 columns (True everywhere when k = N)."""
    return np.ones(len(dist), bool) if k >= len(dist) else dist[:, k - 1] != dist[:, k]


def kth_distance_gap(coords: np.ndarray, k: int, chunk: int = 512) -> np.ndarray:
    """Per point, True where the k-th and (k+1)-th smallest fp64 squared distances differ (True when k = N)."""
    return gap_of(knn_table(coords, k + 1, chunk)[1], k)


def nearest_exact(vertices: np.ndarray, queries: np.ndarray, chunk: int = 512) -> np.ndarray:
    """Vertices with a NaN or Inf coordinate are never chosen; among the finite ones a d2 that overflows to Inf still
    counts (all at Inf: the lowest finite index). -1 for a non-finite query or without finite vertices."""
    v = np.asarray(vertices, np.float64).reshape(-1, 3)
    q = np.asarray(queries, np.float32).reshape(-1, 3)
    out = np.full(len(q), -1, np.int64)
    ok = np.isfinite(v).all(1)
    if not ok.any():
        return out
    fin = np.flatnonzero(ok)
    for s in range(0, len(q), chunk):
        with np.errstate(over="ignore", invalid="ignore"):
            d2 = _d2(q[s:s + chunk], v[ok])
        out[s:s + chunk] = fin[np.argmin(d2, axis=1)]           # argmin: the first of equal minima, Inf included
    out[~np.isfinite(q).all(1)] = -1
    return out


def save_files(coords, part_labels, output_dir, vertices, colors_rgba, part_queries, material_props, grid_shape, mask,
               background_id=7):
    """save_segmented_point_cloud's files, restated in numpy (the colours through cKDTree, as the reference finds them)."""
    from scipy.spatial import cKDTree
    os.makedirs(output_dir, exist_ok=True)
    coords, labels = np.asarray(coords, np.float32), np.asarray(part_labels)
    n = len(coords)
    cols = np.asarray(colors_rgba)
    if cols.max() > 1.0:
        cols = cols / 255.0
    _, idx = cKDTree(np.asarray(vertices, np.float64)).query(coords, k=1)
    rgb = np.zeros((n, 4), np.float32)
    rgb[:, :3] = cols[idx, :3]
    rgb[:, 3] = 1.0
    sem = np.zeros((n, 4), np.float32)
    density, E, nu = np.zeros(n, np.float32), np.zeros(n, np.float32), np.zeros(n, np.float32)
    mid = np.zeros(n, np.int32)
    for i in range(labels.max() + 1):
        m = labels == i
        if not m.any():
            continue
        h = TAB10[i % 10]
        sem[m] = np.array(tuple(int(h[k:k + 2], 16) / 255 for k in (1, 3, 5)) + (1.0,))
        props = material_props[part_queries[i]]
        density[m], E[m], nu[m], mid[m] = props.get("density", 200), props.get("E", 2e6), props.get("nu", 0.4), props.get("material_id", 0)
    dt = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("red", "u1"), ("green", "u1"), ("blue", "u1"), ("alpha", "u1"),
                   ("part_label", "<i4"), ("density", "<f4"), ("E", "<f4"), ("nu", "<f4"), ("material_id", "<i4")])
    ply = {"float": "f4", "uchar": "u1", "int": "i4"}
    inv = {v: k for k, v in ply.items()}
    for name, c in (("segmented_rgb.ply", rgb), ("segmented_semantics.ply", sem)):
        c8 = (c * 255).astype(np.uint8)
        t = np.zeros(n, dt)
        t["x"], t["y"], t["z"] = coords[:, 0], coords[:, 1], coords[:, 2]
        t["red"], t["green"], t["blue"], t["alpha"] = c8.T
        t["part_label"], t["density"], t["E"], t["nu"], t["material_id"] = labels, density, E, nu, mid
        head = ["ply", "format binary_little_endian 1.0", f"element vertex {n}"] + \
               [f"property {inv[dt[f].str[1:]]} {f}" for f in dt.names] + ["end_header"]
        with open(os.path.join(output_dir, name), "wb") as f:
            f.write(("\n".join(head) + "\n").encode("ascii") + t.tobytes())
    grid = np.zeros((*grid_shape, 4), np.float32)
    grid[..., 3] = background_id
    flat = grid.reshape(-1, 4)
    at = np.flatnonzero(np.asarray(mask).astype(bool).ravel())
    flat[at, 0], flat[at, 1], flat[at, 2], flat[at, 3] = density, E, nu, mid
    np.save(os.path.join(output_dir, "material_grid.npy"), grid)
    for i, name in enumerate(("density_grid.npy", "E_grid.npy", "nu_grid.npy", "material_id_grid.npy")):
        np.save(os.path.join(output_dir, name), grid[..., i])
