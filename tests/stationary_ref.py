"""ORACLE (test infrastructure, not product code): CPU restatement of the reference's boundary-condition helpers of the
material-field hand-off, with numpy and scikit-learn as the reference uses them.

  handle_stationary_clusters    third_party/PhysGaussian/material_field.py:365-480   (sklearn DBSCAN, float32 numpy boxes)
  fix_to_ground                 third_party/PhysGaussian/material_field.py:485-550

tests/golden/make_stationary_golden.py executes the reference's own functions to write tests/golden/stationary_golden.npz;
tests/test_stationary_bcs.py holds this file to that fixture bit-exactly and the device path (pixie_b200.material_transfer)
to both. `solver` only needs `set_velocity_on_cuboid(point, size, velocity, start_time, end_time, reset)`.
"""
from __future__ import annotations

import numpy as np

STATIONARY_ID = 6                                                                                       # mpm_solver_warp.py:10-26


def dbscan_labels(positions: np.ndarray, eps: float, min_samples: int) -> np.ndarray:
    from sklearn.cluster import DBSCAN
    return DBSCAN(eps=eps, min_samples=min_samples).fit_predict(positions)


def handle_stationary_clusters(solver, positions, material_ids, eps=0.03, min_samples=10, start_time=0.0, end_time=1e6, buffer=0.0,
                               only_handle_largest_cluster=True):
    pts = positions[np.asarray(material_ids) == STATIONARY_ID]
    if len(pts) == 0:
        return []
    labels = dbscan_labels(pts, eps, min_samples)
    valid = np.unique(labels)
    valid = valid[valid != -1]
    if len(valid) == 0:
        return []
    sizes = {int(lab): int(np.sum(labels == lab)) for lab in valid}
    if only_handle_largest_cluster and len(valid) > 1:
        valid = [max(sizes.items(), key=lambda kv: kv[1])[0]]          # first maximum in label order
    out = []
    for lab in valid:
        cp = pts[labels == lab]
        lo, hi = cp.min(axis=0), cp.max(axis=0)
        center = 0.5 * (lo + hi)
        halfsize = 0.5 * (hi - lo)
        halfsize += buffer                                              # float32: `buffer` is a weak Python float
        solver.set_velocity_on_cuboid(point=center.tolist(), size=halfsize.tolist(), velocity=[0.0, 0.0, 0.0], start_time=start_time,
                                      end_time=end_time, reset=1)
        out.append({"type": "stationary_cluster", "cluster_id": int(lab), "point": center.tolist(), "size": halfsize.tolist(),
                    "velocity": [0.0, 0.0, 0.0], "start_time": start_time, "end_time": end_time, "reset": 1, "cluster_size": sizes[int(lab)]})
    return out


def fix_to_ground(solver, positions, delta_z=0.02, buffer_xy=0.5, min_z_percentile=1, start_time=0.0, end_time=1e6):
    lo, hi = positions[:, :2].min(axis=0), positions[:, :2].max(axis=0)
    size = hi - lo
    min_z = np.percentile(positions[:, 2], min_z_percentile) if min_z_percentile > 1 else positions[:, 2].min()
    point = [(lo[0] + hi[0]) / 2, (lo[1] + hi[1]) / 2, min_z + delta_z / 2]
    half = [size[0] / 2 + buffer_xy, size[1] / 2 + buffer_xy, delta_z / 2]
    solver.set_velocity_on_cuboid(point=point, size=half, velocity=[0.0, 0.0, 0.0], start_time=start_time, end_time=end_time, reset=1)
    return [{"type": "ground", "point": point, "size": half, "velocity": [0.0, 0.0, 0.0], "start_time": start_time, "end_time": end_time,
             "reset": 1}]


class RecordingSolver:
    """Collects set_velocity_on_cuboid calls as the float32 values a solver's collider table holds."""

    def __init__(self):
        self.colliders = []

    def set_velocity_on_cuboid(self, point, size, velocity, start_time=0.0, end_time=999.0, reset=0):
        self.colliders.append(collider_row(point, size, velocity, start_time, end_time, reset))


def collider_row(point, size, velocity, start_time, end_time, reset) -> np.ndarray:
    """point, size, velocity, start_time, end_time, reset as float32 [12] (the Dirichlet_collider fields)."""
    return np.array(list(point) + list(size) + list(velocity) + [start_time, end_time, reset], dtype=np.float32)
