"""Generates tests/golden/stationary_golden.npz by EXECUTING THE REFERENCE'S OWN `handle_stationary_clusters`, `fix_to_ground`
and `apply_material_field_to_simulation` (PG/material_field.py:296-550). PIXIE_REFERENCE names a checkout of the reference:

    python tests/golden/make_stationary_golden.py

The function sources are pulled out of the reference file with make_transfer_golden.extract and run on the reference's own
solver over the warp stand-in (tests/golden/_fake_warp.py), with the real numpy, torch and scikit-learn. The `DBSCAN` they see
is scikit-learn's, wrapped to record the labels it returns. Recorded per scenario: inputs, DBSCAN labels, the returned BC
dicts (JSON) and the reference solver's `collider_params` as float32 rows (tests/stationary_ref.collider_row layout).
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import make_transfer_golden as MTG  # noqa: E402  (installs the warp stand-in, imports the reference solver)
from stationary_ref import collider_row  # noqa: E402
from sklearn.cluster import DBSCAN  # noqa: E402
from sklearn.neighbors import NearestNeighbors  # noqa: E402
from collections import Counter  # noqa: E402

EPS, MIN_SAMPLES = 0.03, 8


class _RecordingDBSCAN(DBSCAN):
    captured = []

    def fit_predict(self, X, y=None, sample_weight=None):
        labels = super().fit_predict(X, y, sample_weight)
        _RecordingDBSCAN.captured.append(np.asarray(labels).copy())
        return labels


def _namespace():
    tns = {"torch": MTG._TorchCPU(), "np": np}
    MTG.extract(MTG.PG + "/utils/transformation_utils.py",
                ["undotransform2origin", "undoshift2center111", "apply_inverse_rotation", "apply_inverse_rotations", "apply_rotation",
                 "apply_rotations", "shift2center111"], tns)
    ns = {"np": np, "os": os, "torch": torch, "Counter": Counter, "NearestNeighbors": NearestNeighbors, "DBSCAN": _RecordingDBSCAN,
          "tqdm": lambda it, **kw: it, "get_material_name": MTG.REFMPM.get_material_name, "save_points_as_ply": lambda *a, **kw: None,
          "save_dbscan_debug_data": lambda *a, **kw: None}
    for k in ("undotransform2origin", "undoshift2center111", "apply_inverse_rotations"):
        ns[k] = tns[k]
    MTG.extract(MTG.PG + "/material_field.py",
                ["DEFAULT_VALUES", "MaterialProperties", "transform_to_original_coordinates", "scene_bounds", "extract_material_properties",
                 "perform_knn_smoothing", "_apply_material_properties_to_solver", "handle_stationary_clusters", "fix_to_ground",
                 "apply_material_field_to_simulation"], ns)
    return ns, tns


def _ref_solver(n=8):
    return MTG.REFMPM.MPM_Simulator_WARP(n, n_grid=16, grid_lim=2.0, device="cpu")


def _colliders(s):
    rows = [collider_row(c.point.a, [float(v) for v in c.size], c.velocity.a, c.start_time, c.end_time, c.reset) for c in s.collider_params]
    return np.stack(rows) if rows else np.zeros((0, 12), np.float32)


def _plain(v):
    if isinstance(v, (list, tuple)):
        return [_plain(x) for x in v]
    if isinstance(v, (np.floating, float)):
        return float(v)
    if isinstance(v, (np.integer, int)):
        return int(v)
    return v


def _bcs_json(bcs):
    return np.array(json.dumps([{k: _plain(v) for k, v in bc.items()} for bc in bcs]))


def _assert_clear_of_eps(pts):
    """No pair within 1e-12 of eps^2 (fp64): summation order cannot flip a neighbour."""
    p = pts.astype(np.float64)
    d = p[:, None, :] - p[None, :, :]
    d2 = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
    assert np.abs(d2 - EPS * EPS).min() > 1e-12


def mixed_scene(rng):
    """Stationary structures with interleaved non-stationary particles (material ids 0-5).
      T1, T2   tight balls of 40 points (all core): the size tie for the largest cluster
      X, Y     chains of 20 points, spacing 0.004 (ends have exactly 8 neighbours with themselves), whose ends face each other
               0.056 apart with the border point P halfway: within eps of one core end of each, 3 neighbours itself
      Q8       8 points within eps of each other: exactly min_samples neighbours each (a cluster only if self counts)
      FAR      a clump of 12 at negative coordinates far from everything
      noise    isolated stationary points"""
    f32 = np.float32
    ball = lambda c, n, r: (np.asarray(c) + rng.uniform(-r, r, size=(n, 3))).astype(f32)
    T1 = ball([0.70, 0.70, 0.60], 40, 0.006)
    T2 = ball([1.30, 0.70, 0.60], 40, 0.006)
    chain = lambda start, d: (np.asarray(start) + np.outer(np.arange(20) * 0.004, d)).astype(f32)
    X = chain([0.6, 1.2, 0.9], [-1.0, 0.0, 0.0])[::-1].copy()         # X ends at x = 0.6 (its last point)
    Y = chain([0.656, 1.2, 0.9], [1.0, 0.0, 0.0])                      # Y starts at x = 0.656
    P = np.array([[0.628, 1.2, 0.9]], f32)
    Q8 = ball([1.0, 1.5, 1.3], 8, 0.008)
    FAR = ball([-37.0, 25.0, -6.5], 12, 0.008)
    noise = np.array([[0.3, 0.3, 0.3], [1.7, 1.6, 0.4], [1.0, 0.2, 1.8], [0.2, 1.8, 1.1]], f32)
    stat = np.concatenate([Y, T2, X, P, Q8, T1, FAR, noise])
    n_other = 90
    other = rng.uniform(0.4, 1.6, size=(n_other, 3)).astype(f32)
    other[:20] = T1[:20] + f32(0.001)                                # non-stationary particles inside the structures
    other[20:30] = X[:10] + f32(0.0015)
    x = np.concatenate([stat, other])
    ids = np.concatenate([np.full(len(stat), 6, np.int32), rng.integers(0, 6, size=n_other).astype(np.int32)])
    perm = rng.permutation(len(x))
    return x[perm].copy(), ids[perm].copy()


def main():
    ns, tns = _namespace()
    rng = np.random.default_rng(11)
    blob = {}

    def run_stationary(name, x, ids, **kw):
        _RecordingDBSCAN.captured = []
        s = _ref_solver()
        bcs = ns["handle_stationary_clusters"](s, x, ids, **kw)
        assert len(_RecordingDBSCAN.captured) <= 1
        blob.update({f"{name}/x": x, f"{name}/ids": ids, f"{name}/kwargs": np.array(json.dumps(kw)), f"{name}/bcs": _bcs_json(bcs),
                     f"{name}/colliders": _colliders(s)})
        if _RecordingDBSCAN.captured:
            blob[f"{name}/labels"] = _RecordingDBSCAN.captured[0].astype(np.int32)
        print(name, "->", [(b["cluster_id"], b["cluster_size"]) for b in bcs])
        return bcs

    x, ids = mixed_scene(rng)
    _assert_clear_of_eps(x[ids == 6])
    kw = dict(eps=EPS, min_samples=MIN_SAMPLES, start_time=0.0, end_time=1e9, buffer=0.1)
    run_stationary("mixed_largest", x, ids, only_handle_largest_cluster=True, **kw)
    every = run_stationary("mixed_all", x, ids, only_handle_largest_cluster=False, **kw)
    sizes = sorted(b["cluster_size"] for b in every)
    assert sizes[-1] == sizes[-2] == 40 and 8 in sizes and 21 in sizes and 20 in sizes, sizes      # tie, Q8, X + P, Y
    lab = blob["mixed_all/labels"]
    assert len(set(lab[lab >= 0].tolist())) == 6 and (lab == -1).sum() == 4
    # the reference's own defaults (min_samples 10, no buffer): Q8 is noise then
    run_stationary("mixed_defaults", x, ids, only_handle_largest_cluster=False)
    # all noise: stationary points 0.1 apart
    g = np.stack(np.meshgrid(*[np.arange(4) * 0.1 + 0.8] * 3, indexing="ij"), -1).reshape(-1, 3).astype(np.float32)
    run_stationary("all_noise", g, np.full(len(g), 6, np.int32), only_handle_largest_cluster=False, **kw)
    run_stationary("none", x, np.where(ids == 6, 0, ids).astype(np.int32), **kw)

    # ---------------------------------------------------------------- fix_to_ground
    for name, args in (("ground_driver", dict(delta_z=0.05, buffer_xy=0.5)), ("ground_defaults", {}),
                       ("ground_p5", dict(delta_z=0.05, buffer_xy=0.5, min_z_percentile=5))):
        s = _ref_solver()
        bcs = ns["fix_to_ground"](s, x, **args)
        blob.update({f"{name}/x": x, f"{name}/kwargs": np.array(json.dumps(args)), f"{name}/bcs": _bcs_json(bcs),
                     f"{name}/colliders": _colliders(s)})
        print(name, "->", bcs[0]["point"], bcs[0]["size"])

    # ---------------------------------------------------------------- apply_material_field_to_simulation (few hundred particles)
    # material field: a "pot" (stationary, lower half) under a jelly crown, in the field's own frame
    fp = rng.uniform(-0.06, 0.06, size=(900, 3)).astype(np.float32)
    fid = np.where(fp[:, 2] < -0.01, 6, 0).astype(np.int32)
    fparams = {"pos": fp, "part_labels": fid.copy(), "material_id": fid, "density": rng.uniform(500, 1500, 900).astype(np.float32),
               "E": (10 ** rng.uniform(4, 6, 900)).astype(np.float32), "nu": rng.uniform(0.25, 0.4, 900).astype(np.float32),
               "conf": rng.uniform(0.5, 1.0, 900).astype(np.float32)}
    n_p = 320
    gp = rng.uniform(-0.05, 0.05, size=(n_p, 3)).astype(np.float32)
    scale, mean = torch.tensor(1.25), torch.tensor([0.01, -0.02, 0.03])
    a = 0.4
    rots = [torch.tensor([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]], dtype=torch.float32)]
    x_sim = tns["shift2center111"](tns["apply_rotations"]((torch.from_numpy(gp) - mean) * scale, rots)).numpy().astype(np.float32)
    vol = rng.uniform(1e-5, 2e-5, size=n_p).astype(np.float32)
    s = MTG.REFMPM.MPM_Simulator_WARP(n_p, n_grid=16, grid_lim=2.0, device="cpu")
    s.load_initial_data_from_torch(torch.from_numpy(x_sim), torch.from_numpy(vol), None, n_grid=16, grid_lim=2.0, device="cpu")
    s.set_parameters_dict({"material": "jelly", "E": 1e5, "nu": 0.3, "density": 1000.0}, device="cpu")
    _assert_clear_of_eps(x_sim)
    _RecordingDBSCAN.captured = []
    conf, bcs = ns["apply_material_field_to_simulation"](s, dict(fparams), "cpu", scale, mean, rots)
    for k, v in fparams.items():
        blob[f"apply/field/{k}"] = v
    blob.update({"apply/x": x_sim, "apply/vol": vol, "apply/scale": scale.numpy(), "apply/mean": mean.numpy(), "apply/rots": torch.stack(rots).numpy(),
                 "apply/conf": np.asarray(conf).copy(), "apply/bcs": _bcs_json(bcs), "apply/colliders": _colliders(s),
                 "apply/labels": _RecordingDBSCAN.captured[0].astype(np.int32),
                 "apply/E": s.mpm_model.E.numpy().copy(), "apply/nu": s.mpm_model.nu.numpy().copy(),
                 "apply/density": s.mpm_state.particle_density.numpy().copy(), "apply/material": s.mpm_state.particle_material.numpy().copy(),
                 "apply/mass": s.mpm_state.particle_mass.numpy().copy()})
    print("apply ->", [b["type"] for b in bcs], "stationary particles", int((s.mpm_state.particle_material.numpy() == 6).sum()))
    assert [b["type"] for b in bcs] == ["ground", "stationary_cluster"]

    out = os.path.join(HERE, "stationary_golden.npz")
    np.savez_compressed(out, **blob)
    print("wrote", out, len(blob), "arrays,", os.path.getsize(out) // 1024, "KiB")


if __name__ == "__main__":
    main()
