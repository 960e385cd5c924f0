"""Material field -> MPM particles, on the device (SURVEY.md 8f-1).

The reference goes through files and the CPU: `map_pred_to_ply` (pixie/voxel/map_pred_to_coords.py:128-283) unscales the
packed (3+8, D, D, D) prediction, keeps the occupied voxels and writes a PLY; `apply_material_field_to_simulation`
(PG/material_field.py:295-341) reads it back, runs a scikit-learn kNN (k = 10) with a Python loop over every particle
(`perform_knn_smoothing`, :228-293) and uploads the result with one kernel launch per particle
(`_apply_material_properties_to_solver`, :343-363). Here the same three steps stay on the GPU:

    field = extract_material_points(pred, mask, min_bounds, max_bounds, ranges)      # = the PLY's vertex table
    props = perform_knn_smoothing(query_positions, field)                            # same tuple as the reference returns
    apply_material_properties_to_solver(mpm_solver, *props[1:5])

`apply_material_field_to_simulation` chains the whole hand-off as the reference does (kNN smoothing, the ground cuboid of
`fix_to_ground`, the stationary-cluster cuboids of `handle_stationary_clusters`, upload); the DBSCAN behind the latter runs
on the device (csrc/cluster.cu) instead of scikit-learn on the host.

Names, argument meaning, defaults and return order follow the reference functions. No CPU fallback (`fix_to_ground` is
host arithmetic on a min / max and runs wherever its tensor lives).
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib, frame_export
from .mpm_solver_warp import MAX_BCS, get_material_name

#: normalization_stats/normalization_ranges.yaml p1/p99 (SURVEY.md 8a; config keys training.{density,E,nu}_{min,max})
DEFAULT_RANGES = dict(density_min=1.703, density_max=3.871, E_min=3.018, E_max=10.882, nu_min=0.2103, nu_max=0.4493)
#: material_field.py:16-23
DEFAULT_VALUES = {"density": 1000.0, "E": 5000.0, "nu": 0.3, "part_label": 0, "material_id": "stationary"}


def extract_material_points(pred: torch.Tensor, mask: torch.Tensor, min_bounds: Sequence[float], max_bounds: Sequence[float],
                            ranges: Optional[Dict[str, float]] = None) -> Dict[str, torch.Tensor]:
    """`unscale_prediction` + the vertex table of `map_pred_to_ply` (map_pred_to_coords.py:41-75, 198-245).

    pred: (3 + n_classes, D, D, D) float32 cuda — 3 continuous channels in ~[-1, 1] followed by class scores / one-hot;
    mask: (D, D, D), occupied where > 0. Returns the `params` dict PG/material_field.py works on: pos (M,3), density, E, nu,
    material_id, part_labels (= material_id, map_pred_to_coords.py:232), conf — device tensors, voxels in C order."""
    _lib.require_device()
    r = dict(DEFAULT_RANGES if ranges is None else ranges)
    if pred.dim() != 4 or pred.shape[1] != pred.shape[2] or pred.shape[2] != pred.shape[3] or pred.shape[0] < 4:
        raise ValueError(f"pred must be (3 + n_classes, D, D, D), got {tuple(pred.shape)}")
    D, K = int(pred.shape[1]), int(pred.shape[0]) - 3
    if tuple(mask.shape) != (D, D, D):
        raise ValueError(f"Mask shape {tuple(mask.shape)} does not match grid shape {(D, D, D)}")      # map_pred_to_coords.py:190-191
    _lib.require_cuda("extract_material_points", pred)
    dev = pred.device
    pred = pred.detach().to(torch.float32).contiguous()
    maskf = mask.detach().to(dev, torch.float32).contiguous()
    n = D ** 3
    pos = torch.empty((n, 3), dtype=torch.float32, device=dev)
    dens, E, nu, conf = (torch.empty(n, dtype=torch.float32, device=dev) for _ in range(4))
    mat = torch.empty(n, dtype=torch.int32, device=dev)
    rng = (C.c_double * 6)(r["density_min"], r["density_max"], r["E_min"], r["E_max"], r["nu_min"], r["nu_max"])
    bmin = (C.c_double * 3)(*[float(v) for v in min_bounds])
    bmax = (C.c_double * 3)(*[float(v) for v in max_bounds])
    cnt = C.c_int(0)
    _lib.call("pixie_field_extract", dev, pred, K, maskf, D, rng, bmin, bmax, pos, dens, E, nu, mat, conf, C.byref(cnt))
    m = cnt.value
    return {"pos": pos[:m], "density": dens[:m], "E": E[:m], "nu": nu[:m], "material_id": mat[:m], "part_labels": mat[:m].clone(),
            "conf": conf[:m]}


def perform_knn_smoothing(query_positions: torch.Tensor, params: Dict[str, torch.Tensor], k_smoothing_neighbors: int = 10,
                          nn_distance_threshold: float = 0.1, weighted_assignment: bool = False
                          ) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
    """material_field.py:228-293. `query_positions`: (Np, 3) MPM particle positions ALREADY in the material field's frame
    (the reference applies undoshift2center111 / undotransform2origin / inverse rotations first, :245-248 — elementwise torch).
    Returns (part_labels, densities, E_values, nu_values, material_ids, conf_values) like the reference."""
    n_particles = int(query_positions.shape[0])
    keys = ("part_labels", "density", "E", "nu", "material_id", "conf")
    if len(params["part_labels"]) == n_particles:                                   # :236-238 no smoothing needed
        return tuple(params[k] for k in keys)
    m = int(params["pos"].shape[0])
    if int(k_smoothing_neighbors) > m:                                              # NearestNeighbors.kneighbors raises here too
        raise ValueError(f"Expected n_neighbors <= n_samples_fit, but n_neighbors = {k_smoothing_neighbors}, n_samples_fit = {m}")
    _lib.require_device()
    _lib.require_cuda("perform_knn_smoothing", query_positions)
    dev = query_positions.device
    f = lambda t: t.detach().to(dev, torch.float32).contiguous()
    i = lambda t: t.detach().to(dev, torch.int32).contiguous()
    q, pos = f(query_positions), f(params["pos"])
    dens, E, nu, conf = f(params["density"]), f(params["E"]), f(params["nu"]), f(params["conf"])
    mat, part = i(params["material_id"]), i(params["part_labels"])
    # get_defaults (:38-50): mean of each continuous property, "stationary" material, part label 0
    mean = lambda t, key: float(t.mean().item()) if m > 0 else float(DEFAULT_VALUES.get(key, 0.0))
    defaults = (C.c_float * 4)(mean(dens, "density"), mean(E, "E"), mean(nu, "nu"), mean(conf, "conf"))
    o_d, o_E, o_nu, o_c = (torch.empty(n_particles, dtype=torch.float32, device=dev) for _ in range(4))
    o_m, o_p = (torch.empty(n_particles, dtype=torch.int32, device=dev) for _ in range(2))
    too_far = C.c_int(0)
    _lib.call("pixie_knn_assign", dev, q, n_particles, pos, dens, E, nu, mat, part, conf, m, int(k_smoothing_neighbors),
              float(nn_distance_threshold), int(bool(weighted_assignment)), defaults, int(get_material_name("stationary")),
              int(DEFAULT_VALUES["part_label"]), o_d, o_E, o_nu, o_m, o_p, o_c, C.byref(too_far))
    n_too_far = too_far.value
    print(f"Particles too far from nearest neighbor: {n_too_far}, Assigned: {n_particles - n_too_far}")
    assert n_too_far <= 0.1 * n_particles, (f"[CRITICAL] More than 10% of particles are too far from nearest neighbor. "
                                            f"Distance threshold: {nn_distance_threshold}.")           # :271
    return o_p, o_d, o_E, o_nu, o_m, o_c


def apply_material_properties_to_solver(mpm_solver, densities: torch.Tensor, E_values: torch.Tensor, nu_values: torch.Tensor,
                                        material_ids: torch.Tensor, device="cuda:0", exact_box_semantics: bool = True):
    """material_field.py:343-363. The reference passes one tiny box (+-0.001) per particle to `apply_additional_params`
    (mpm_utils.py:591-610), so a particle takes the properties of the LAST particle whose box contains it — itself unless a
    later particle sits within 1e-3 of it on every axis. `exact_box_semantics=True` reproduces that (one launch over all
    boxes, O(Np^2) box tests on the device); False writes each particle's own properties (what the loop intends)."""
    n = mpm_solver.n_particles
    dev = mpm_solver._device
    f = lambda t: t.detach().to(dev, torch.float32).contiguous()
    d, E, nu = f(densities), f(E_values), f(nu_values)
    mat = material_ids.detach().to(dev, torch.int32).contiguous()
    assert d.numel() == n and E.numel() == n and nu.numel() == n and mat.numel() == n
    if exact_box_semantics:
        x = mpm_solver.mpm_state.particle_x.tensor.reshape(n, 3)
        size = torch.full((n, 3), 0.001, dtype=torch.float32, device=dev)
        boxes = torch.cat([x, size, E.view(n, 1), nu.view(n, 1), d.view(n, 1), mat.to(torch.float32).view(n, 1)], dim=1).contiguous()
        mpm_solver._apply_additional_params_boxes(boxes)
    else:
        mpm_solver.mpm_model.E = E
        mpm_solver.mpm_model.nu = nu
        mpm_solver.mpm_state.particle_density = d
        mpm_solver.mpm_state.particle_material = mat
        _lib.check(_lib.load().pixie_mpm_compute_mass(mpm_solver._handle, mpm_solver._stream()))
    mpm_solver.finalize_mu_lam(device=device)


# ------------------------------------------------------------------------------------------ boundary conditions of the hand-off
def _dbscan(positions: torch.Tensor, eps: float, min_samples: int, select: Optional[torch.Tensor], select_id: int):
    """(labels, index, n_clusters) of pixie_dbscan: index[t] = particle index of the t-th selected point."""
    if not float(eps) > 0.0:
        raise ValueError(f"eps must be > 0, got {eps}")
    if int(min_samples) < 1:
        raise ValueError(f"min_samples must be >= 1, got {min_samples}")
    _lib.require_device()
    if not torch.is_tensor(positions) or not positions.is_cuda:
        raise _lib.PixieError("dbscan requires CUDA tensors; there is no CPU fallback")
    dev = positions.device
    p = positions.detach().reshape(-1, 3).to(torch.float32).contiguous()
    n = int(p.shape[0])
    ids = None
    if select is not None:
        ids = torch.as_tensor(select).detach().reshape(-1).to(dev, torch.int32).contiguous()
        if ids.numel() != n:
            raise ValueError(f"select has {ids.numel()} entries for {n} points")
    index = torch.empty(n, dtype=torch.int32, device=dev)
    labels = torch.empty(n, dtype=torch.int32, device=dev)
    m, k = C.c_int(0), C.c_int(0)
    _lib.call("pixie_dbscan", dev, p, n, ids, int(select_id), float(eps), int(min_samples), index, labels, C.byref(m), C.byref(k))
    return labels[:m.value], index[:m.value], k.value


def _cluster_stats(positions: torch.Tensor, index: torch.Tensor, labels: torch.Tensor, n_clusters: int):
    """Host float32 / int arrays: (sizes [K], bbox_min [K, 3], bbox_max [K, 3]) of the clusters `_dbscan` found."""
    dev = positions.device
    p = positions.detach().reshape(-1, 3).to(torch.float32).contiguous()
    sizes = torch.empty(n_clusters, dtype=torch.int32, device=dev)
    lo, hi = (torch.empty((n_clusters, 3), dtype=torch.float32, device=dev) for _ in range(2))
    _lib.call("pixie_cluster_stats", dev, p, index, labels, int(labels.numel()), int(n_clusters), sizes, lo, hi)
    return sizes.cpu().numpy(), lo.cpu().numpy(), hi.cpu().numpy()


def dbscan(positions: torch.Tensor, eps: float, min_samples: int, select: Optional[torch.Tensor] = None,
           select_id: int = get_material_name("stationary")) -> torch.Tensor:
    """`sklearn.cluster.DBSCAN(eps, min_samples).fit_predict(positions[select == select_id])` on the device (all of `positions`
    when `select` is None): int32 labels of the selected points in particle order, -1 for noise. Neighbourhoods use fp64
    squared distances of the float32 positions (<= eps^2, the point itself counted), like scikit-learn's KD-tree."""
    return _dbscan(positions, eps, min_samples, select, select_id)[0]


def _device_tensor(x, dev) -> torch.Tensor:
    return x.detach().to(dev) if torch.is_tensor(x) else torch.as_tensor(np.asarray(x), device=dev)


def handle_stationary_clusters(mpm_solver, positions, material_ids, eps=0.03, min_samples=10, start_time=0.0, end_time=1e6, buffer=0.0,
                               only_handle_largest_cluster=True, debug_output_dir="stationary_clusters_debug", debug=False) -> List[Dict]:
    """material_field.py:365-480: DBSCAN over the particles whose material id is "stationary" and one zero-velocity cuboid
    (reset=1) around the bounding box (+ `buffer`) of the largest cluster (first one on ties), or of every cluster. Returns
    the reference's list of BC dicts. Centre and half-size are computed in float32 numpy from the device bounding box, so
    they are the reference's values bit for bit. `debug` / `debug_output_dir` are accepted but nothing is written (the
    reference always writes stationary_particles.ply). With `only_handle_largest_cluster=False`, clusters that do not fit the
    solver's BC table raise `PixieError` before any is registered."""
    dev = mpm_solver._device
    pos = _device_tensor(positions, dev)
    labels, index, n_clusters = _dbscan(pos, eps, min_samples, _device_tensor(material_ids, dev), get_material_name("stationary"))
    if labels.numel() == 0 or n_clusters == 0:          # no stationary particles / all of them noise
        return []
    sizes, bbox_min, bbox_max = _cluster_stats(pos, index, labels, n_clusters)
    valid_labels = list(range(n_clusters))
    if only_handle_largest_cluster and n_clusters > 1:
        valid_labels = [int(np.argmax(sizes))]          # max(dict.items()): first maximum in label order
    if mpm_solver.n_bcs + len(valid_labels) > MAX_BCS:
        raise _lib.PixieError(f"{len(valid_labels)} stationary clusters do not fit the solver's boundary-condition table "
                              f"({mpm_solver.n_bcs} of {MAX_BCS} entries used); no cluster BC was registered")
    bc_conditions = []
    for cluster_id in valid_labels:
        min_xyz, max_xyz = bbox_min[cluster_id], bbox_max[cluster_id]
        center = 0.5 * (min_xyz + max_xyz)
        halfsize = 0.5 * (max_xyz - min_xyz)
        halfsize += buffer
        mpm_solver.set_velocity_on_cuboid(point=center.tolist(), size=halfsize.tolist(), velocity=[0.0, 0.0, 0.0], start_time=start_time,
                                          end_time=end_time, reset=1)
        bc_conditions.append({"type": "stationary_cluster", "cluster_id": int(cluster_id), "point": center.tolist(), "size": halfsize.tolist(),
                              "velocity": [0.0, 0.0, 0.0], "start_time": start_time, "end_time": end_time, "reset": 1,
                              "cluster_size": int(sizes[cluster_id])})
    return bc_conditions


def fix_to_ground(mpm_solver, positions, delta_z=0.02, buffer_xy=0.5, min_z_percentile=1, start_time=0.0, end_time=1e6) -> List[Dict]:
    """material_field.py:485-550: one thin zero-velocity cuboid (reset=1) under the particles, `delta_z` thick, their xy extent
    plus `buffer_xy` on each side, resting on their lowest z (or the `min_z_percentile` percentile when it is > 1). Only a
    min / max of `positions` (a tensor on any device, or an array) and the reference's float32 host arithmetic."""
    if torch.is_tensor(positions):
        p = positions.detach().reshape(-1, 3)
        lo, hi = torch.stack([p.amin(0), p.amax(0)]).cpu().numpy()
        z = p[:, 2].cpu().numpy() if min_z_percentile > 1 else None
    else:
        p = np.asarray(positions)
        lo, hi = p.min(axis=0), p.max(axis=0)
        z = p[:, 2]
    min_xy, max_xy = lo[:2], hi[:2]
    size_xy = max_xy - min_xy
    min_z = np.percentile(z, min_z_percentile) if min_z_percentile > 1 else lo[2]
    ground_center = [(min_xy[0] + max_xy[0]) / 2, (min_xy[1] + max_xy[1]) / 2, min_z + delta_z / 2]
    ground_halfsize = [size_xy[0] / 2 + buffer_xy, size_xy[1] / 2 + buffer_xy, delta_z / 2]
    mpm_solver.set_velocity_on_cuboid(point=ground_center, size=ground_halfsize, velocity=[0.0, 0.0, 0.0], start_time=start_time,
                                      end_time=end_time, reset=1)
    return [{"type": "ground", "point": ground_center, "size": ground_halfsize, "velocity": [0.0, 0.0, 0.0], "start_time": start_time,
             "end_time": end_time, "reset": 1}]


def _apply_material_field(mpm_solver, params, device, scale_origin, original_mean_pos, rotation_matrices, only_handle_largest_cluster,
                          fix_ground, ground_delta_z, ground_buffer_xy, k_smoothing_neighbors, nn_distance_threshold, weighted_assignment,
                          exact_box_semantics):
    missing = [k for k in ("part_labels", "density", "E", "nu", "material_id", "conf") if k not in params]
    assert not missing, f"Missing required keys: {missing}, Available: {list(params.keys())}"
    x = mpm_solver.export_particle_x_to_torch()
    # the reference's query transform (material_field.py:245-248): undoshift2center111 with its default z shift of 0
    q, _ = frame_export.render_frame_transform(x, None, 0.0, scale_origin, original_mean_pos, list(rotation_matrices or ()))
    props = perform_knn_smoothing(q, params, k_smoothing_neighbors, nn_distance_threshold, weighted_assignment)
    positions = mpm_solver.export_particle_x_to_torch()
    bc_conditions = []
    if fix_ground:
        bc_conditions += fix_to_ground(mpm_solver, positions, ground_delta_z, ground_buffer_xy)
    bc_conditions += handle_stationary_clusters(mpm_solver, positions, props[4], eps=0.03, min_samples=8, start_time=0.0, end_time=1e9,
                                                buffer=0.1, only_handle_largest_cluster=only_handle_largest_cluster)
    apply_material_properties_to_solver(mpm_solver, props[1], props[2], props[3], props[4], device=device,
                                        exact_box_semantics=exact_box_semantics)
    return props, bc_conditions


def apply_material_field_to_simulation(mpm_solver, params, device="cuda:0", scale_origin=None, original_mean_pos=None, rotation_matrices=None,
                                       only_handle_largest_cluster=True, fix_ground=True, ground_delta_z=0.05, ground_buffer_xy=0.5,
                                       k_smoothing_neighbors=10, nn_distance_threshold=0.1, weighted_assignment=False, debug=False,
                                       exact_box_semantics=True):
    """material_field.py:296-340: kNN smoothing of the material point cloud `params` (extract_material_points) onto the
    solver's particles, then the ground cuboid (`fix_ground`), then the stationary-cluster cuboid(s) (DBSCAN eps 0.03,
    min_samples 8, buffer 0.1), then the per-particle upload — in the reference's order, on the particles' setup positions.
    `scale_origin` / `original_mean_pos` / `rotation_matrices` are what transform2origin / the rotations produced. Returns
    (conf_values, bc_conditions). `exact_box_semantics`: see apply_material_properties_to_solver."""
    props, bc_conditions = _apply_material_field(mpm_solver, params, device, scale_origin, original_mean_pos, rotation_matrices,
                                                 only_handle_largest_cluster, fix_ground, ground_delta_z, ground_buffer_xy,
                                                 k_smoothing_neighbors, nn_distance_threshold, weighted_assignment, exact_box_semantics)
    return props[5], bc_conditions
