"""Batched multi-scene driver (SURVEY.md 8f-4): many scenes through material field -> transfer -> MPM rollout in ONE warm
process per GPU.

The reference chains sub-processes per scene: `generate_neural_segmentation` (pixie/utils.py:724-786) shells out to
`inference_combined.py` (networks re-created, checkpoints re-loaded, Warp / Taichi / torch re-initialised) and to
`map_pred_to_coords.py` (PLY round trip), then `run_physics_simulation` (pipeline.py:188-244) shells out to
`gs_simulation.py`, which re-reads the PLY, runs a CPU kNN and the substep loop from Python. Tens of seconds of start-up
per scene, none of it arithmetic. Here the two networks and one solver stay resident and a scene is:

    grid (fp16 NDHWC .npy or tensor) --predict_packed_host_stream--> (3+8, D,D,D) field     [inference_combined.py:122-199]
    field + mask --extract_material_points--> material point cloud (the PLY's vertex table)   [map_pred_to_coords.py:128-283]
    particles --get_particle_volume / load_initial_data / set_parameters_dict / BCs-->        [gs_simulation.py:464-489]
    kNN smoothing (+ ground / stationary cuboids) + upload (apply_material_field_to_simulation) [material_field.py:295-550]
    frame loop: export positions / covariances in the Gaussians' frame, step_per_frame x p2g2p [gs_simulation.py:585-634]

Function names and argument meaning follow those reference functions; rendering, Hydra and the file layout stay outside.
Scenes shard over ranks like the reference's `DistributedSampler(shuffle=False)` (dist_utils.shard_scenes); there is no
data-path collective.
"""
from __future__ import annotations

import os
from dataclasses import dataclass, field
from typing import Callable, Dict, Iterable, List, Optional, Sequence

import numpy as np
import torch

from . import dist_utils, frame_export, material_transfer, voxel_io
from .inference import MaterialFieldPredictor
from .mpm_solver_warp import MPM_Simulator_WARP


@dataclass
class Scene:
    """One object: where its voxel grid lives and what the simulation needs (what gs_simulation.py reads from its config
    JSON and the trained Gaussians; positions / covariances are in the Gaussians' own frame)."""
    name: str
    grid: object                                   # path of clip_features_features.npy, or a pinned fp16 (1, D, D, D, C) tensor
    mask: object                                   # path of clip_features_mask.npy, or a (D, D, D) tensor (occupied where > 0)
    min_bounds: Sequence[float]
    max_bounds: Sequence[float]
    particles: torch.Tensor                        # (N, 3) Gaussian centres to simulate
    cov: Optional[torch.Tensor] = None             # (N, 6) upper-triangular covariances
    material_params: Dict = field(default_factory=dict)   # set_parameters_dict keys: n_grid, grid_lim, material, g, density, E, nu, ...
    bc_params: List[Dict] = field(default_factory=list)   # [{"type": "bounding_box"}, {"type": "cuboid", ...}, ...]
    time_params: Dict = field(default_factory=lambda: {"substep_dt": 1e-4, "frame_dt": 4e-2, "frame_num": 4})
    rotation_matrices: Sequence[torch.Tensor] = ()
    z_shift_value: float = 0.0
    k_smoothing_neighbors: int = 10
    nn_distance_threshold: float = 0.1
    # the ground and stationary-cluster cuboids of apply_material_field_to_simulation (material_field.py:325-336); off by
    # default. fix_ground / only_handle_largest_cluster (decode_param.py defaults) are read only when it is on.
    material_field_bcs: bool = False
    fix_ground: bool = True
    only_handle_largest_cluster: bool = True


def transform2origin(position_tensor: torch.Tensor):
    """utils/transformation_utils.py:6-16 (elementwise torch, stays on the device the tensor is on)."""
    min_pos = torch.min(position_tensor, 0)[0]
    max_pos = torch.max(position_tensor, 0)[0]
    max_diff = torch.max(max_pos - min_pos)
    original_mean_pos = (min_pos + max_pos) / 2.0
    scale = 1.0 / max_diff
    return (position_tensor - original_mean_pos) * scale, scale, original_mean_pos


def apply_rotations(position_tensor: torch.Tensor, rotation_matrices) -> torch.Tensor:
    for R in rotation_matrices:                    # transformation_utils.py:54-56, 90-93
        position_tensor = torch.mm(position_tensor, R.to(position_tensor).T)
    return position_tensor


def set_boundary_conditions(mpm_solver: MPM_Simulator_WARP, bc_params: Iterable[Dict], time_params: Dict):
    """The subset of utils/decode_param.set_boundary_conditions (:277-396) whose BCs do not carry per-particle masks plus
    the masked ones the solver shim implements; unknown types raise like the reference's final else."""
    for bc in bc_params:
        t = bc["type"]
        kw = {k: v for k, v in bc.items() if k != "type"}
        if t == "bounding_box":
            mpm_solver.add_bounding_box(**kw)
        elif t == "cuboid":
            mpm_solver.set_velocity_on_cuboid(**kw)
        elif t == "surface_collider":
            mpm_solver.add_surface_collider(**kw)
        elif t == "particle_impulse":
            mpm_solver.add_impulse_on_particles(dt=time_params["substep_dt"], **kw)
        elif t == "enforce_particle_translation":
            mpm_solver.enforce_particle_velocity_translation(**kw)
        elif t == "enforce_particle_velocity_rotation":
            mpm_solver.enforce_particle_velocity_rotation(**kw)
        elif t == "release_particles_sequentially":
            mpm_solver.release_particles_sequentially(**kw)
        else:
            raise TypeError("Undefined BC type")


class SceneBatchDriver:
    """Networks + solver resident on one GPU; `run(scenes)` processes this rank's share of the scenes."""

    def __init__(self, feature_channels: int, grid_size: int = 64, device="cuda:0", precision: str = "fp16e5",
                 seg_state_dict=None, cont_state_dict=None, ranges: Optional[Dict[str, float]] = None, **unet_cfg):
        self.device = torch.device(device)
        self.predictor = MaterialFieldPredictor(feature_channels=feature_channels, grid_size=grid_size, device=device, max_batch=1,
                                                precision=precision, **unet_cfg)
        if seg_state_dict is not None:
            self.predictor.load_state_dicts(seg_state_dict, cont_state_dict)
        self.ranges = ranges
        self.grid_size = grid_size

    # ------------------------------------------------------------------------------ neural half
    def generate_neural_segmentation(self, scenes: Sequence[Scene], out_dir: Optional[str] = None) -> List[Dict[str, torch.Tensor]]:
        """Material point clouds of `scenes` (what mapped_preds.ply holds in the reference, utils.py:724-786), the voxel grids
        streamed through the host pipeline (H2D of scene i+1 under the networks of scene i). With `out_dir`, also writes
        `<out_dir>/<scene>/sample_0_pred.npy` exactly as save_predictions does (inference_combined.py:173-199)."""
        def grids():
            for sc in scenes:
                if isinstance(sc.grid, str):
                    yield voxel_io.load_feature_grid(sc.grid)
                else:
                    yield sc.grid
        packed = self.predictor.predict_packed_host_stream(grids())
        clouds = []
        for sc, field_host in zip(scenes, packed):
            mask = voxel_io.load_mask(sc.mask) if isinstance(sc.mask, str) else sc.mask
            if out_dir is not None:
                d = os.path.join(out_dir, sc.name)
                os.makedirs(d, exist_ok=True)
                np.save(os.path.join(d, "sample_0_pred.npy"), field_host[0].numpy())
            clouds.append(material_transfer.extract_material_points(field_host[0].to(self.device), mask.to(self.device),
                                                                   sc.min_bounds, sc.max_bounds, self.ranges))
        return clouds

    # ------------------------------------------------------------------------------ physics half
    def run_physics_simulation(self, sc: Scene, cloud: Dict[str, torch.Tensor],
                               on_frame: Optional[Callable[[int, torch.Tensor, Optional[torch.Tensor]], None]] = None) -> Dict:
        """One scene's rollout (gs_simulation.py:395-634 without the rasteriser): returns the per-frame render-space positions
        (and covariances when the scene has them) unless `on_frame(frame, pos, cov)` consumes them."""
        dev = self.device
        mp, tp = dict(sc.material_params), sc.time_params
        n_grid, grid_lim = int(mp.get("n_grid", 64)), float(mp.get("grid_lim", 2.0))
        rots = [r.to(dev, torch.float32) for r in sc.rotation_matrices]
        rotated = apply_rotations(sc.particles.to(dev, torch.float32), rots)
        transformed, scale_origin, original_mean_pos = transform2origin(rotated)
        pos0 = transformed + torch.tensor([1.0, 1.0, 1.0 + sc.z_shift_value], device=dev)          # shift2center111 :103-105
        vol = frame_export.get_particle_volume(pos0, n_grid, grid_lim / n_grid, unifrom=mp.get("material") == "sand")
        cov0 = None
        if sc.cov is not None:
            # apply_cov_rotations(init_cov, R) * scale^2  (gs_simulation.py:438): R C R^T per rotation, on the device
            c = sc.cov.to(dev, torch.float32)
            m = torch.stack([c[:, 0], c[:, 1], c[:, 2], c[:, 1], c[:, 3], c[:, 4], c[:, 2], c[:, 4], c[:, 5]], dim=1).view(-1, 3, 3)
            for R in rots:
                m = R @ m @ R.T
            cov0 = torch.stack([m[:, 0, 0], m[:, 0, 1], m[:, 0, 2], m[:, 1, 1], m[:, 1, 2], m[:, 2, 2]], dim=1) * (scale_origin ** 2)
        solver = MPM_Simulator_WARP(10, device=str(dev))
        solver.load_initial_data_from_torch(pos0, vol, cov0, n_grid=n_grid, grid_lim=grid_lim, device=str(dev))
        solver.set_parameters_dict(mp, device=str(dev))
        set_boundary_conditions(solver, sc.bc_params, tp)
        bc_conditions = []
        if sc.material_field_bcs:
            # apply_material_field_to_simulation (material_field.py:295-341): kNN, ground + stationary-cluster cuboids, upload
            props, bc_conditions = material_transfer._apply_material_field(
                solver, cloud, str(dev), scale_origin, original_mean_pos, rots, sc.only_handle_largest_cluster, sc.fix_ground, 0.05, 0.5,
                sc.k_smoothing_neighbors, sc.nn_distance_threshold, False, exact_box_semantics=False)
        else:
            # the same without the ground / stationary-cluster BCs
            q, _ = frame_export.render_frame_transform(solver.export_particle_x_to_torch(), None, 0.0, scale_origin, original_mean_pos, rots)
            props = material_transfer.perform_knn_smoothing(q, cloud, sc.k_smoothing_neighbors, sc.nn_distance_threshold)
            material_transfer.apply_material_properties_to_solver(solver, props[1], props[2], props[3], props[4], device=str(dev),
                                                                  exact_box_semantics=False)
        substep_dt = tp["substep_dt"]
        step_per_frame = int(tp["frame_dt"] / substep_dt)                                           # float division like :627
        frames_pos, frames_cov = [], []
        for frame in range(int(tp["frame_num"])):
            pos = solver.export_particle_x_to_torch()
            cov = solver.export_particle_cov_to_torch().view(-1, 6) if sc.cov is not None else None
            pr, cr = frame_export.render_frame_transform(pos, cov, sc.z_shift_value, scale_origin, original_mean_pos, rots)
            if on_frame is not None:
                on_frame(frame, pr, cr)
            else:
                frames_pos.append(pr.clone())
                frames_cov.append(None if cr is None else cr.clone())
            solver.p2g2p_n(step_per_frame, substep_dt)
        return {"name": sc.name, "n_particles": int(pos0.shape[0]), "frames_pos": frames_pos, "frames_cov": frames_cov,
                "material_ids": props[4], "E": props[2], "substeps": step_per_frame * int(tp["frame_num"]), "time": solver.time,
                "bc_conditions": bc_conditions}

    # ------------------------------------------------------------------------------ batch
    def run(self, scenes: Sequence[Scene], out_dir: Optional[str] = None) -> List[Dict]:
        """This rank's share of `scenes` end to end; returns one record per processed scene (in scene order)."""
        rank, world, _ = dist_utils.env_rank_world()
        mine = [scenes[i] for i in dict.fromkeys(dist_utils.shard_scenes(len(scenes), rank, world))]
        clouds = self.generate_neural_segmentation(mine, out_dir)
        return [self.run_physics_simulation(sc, cl) for sc, cl in zip(mine, clouds)]
