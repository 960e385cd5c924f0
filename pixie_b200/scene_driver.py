"""Batched multi-scene driver (SURVEY.md 8f-4): many scenes through material field -> transfer -> MPM rollout in ONE warm
process per GPU.

The reference chains sub-processes per scene: `generate_neural_segmentation` (pixie/utils.py:724-786) shells out to
`inference_combined.py` (networks re-created, checkpoints re-loaded, Warp / Taichi / torch re-initialised) and to
`map_pred_to_coords.py` (PLY round trip), then `run_physics_simulation` (pipeline.py:188-244) shells out to
`gs_simulation.py`, which re-reads the PLY, runs a CPU kNN and the substep loop from Python. Tens of seconds of start-up
per scene, none of it arithmetic. Here the two networks and one solver stay resident and a scene is:

    grid (fp16 NDHWC .npy or tensor) --predict_packed_host_stream--> (3+8, D,D,D) field     [inference_combined.py:122-199]
    field + mask --extract_material_points--> material point cloud (the PLY's vertex table)   [map_pred_to_coords.py:128-283]
    Gaussians --fill_particles, when the scene has a particle_filling block-->                [gs_simulation.py:442-462]
    particles --get_particle_volume / load_initial_data / set_parameters_dict / BCs-->        [gs_simulation.py:464-489]
    kNN smoothing (+ ground / stationary cuboids) + upload (apply_material_field_to_simulation) [material_field.py:295-550]
    frame loop: export positions / covariances in the Gaussians' frame, step_per_frame x p2g2p [gs_simulation.py:585-634]
    + the rendered frame, when the scene has SH coefficients and camera parameters         [gs_simulation.py:573-619]
    + the frame's Gaussians as a 3DGS PLY, when the scene sets save_ply                    [gs_simulation.py:621-628]

Function names and argument meaning follow those reference functions; image / video files, Hydra and the file layout stay
outside.
Scenes shard over ranks like the reference's `DistributedSampler(shuffle=False)` (dist_utils.shard_scenes); there is no
data-path collective.
"""
from __future__ import annotations

import contextlib
import os
from dataclasses import dataclass, field
from typing import Callable, Dict, Iterable, List, Optional, Sequence

import numpy as np
import torch

from . import dist_utils, frame_export, gs_render, material_transfer, particle_filling, scene_files, voxel_io
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
    opacity: Optional[torch.Tensor] = None         # (N,) or (N, 1) opacities; needed by particle filling
    # the config's `particle_filling` block (decode_param.py:177-208 defaults applied here); None simulates the Gaussians only
    particle_filling: Optional[Dict] = None
    # preprocessing_params["sim_area"] (gs_simulation.py:419-434): [x0, x1, y0, y1, z0, z1] in the rotated frame. Only the
    # Gaussians strictly inside are simulated; the others are drawn unchanged in every rendered frame. None simulates all.
    sim_area: Optional[Sequence[float]] = None
    # rendering (gs_simulation.py --render_img): with both `shs` and `camera_params`, every frame is rendered from the
    # scene's own opacity and SH coefficients; otherwise nothing is rendered
    shs: Optional[torch.Tensor] = None             # (N, 16, 3) SH coefficients, as GaussianModel.get_features
    sh_degree: int = 3                             # the model's active SH degree
    camera_params: Optional[Dict] = None           # the config's camera keys, raw or decode_camera_params'd
    cameras: object = None                         # the model's cameras.json list, or its path
    white_bg: bool = False
    # --save_ply (gs_simulation.py:621-628): every frame's rendered Gaussians as <ply_dir>/frame_{frame:05d}.ply; needs
    # shs, opacity and cov, not the cameras. to_original_coord (decode_param.py:128-131 default) writes the Gaussians'
    # frame positions; off, the solver's positions (the covariances stay in the Gaussians' frame either way)
    save_ply: bool = False
    to_original_coord: bool = True
    # --optimization_output_path (gs_simulation.py:508-530): per-particle Young's moduli that replace the material field's
    # after the hand-off (one per simulated particle, filled ones included); None keeps the hand-off's
    e_field: Optional[torch.Tensor] = None

    @classmethod
    def from_files(cls, name: str, model_path: str, config: str, sh_degree: int = 3, iteration: int = -1, white_bg: bool = False,
                   save_ply: bool = False, device="cuda:0", grid=None, mask=None, min_bounds=None, max_bounds=None) -> "Scene":
        """The scene gs_simulation.py sets up (:355-437, :491-501) from a trained model directory and a physics config:
        the checkpoint decoded on the device and filtered by the config's opacity_threshold, the config's rotations,
        sim_area, particle_filling, camera keys, to_original_coord, fix_ground / only_handle_largest_cluster / k / nn
        threshold and z shift, the model's cameras.json, and the material field's ground and stationary-cluster BCs,
        which the reference always applies. `grid` / `mask` / bounds are only needed to take the neural path
        (`SceneBatchDriver.run`). A config whose particle filling asks for `smooth` raises NotImplementedError before any
        device work."""
        mp, bc, tp, pp, cp = scene_files.decode_param_json(config)
        check_supported(name, pp)
        g = scene_files.load_gaussians(model_path, pp["opacity_threshold"], sh_degree, iteration, device)
        return cls(name=name, grid=grid, mask=mask, min_bounds=min_bounds, max_bounds=max_bounds, particles=g["pos"], cov=g["cov3D_precomp"],
                   material_params=mp, bc_params=list(bc), time_params=tp,
                   rotation_matrices=scene_files.generate_rotation_matrices(pp["rotation_degree"], pp["rotation_axis"], device),
                   z_shift_value=pp["z_shift_value"], k_smoothing_neighbors=pp["k_smoothing_neighbors"],
                   nn_distance_threshold=pp["nn_distance_threshold"], material_field_bcs=True, fix_ground=pp["fix_ground"],
                   only_handle_largest_cluster=pp["only_handle_largest_cluster"], opacity=g["opacity"], particle_filling=pp["particle_filling"],
                   sim_area=pp["sim_area"], shs=g["shs"], sh_degree=sh_degree, camera_params=cp,
                   cameras=os.path.join(model_path, "cameras.json"), white_bg=white_bg, save_ply=save_ply,
                   to_original_coord=pp["to_original_coord"])


def check_supported(name: str, preprocessing_params: Dict):
    """Raises NotImplementedError for a config this package cannot simulate: particle filling with `smooth`, which needs
    PyMCubes' constrained smoothing."""
    pf = preprocessing_params.get("particle_filling")
    if pf and pf.get("smooth", False):
        raise NotImplementedError(f"scene {name}: particle filling with smooth needs mcubes.smooth (PyMCubes), which is not available")


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

    @classmethod
    def physics_only(cls, device="cuda:0") -> "SceneBatchDriver":
        """A driver for scenes whose material point cloud is already at hand (gs_simulation.py's --point_cloud_path): no
        networks are built, so only run_physics_simulation is available."""
        self = cls.__new__(cls)
        self.device, self.predictor, self.ranges, self.grid_size = torch.device(device), None, None, None
        return self

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
                               on_frame: Optional[Callable[[int, torch.Tensor, Optional[torch.Tensor]], None]] = None,
                               on_image: Optional[Callable[[int, torch.Tensor], None]] = None, ply_dir: Optional[str] = None) -> Dict:
        """One scene's rollout (gs_simulation.py:395-634): returns the per-frame render-space positions (and covariances when
        the scene has them) unless `on_frame(frame, pos, cov)` consumes them. A scene with `shs` and `camera_params` is also
        rendered each frame (the Gaussians only, from the frame's camera); the (3, H, W) images go to `on_image(frame, image)`
        or to the record's `frames_rgb`. With `sim_area`, only the Gaussians inside it are simulated and exported; the others
        are appended, unchanged, to every rendered frame. With the filling block's `visualize`, the filled particles carry
        their nearest Gaussian's SH, opacity and covariance and are exported and rendered like Gaussians. With `save_ply`,
        each frame's rendered particles (not the Gaussians outside sim_area) with their render SH and opacity are also
        written to `ply_dir/frame_{frame:05d}.ply` (export_gaussians_to_ply's file), the copy and the write overlapping the
        next frame's substeps; existing files there are overwritten, nothing is deleted."""
        if sc.save_ply:
            if sc.shs is None or sc.opacity is None or sc.cov is None:
                raise ValueError(f"scene {sc.name}: save_ply needs the Gaussians' shs, opacity and cov")
            if ply_dir is None:
                raise ValueError(f"scene {sc.name}: save_ply needs a ply_dir")
        dev = self.device
        mp, tp = dict(sc.material_params), sc.time_params
        n_grid, grid_lim = int(mp.get("n_grid", 64)), float(mp.get("grid_lim", 2.0))
        rots = [r.to(dev, torch.float32) for r in sc.rotation_matrices]
        init_pos = sc.particles.to(dev, torch.float32)
        rotated = apply_rotations(init_pos, rots)
        init_cov = None if sc.cov is None else sc.cov.to(dev, torch.float32)
        init_opacity = None if sc.opacity is None else sc.opacity.to(dev, torch.float32)
        init_shs = None if sc.shs is None else sc.shs.to(dev, torch.float32)
        unselected = None
        if sc.sim_area is not None:
            # gs_simulation.py:419-434: the Gaussians strictly inside the box (float32 positions against float32 bounds, as
            # torch compares them) are simulated; the others keep their original frame, opacity and SH for rendering
            b = [float(v) for v in sc.sim_area]
            if len(b) != 6:
                raise ValueError(f"scene {sc.name}: sim_area must be [x0, x1, y0, y1, z0, z1]")
            mask = torch.ones(rotated.shape[0], dtype=torch.bool, device=dev)
            for i in range(3):
                mask &= (rotated[:, i] > b[2 * i]) & (rotated[:, i] < b[2 * i + 1])
            if not bool(mask.any()):
                raise ValueError(f"scene {sc.name}: no Gaussian lies strictly inside sim_area {b}")
            keep = lambda t: None if t is None else t[mask]                                # noqa: E731
            drop = lambda t: None if t is None else t[~mask]                               # noqa: E731
            unselected = {"pos": drop(init_pos), "cov": drop(init_cov), "opacity": drop(init_opacity), "shs": drop(init_shs)}
            rotated, init_cov, init_opacity, init_shs = rotated[mask], keep(init_cov), keep(init_opacity), keep(init_shs)
        transformed, scale_origin, original_mean_pos = transform2origin(rotated)
        pos0 = transformed + torch.tensor([1.0, 1.0, 1.0 + sc.z_shift_value], device=dev)          # shift2center111 :103-105
        cov0 = None
        if init_cov is not None:
            # apply_cov_rotations(init_cov, R) * scale^2  (gs_simulation.py:438): R C R^T per rotation, on the device
            c = init_cov
            m = torch.stack([c[:, 0], c[:, 1], c[:, 2], c[:, 1], c[:, 3], c[:, 4], c[:, 2], c[:, 4], c[:, 5]], dim=1).view(-1, 3, 3)
            for R in rots:
                m = R @ m @ R.T
            cov0 = torch.stack([m[:, 0, 0], m[:, 0, 1], m[:, 0, 2], m[:, 1, 1], m[:, 1, 2], m[:, 2, 2]], dim=1) * (scale_origin ** 2)
        gs_num = int(pos0.shape[0])
        shs_render, opacity_render, n_render = init_shs, init_opacity, gs_num
        if sc.particle_filling is not None:
            pos0, cov0, filled_attrs = self._fill(sc, pos0, cov0, init_opacity, init_shs, n_grid, grid_lim)
            if filled_attrs is not None:                     # visualize: every particle is a Gaussian from here on (:473-477)
                shs_render, opacity_render = filled_attrs
                n_render = int(pos0.shape[0])
        n_filled = int(pos0.shape[0]) - gs_num
        vol = frame_export.get_particle_volume(pos0, n_grid, grid_lim / n_grid, unifrom=mp.get("material") == "sand")
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
        if sc.e_field is not None:                                                                  # gs_simulation.py:527-531
            E = sc.e_field.detach().to(dev, torch.float32).reshape(-1).contiguous()
            if E.numel() != solver.n_particles:
                raise ValueError(f"scene {sc.name}: the E field has {E.numel()} values for {solver.n_particles} particles")
            solver.mpm_model.E = E
            solver.finalize_mu_lam()
        substep_dt = tp["substep_dt"]
        step_per_frame = int(tp["frame_dt"] / substep_dt)                                           # float division like :627
        frames_pos, frames_cov, frames_rgb = [], [], []
        filled = n_render != int(pos0.shape[0])
        render = self._render_setup(sc, rots, scale_origin, original_mean_pos, shs_render, opacity_render, n_render, unselected) \
            if sc.shs is not None and sc.camera_params is not None else None
        with frame_export.PlyFrameWriter(ply_dir, dev) if sc.save_ply else contextlib.nullcontext() as ply:
            for frame in range(int(tp["frame_num"])):
                pos = solver.export_particle_x_to_torch()
                cov = solver.export_particle_cov_to_torch().view(-1, 6) if sc.cov is not None else None
                if filled:                                                                         # the Gaussians only (:591, 594)
                    pos, cov = pos[:n_render], cov[:n_render]
                pr, cr = frame_export.render_frame_transform(pos, cov, sc.z_shift_value, scale_origin, original_mean_pos, rots)
                if render is not None:
                    image = render(frame, pr, cr)
                    if on_image is not None:
                        on_image(frame, image)
                    else:
                        frames_rgb.append(image)
                if ply is not None:                                                                # export_gaussians_to_ply
                    ply.submit(frame, pr if sc.to_original_coord else pos, cr, shs_render, opacity_render)
                if on_frame is not None:
                    on_frame(frame, pr, cr)
                else:
                    frames_pos.append(pr.clone())
                    frames_cov.append(None if cr is None else cr.clone())
                solver.p2g2p_n(step_per_frame, substep_dt)
        record = {"name": sc.name, "n_particles": int(pos0.shape[0]), "n_gaussians": gs_num, "frames_pos": frames_pos, "frames_cov": frames_cov,
                  "material_ids": props[4], "E": props[2], "substeps": step_per_frame * int(tp["frame_num"]), "time": solver.time,
                  "bc_conditions": bc_conditions, "n_filled": n_filled, "n_unselected": 0 if unselected is None else int(unselected["pos"].shape[0])}
        if render is not None:
            record["frames_rgb"] = frames_rgb
        return record

    def _render_setup(self, sc: Scene, rots, scale_origin, original_mean_pos, shs: torch.Tensor, opacity: torch.Tensor, n_render: int,
                      unselected: Optional[Dict[str, torch.Tensor]]):
        """gs_simulation.py:529-540, 573-619: the view centre and orbit basis once, then per frame the camera for that frame
        index and the first n_render simulated particles rasterised with `shs` / `opacity` (the Gaussians' own, or with
        `visualize` those of init_filled_particles), followed by the Gaussians outside sim_area, unchanged (roll 0: the
        reference passes none)."""
        if sc.cov is None or sc.opacity is None:
            raise ValueError(f"scene {sc.name}: rendering needs the Gaussians' cov and opacity")
        if sc.cameras is None:
            raise ValueError(f"scene {sc.name}: rendering needs the model's cameras (the cameras.json list or its path)")
        shs = shs.contiguous()
        opacity = opacity.reshape(-1).contiguous()
        if shs.dim() != 3 or shs.shape[0] != n_render or opacity.shape[0] != n_render:
            raise ValueError(f"scene {sc.name}: shs must be (N, K, 3) and opacity (N,) for the N = {n_render} Gaussians")
        if unselected is not None:
            u_shs, u_opacity = unselected["shs"], unselected["opacity"].reshape(-1)
            if u_shs.dim() != 3 or u_shs.shape[1:] != shs.shape[1:]:
                raise ValueError(f"scene {sc.name}: shs must be (N, K, 3)")
            shs = torch.cat([shs, u_shs]).contiguous()
            opacity = torch.cat([opacity, u_opacity]).contiguous()
        cp = gs_render.decode_camera_params(sc.camera_params)
        cams = gs_render.load_cameras(sc.cameras)
        center, basis = gs_render.get_center_view_worldspace_and_observant_coordinate(
            cp["mpm_space_viewpoint_center"], cp["mpm_space_vertical_upward_axis"], rots, scale_origin, original_mean_pos)
        bg = [1.0, 1.0, 1.0] if sc.white_bg else [0.0, 0.0, 0.0]

        def render(frame: int, pos: torch.Tensor, cov: torch.Tensor) -> torch.Tensor:
            cam = gs_render.get_camera_view(cams, cp["default_camera_index"], center, basis, False, cp["init_azimuthm"], cp["init_elevation"],
                                            cp["init_radius"], None, cp["move_camera"], frame, cp["delta_a"], cp["delta_e"], cp["delta_r"])
            if unselected is not None:                                                            # gs_simulation.py:602-606
                pos, cov = torch.cat([pos, unselected["pos"]]), torch.cat([cov, unselected["cov"]])
            return gs_render.rasterize(pos, cov, opacity, cam, bg, shs=shs, sh_degree=sc.sh_degree)[0]
        return render

    def _fill(self, sc: Scene, pos0: torch.Tensor, cov0: Optional[torch.Tensor], opacity: Optional[torch.Tensor],
              shs: Optional[torch.Tensor], n_grid: int, grid_lim: float):
        """Particle filling of gs_simulation.py:442-462, 473-481: (positions, covariances, render attributes), the Gaussians
        first, then the filled particles. Without `visualize` the filled particles get covariance 0 and the render
        attributes are None; with it, each takes the SH, opacity and covariance of its nearest Gaussian
        (init_filled_particles) and the render attributes are (shs, opacity) of all particles."""
        fp = particle_filling.decode_filling_params(sc.particle_filling, {"n_grid": n_grid})
        if fp["smooth"]:
            raise NotImplementedError(
                f"scene {sc.name}: particle filling with smooth needs mcubes.smooth (PyMCubes), which is not available")
        if opacity is None or cov0 is None:
            raise ValueError(f"scene {sc.name}: particle filling needs the Gaussians' opacity and cov")
        if fp["visualize"] and shs is None:
            raise ValueError(f"scene {sc.name}: particle filling with visualize needs the Gaussians' shs, opacity and cov")
        pos = particle_filling.fill_particles(
            pos=pos0, opacity=opacity, cov=cov0, grid_n=fp["n_grid"], max_samples=fp["max_particles_num"],
            grid_dx=grid_lim / fp["n_grid"], density_thres=fp["density_threshold"], search_thres=fp["search_threshold"],
            max_particles_per_cell=fp["max_partciels_per_cell"], search_exclude_dir=fp["search_exclude_direction"],
            ray_cast_dir=fp["ray_cast_direction"], boundary=fp["boundary"], smooth=False)
        n = pos0.shape[0]
        if fp["visualize"]:
            shs_all, opacity_all, cov = particle_filling.init_filled_particles(pos[:n], shs, cov0, opacity, pos[n:])
            return pos, cov, (shs_all, opacity_all)
        cov = torch.zeros((pos.shape[0], 6), dtype=torch.float32, device=pos.device)
        cov[:n] = cov0
        return pos, cov, None

    # ------------------------------------------------------------------------------ batch
    def run(self, scenes: Sequence[Scene], out_dir: Optional[str] = None) -> List[Dict]:
        """This rank's share of `scenes` end to end; returns one record per processed scene (in scene order). A scene with
        save_ply writes its frames to `<out_dir>/<scene>/ply_files`."""
        rank, world, _ = dist_utils.env_rank_world()
        mine = [scenes[i] for i in dict.fromkeys(dist_utils.shard_scenes(len(scenes), rank, world))]
        clouds = self.generate_neural_segmentation(mine, out_dir)
        return [self.run_physics_simulation(sc, cl, ply_dir=None if out_dir is None else os.path.join(out_dir, sc.name, "ply_files"))
                for sc, cl in zip(mine, clouds)]
