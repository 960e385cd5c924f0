"""Generates tests/golden/render_golden.npz by EXECUTING THE REFERENCE'S OWN camera and SH functions (PhysGaussian's
utils/camera_view_utils.py, utils/transformation_utils.py, utils/render_utils.py:convert_SH and gaussian-splatting's
utils/graphics_utils.py, utils/sh_utils.py). PIXIE_REFERENCE names a checkout of the reference:

    PIXIE_REFERENCE=<checkout> python tests/golden/make_render_golden.py

The function sources are pulled out of the reference files with `ast` and exec'd in a namespace whose `torch` ignores
device="cuda" (everything runs on the CPU, in float64 where the inputs are float64) and whose `GSCamera` records what
get_camera_view hands it. Cases:
  cam_index_k      get_camera_view at default_camera_index k of a synthetic three-camera cameras.json
  orbit_f          the orbit camera (index -1) with move_camera and every delta set, frames 0..5
  orbit_roll_f     the same with init_roll / delta_roll (camera_view_utils supports them; gs_simulation passes none)
  center_*         get_center_view_worldspace_and_observant_coordinate for two rotation stacks
  sh_d             convert_SH at active degree d = 0..3 (max degree 3), float64
each with R, T, FoVx, FoVy, width, height and the float32 getWorld2View2 / getProjectionMatrix of that camera.
"""
import ast
import json
import math
import os
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ["PIXIE_REFERENCE"]
PG = os.path.join(REF, "third_party", "PhysGaussian")
GS = os.path.join(PG, "gaussian-splatting")


def extract(path, names, ns):
    tree = ast.parse(open(path).read())
    for node in tree.body:
        nm = None
        if isinstance(node, (ast.FunctionDef, ast.ClassDef)):
            nm = node.name
        elif isinstance(node, ast.Assign) and isinstance(node.targets[0], ast.Name):
            nm = node.targets[0].id
        if nm in names:
            exec(compile(ast.Module(body=[node], type_ignores=[]), path, "exec"), ns)


class _CpuTorch(types.ModuleType):
    """torch with device="cuda" dropped from tensor construction."""

    def __getattr__(self, name):
        return getattr(torch, name)

    @staticmethod
    def tensor(*a, device=None, **k):
        return torch.tensor(*a, **k)


class GSCamera:
    def __init__(self, colmap_id, R, T, FoVx, FoVy, image, gt_alpha_mask, image_name, uid):
        self.R, self.T, self.FoVx, self.FoVy = R, T, FoVx, FoVy
        self.height, self.width = image.shape[1], image.shape[2]


def namespace():
    ns = {"np": np, "torch": _CpuTorch("torch"), "json": json, "os": os, "math": math, "GSCamera": GSCamera, "GaussianModel": object}
    extract(os.path.join(GS, "utils", "graphics_utils.py"), {"getWorld2View2", "getProjectionMatrix", "focal2fov"}, ns)
    extract(os.path.join(GS, "utils", "sh_utils.py"), {"C0", "C1", "C2", "C3", "C4", "eval_sh"}, ns)
    extract(os.path.join(PG, "utils", "camera_view_utils.py"),
            {"_rodrigues_rotation", "generate_camera_rotation_matrix", "generate_local_coord", "get_point_on_sphere",
             "get_camera_position_and_rotation", "get_camera_view"}, ns)
    extract(os.path.join(PG, "utils", "transformation_utils.py"),
            {"undotransform2origin", "undoshift2center111", "apply_inverse_rotation", "apply_inverse_rotations",
             "undo_all_transforms", "get_center_view_worldspace_and_observant_coordinate"}, ns)
    extract(os.path.join(PG, "utils", "render_utils.py"), {"convert_SH"}, ns)
    return ns


def rot(rng):
    q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    return q * np.sign(np.linalg.det(q))


def main():
    ns = namespace()
    rng = np.random.default_rng(20261016)
    cams = []
    for k, (w, h) in enumerate([(800, 800), (801, 577), (1920, 1080)]):
        cams.append({"id": k, "img_name": f"{k:05d}", "width": w, "height": h, "position": rng.normal(size=3).tolist(),
                     "rotation": rot(rng).tolist(), "fx": float(rng.uniform(0.6, 1.4) * w), "fy": float(rng.uniform(0.6, 1.4) * h)})
    out = {"cameras_json": np.frombuffer(json.dumps(cams).encode(), dtype=np.uint8)}

    def put(prefix, cam):
        out[prefix + "_R"], out[prefix + "_T"] = np.asarray(cam.R, np.float64), np.asarray(cam.T, np.float64)
        out[prefix + "_fov"] = np.array([cam.FoVx, cam.FoVy])
        out[prefix + "_wh"] = np.array([cam.width, cam.height])
        out[prefix + "_world_view"] = ns["getWorld2View2"](cam.R, cam.T)
        out[prefix + "_proj"] = ns["getProjectionMatrix"](znear=0.01, zfar=100.0, fovX=cam.FoVx, fovY=cam.FoVy).numpy()

    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "cameras.json"), "w") as f:
            json.dump(cams, f)
        for k in range(len(cams)):
            put(f"cam_index_{k}", ns["get_camera_view"](d, default_camera_index=k))

        # view centre / observant basis, as gs_simulation.py:529-540 computes them (float64 inputs here)
        for name, n_rot in (("center_a", 1), ("center_b", 3)):
            Rs = [torch.from_numpy(rot(rng)) for _ in range(n_rot)]
            scale = torch.tensor(float(rng.uniform(0.2, 2.0)), dtype=torch.float64)
            mean = torch.from_numpy(rng.normal(size=3))
            center = torch.from_numpy(rng.uniform(0.5, 1.5, size=3)).view(1, 3)
            up = torch.from_numpy(rng.normal(size=3)).view(1, 3)
            vc, oc = ns["get_center_view_worldspace_and_observant_coordinate"](center, up, Rs, scale, mean)
            out[name + "_in_rots"] = np.stack([R.numpy() for R in Rs])
            out[name + "_in_scale"] = scale.numpy()
            out[name + "_in_mean"] = mean.numpy()
            out[name + "_in_center"] = center.numpy().reshape(3)
            out[name + "_in_up"] = up.numpy().reshape(3)
            out[name + "_view_center"], out[name + "_observant"] = np.asarray(vc), np.asarray(oc)

        vc, oc = out["center_b_view_center"], out["center_b_observant"]
        orbit = dict(init_azimuthm=-30.0, init_elevation=15.0, init_radius=2.5, move_camera=True, delta_a=1.7, delta_e=-0.4,
                     delta_r=0.03)
        out["orbit_params"] = np.array([orbit[k] for k in ("init_azimuthm", "init_elevation", "init_radius", "delta_a", "delta_e", "delta_r")])
        for f in range(6):
            put(f"orbit_{f}", ns["get_camera_view"](d, default_camera_index=-1, center_view_world_space=vc, observant_coordinates=oc,
                                                   current_frame=f, **orbit))
            put(f"orbit_roll_{f}", ns["get_camera_view"](d, default_camera_index=-1, center_view_world_space=vc,
                                                        observant_coordinates=oc, current_frame=f, init_roll=12.0, delta_roll=2.5, **orbit))

    # convert_SH in float64: shs (N, 16, 3) as GaussianModel.get_features, max degree 3
    n = 64
    shs = torch.from_numpy(rng.normal(scale=0.6, size=(n, 16, 3)))
    pos = torch.from_numpy(rng.normal(size=(n, 3)))
    campos = torch.from_numpy(rng.normal(size=3) * 3.0)
    out["sh_in_shs"], out["sh_in_pos"], out["sh_in_campos"] = shs.numpy(), pos.numpy(), campos.numpy()
    for deg in range(4):
        pc = types.SimpleNamespace(max_sh_degree=3, active_sh_degree=deg)
        cam = types.SimpleNamespace(camera_center=campos)
        out[f"sh_{deg}"] = ns["convert_SH"](shs, cam, pc, pos).numpy()
    np.savez_compressed(os.path.join(HERE, "render_golden.npz"), **out)
    print(f"wrote {len(out)} arrays")


if __name__ == "__main__":
    main()
