"""Generates tests/golden/gaussian_ply_golden.npz by EXECUTING THE REFERENCE'S OWN per-frame PLY export:
cov3D_to_log_scales_and_quats and export_gaussians_to_ply (PhysGaussian's gs_simulation.py:253-322), the
transformation_utils chain with material_field.transform_to_original_coordinates, and GaussianModel's
construct_list_of_attributes / save_ply (gaussian-splatting/scene/gaussian_model.py:177-208). PIXIE_REFERENCE names a
checkout of the reference:

    PIXIE_REFERENCE=<checkout> python tests/golden/make_gaussian_ply_golden.py

The function sources are pulled out of the reference files with `ast` and exec'd in a namespace whose `torch` ignores
device="cuda" (everything runs on the CPU in float32, as the reference's float32 tensors do). plyfile is replaced by a
stand-in that keeps the structured array PlyData.write would serialise, and the solver by a stub whose
export_particle_{x,cov}_to_torch return CPU tensors. Cases:
  eig/*              cov3D_to_log_scales_and_quats on random SPD covariances and the degenerate ones: zero, isotropic, two
                     equal eigenvalues, diagonal, rotated diagonal, 1e6-anisotropic, and a -1e-9 eigenvalue (the clamp)
  k{16,4}_{orig,raw} export_gaussians_to_ply with K SH coefficients and to_original_coord True / False: a solver of
                     gs_num + 7 particles (only gs_num are written), two rotations and a z_shift; covariances are the
                     scaled, rotated images of random SPD and degenerate world covariances
each export case with its inputs, the reference's cov_world (apply_inverse_cov_rotations(cov / scale^2, Rs)), the
records (N, 14 + 3K) float32 in attribute order and the attribute names.
"""
import ast
import errno
import os
import tempfile
import types

import numpy as np
import torch
from scipy.spatial.transform import Rotation

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ["PIXIE_REFERENCE"]
PG = os.path.join(REF, "third_party", "PhysGaussian")
GS = os.path.join(PG, "gaussian-splatting")


def _nodes(path):
    return ast.parse(open(path).read()).body


def extract(path, names, ns):
    for node in _nodes(path):
        nm = node.name if isinstance(node, (ast.FunctionDef, ast.ClassDef)) else None
        if nm in names:
            exec(compile(ast.Module(body=[node], type_ignores=[]), path, "exec"), ns)


def extract_methods(path, cls, names, ns):
    """The methods `names` of class `cls`, as plain functions."""
    out = {}
    for node in _nodes(path):
        if isinstance(node, ast.ClassDef) and node.name == cls:
            for m in node.body:
                if isinstance(m, ast.FunctionDef) and m.name in names:
                    exec(compile(ast.Module(body=[m], type_ignores=[]), path, "exec"), ns)
                    out[m.name] = ns[m.name]
    return out


class _CpuTorch(types.ModuleType):
    """torch with device="cuda" dropped from tensor construction."""

    def __getattr__(self, name):
        return getattr(torch, name)

    @staticmethod
    def tensor(*a, device=None, **k):
        return torch.tensor(*a, **k)

    @staticmethod
    def zeros(*a, device=None, **k):
        return torch.zeros(*a, **k)


WRITTEN = {}


class PlyElement:
    @staticmethod
    def describe(elements, name):
        return (name, elements)


class PlyData:
    def __init__(self, elements):
        self.elements = elements

    def write(self, path):
        (name, arr), = self.elements
        WRITTEN[path] = (name, arr.copy())


class StubSolver:
    def __init__(self, x, cov):
        self.x, self.cov = x, cov

    def export_particle_x_to_torch(self):
        return self.x.clone()

    def export_particle_cov_to_torch(self):
        return self.cov.clone().reshape(-1)


def namespace():
    ns = {"np": np, "torch": _CpuTorch("torch"), "os": os, "scipy_R": Rotation, "PlyData": PlyData, "PlyElement": PlyElement,
          "makedirs": os.makedirs, "path": os.path, "EEXIST": errno.EEXIST}
    extract(os.path.join(PG, "utils", "transformation_utils.py"),
            {"undotransform2origin", "get_mat_from_upper", "get_uppder_from_mat", "apply_cov_rotation", "apply_cov_rotations",
             "undoshift2center111", "apply_inverse_rotation", "apply_inverse_rotations", "apply_inverse_cov_rotations"}, ns)
    extract(os.path.join(PG, "material_field.py"), {"transform_to_original_coordinates"}, ns)
    extract(os.path.join(GS, "utils", "system_utils.py"), {"mkdir_p"}, ns)
    methods = extract_methods(os.path.join(GS, "scene", "gaussian_model.py"), "GaussianModel", {"construct_list_of_attributes", "save_ply"}, ns)

    def __init__(self, sh_degree):
        self.max_sh_degree = sh_degree
    ns["GaussianModel"] = type("GaussianModel", (), dict(methods, __init__=__init__))
    extract(os.path.join(PG, "gs_simulation.py"), {"cov3D_to_log_scales_and_quats", "export_gaussians_to_ply"}, ns)
    return ns


def rot(rng):
    q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    return q * np.sign(np.linalg.det(q))


def upper(m):
    return np.stack([m[..., 0, 0], m[..., 0, 1], m[..., 0, 2], m[..., 1, 1], m[..., 1, 2], m[..., 2, 2]], axis=-1)


def covariances(rng, n_random):
    """Random SPD covariances (log-uniform eigenvalues over four decades) followed by the degenerate ones, (M, 6) float64."""
    ev = 10.0 ** rng.uniform(-6, -2, size=(n_random, 3))
    Q = np.stack([rot(rng) for _ in range(n_random)])
    spd = upper(Q @ (ev[:, :, None] * np.eye(3)) @ Q.transpose(0, 2, 1))
    Rr = rot(rng)

    def rotated(d):
        return upper(Rr @ np.diag(d) @ Rr.T)
    special = [
        np.zeros(6),                                                    # zero: every eigenvalue clamped
        upper(np.eye(3) * 2.5e-4),                                      # isotropic
        rotated([4e-4, 4e-4, 1e-5]),                                    # two equal eigenvalues (largest pair)
        rotated([4e-4, 1e-5, 1e-5]),                                    # two equal eigenvalues (smallest pair)
        upper(np.diag([1e-5, 3e-3, 4e-4])),                             # diagonal, not sorted
        rotated([3e-3, 4e-4, 1e-5]),                                    # rotated diagonal
        rotated([1e-2, 1e-5, 1e-8]),                                    # 1e6-anisotropic
        upper(np.diag([1e-3, 5e-4, -1e-9])),                            # a -1e-9 eigenvalue, exact
        rotated([1e-3, 5e-4, -1e-9]),                                   # and rotated
    ]
    return np.concatenate([spd, np.stack(special)])


def main():
    ns = namespace()
    rng = np.random.default_rng(20261017)
    out = {}

    cov = torch.from_numpy(covariances(rng, 200).astype(np.float32))
    ls, q = ns["cov3D_to_log_scales_and_quats"](cov.clone())
    out["eig/cov"], out["eig/log_scales"], out["eig/quats"] = cov.numpy(), ls.numpy(), q.numpy()

    with tempfile.TemporaryDirectory() as d:
        for K in (16, 4):
            Rs = [torch.from_numpy(rot(rng).astype(np.float32)) for _ in range(2)]
            scale = torch.tensor(float(rng.uniform(0.3, 0.9)), dtype=torch.float32)
            mean = torch.from_numpy(rng.normal(scale=0.2, size=3).astype(np.float32))
            z_shift = float(rng.uniform(0.05, 0.3))
            gs_num, extra = 150, 7
            world = torch.from_numpy(covariances(rng, gs_num + extra - 10).astype(np.float32))
            sim_cov = ns["apply_cov_rotations"](world, Rs) * scale ** 2
            x = torch.from_numpy(rng.uniform(0.6, 1.4, size=(gs_num + extra, 3)).astype(np.float32))
            shs = torch.from_numpy((rng.normal(scale=0.5, size=(gs_num + extra, K, 3))).astype(np.float32))
            opacity = torch.from_numpy(rng.uniform(0.0, 1.0, size=(gs_num + extra, 1)).astype(np.float32))
            for to_orig in (True, False):
                name = f"k{K}_{'orig' if to_orig else 'raw'}"
                solver = StubSolver(x, sim_cov)
                WRITTEN.clear()
                ns["export_gaussians_to_ply"](d, solver, 3, gs_num, scale, Rs, opacity, shs, 7, {"z_shift_value": z_shift}, mean,
                                              to_original_coord=to_orig)
                (path, (el_name, arr)), = WRITTEN.items()
                assert os.path.basename(path) == "frame_00007.ply" and el_name == "vertex"
                names = list(arr.dtype.names)
                cov_world = ns["apply_inverse_cov_rotations"](sim_cov[:gs_num] / scale ** 2, Rs)
                out.update({f"{name}/x": x.numpy(), f"{name}/sim_cov": sim_cov.numpy(), f"{name}/shs": shs.numpy(),
                            f"{name}/opacity": opacity.numpy(), f"{name}/rots": np.stack([r.numpy() for r in Rs]),
                            f"{name}/scale": scale.numpy(), f"{name}/mean": mean.numpy(), f"{name}/z_shift": np.float64(z_shift),
                            f"{name}/gs_num": np.int64(gs_num), f"{name}/cov_world": cov_world.numpy(),
                            f"{name}/records": np.stack([arr[nm] for nm in names], axis=1).astype(np.float32),
                            f"{name}/names": np.array(names)})
    np.savez_compressed(os.path.join(HERE, "gaussian_ply_golden.npz"), **out)
    print(f"wrote {len(out)} arrays")


if __name__ == "__main__":
    main()
