"""Generates tests/golden/transfer_golden.npz by EXECUTING THE REFERENCE'S OWN FUNCTIONS for the steps either side of
the two hot halves (SURVEY.md §8 f-1, f-2).  PIXIE_REFERENCE names a checkout of the reference:

    python tests/golden/make_transfer_golden.py

The reference modules cannot be imported whole (hydra, plyfile, warp, taichi, matplotlib-at-import, device="cuda"
literals), so the function SOURCES are pulled out of the reference files with `ast` and exec'd in a namespace whose
imports are stand-ins that do no arithmetic of their own:

  pixie/voxel/map_pred_to_coords.py     unscale_prediction, get_mat_id, map_pred_to_ply     (PlyData/PlyElement capture the table)
  PG/material_field.py                  DEFAULT_VALUES, MaterialProperties, transform_to_original_coordinates, scene_bounds,
                                        extract_material_properties, perform_knn_smoothing, _apply_material_properties_to_solver
  PG/utils/transformation_utils.py      undotransform2origin, undoshift2center111, apply_inverse_rotation(s), get_mat_from_upper,
                                        get_uppder_from_mat, apply_cov_rotation, apply_inverse_cov_rotations    (torch on the CPU)
  PG/particle_filling/filling.py        assign_particle_to_grid, compute_particle_volume, get_particle_volume   (mini `ti` below)
  PG/mpm_solver_warp/*                  the solver `_apply_material_properties_to_solver` talks to, on tests/golden/_fake_warp.py

scikit-learn, numpy and torch are the real libraries (the reference uses them too).
"""
import ast
import logging
import os
import sys
import tempfile
import types
from collections import Counter
from pathlib import Path

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
REF = os.environ["PIXIE_REFERENCE"]
PG = REF + "/third_party/PhysGaussian"

import _fake_warp as wp  # noqa: E402

wp.install()
for missing in ("h5py", "plyfile"):
    if missing not in sys.modules:
        m = types.ModuleType(missing)
        m.PlyData = m.PlyElement = m.File = None
        sys.modules[missing] = m
sys.path.insert(0, PG + "/mpm_solver_warp")
import mpm_solver_warp as REFMPM  # noqa: E402  (the reference solver, on the warp stand-in)


def extract(path, names, ns):
    """exec the top-level definitions `names` of the reference file `path` inside namespace `ns`."""
    src = open(path).read()
    tree = ast.parse(src)
    want = set(names)
    for node in tree.body:
        nm = None
        if isinstance(node, (ast.FunctionDef, ast.ClassDef)):
            nm = node.name
        elif isinstance(node, ast.Assign) and isinstance(node.targets[0], ast.Name):
            nm = node.targets[0].id
        if nm in want:
            code = compile(ast.Module(body=[node], type_ignores=[]), path, "exec")
            exec(code, ns)
            if not (isinstance(node, ast.FunctionDef) and nm in ns.get("_seen", set())):
                ns.setdefault("_seen", set()).add(nm)
    missing = want - ns.get("_seen", set())
    assert not missing, (path, missing)
    return ns


class _TorchCPU:
    """`torch`, except that factory calls ignore device="cuda" (transformation_utils.py hard-codes it)."""

    def __getattr__(self, k):
        f = getattr(torch, k)
        if k in ("tensor", "zeros"):
            def g(*a, **kw):
                kw.pop("device", None)
                return f(*a, **kw)
            return g
        return f


# ----------------------------------------------------------------------------------------- mini taichi (f32 / i32)
class _Ref:
    """`field[i, j, k]` inside a kernel: readable as a number, and a target for ti.atomic_add."""

    def __init__(self, fld, idx):
        self.f, self.i = fld, idx

    def value(self):
        return self.f.a[self.i]

    def __rtruediv__(self, other):
        return np.float32(other) / np.float32(self.value())

    def __getitem__(self, c):          # vector field element component
        return self.f.a[self.i][c]


class _Field:
    def __init__(self, dtype, shape, n=None):
        shp = (shape,) if np.isscalar(shape) else tuple(shape)
        self.a = np.zeros(shp + ((n,) if n else ()), np.float32 if dtype is float else np.int32)
        self.shape = shp

    def from_torch(self, t):
        self.a[...] = t.detach().cpu().numpy()

    def to_torch(self):
        return torch.from_numpy(self.a.copy())

    def __getitem__(self, idx):
        return _Ref(self, idx)

    def __setitem__(self, idx, v):
        self.a[idx] = v


def _make_ti():
    ti = types.SimpleNamespace()
    ti.kernel = lambda fn: (lambda *a: fn(*[np.float32(x) if isinstance(x, float) else x for x in a]))
    ti.template = lambda: None
    ti.floor = lambda x, dtype=int: int(np.floor(np.float32(x)))
    ti.field = lambda dtype, shape: _Field(dtype, shape)
    ti.Vector = types.SimpleNamespace(field=lambda n, dtype, shape: _Field(dtype, shape, n))

    def atomic_add(ref, v):
        ref.f.a[ref.i] += v
    ti.atomic_add = atomic_add
    return ti


# ------------------------------------------------------------------------------------------------------- stand-ins
class _Capture:
    table = None

    class PlyElement:
        @staticmethod
        def describe(data, name):
            _Capture.table = data.copy()
            return data

    class PlyData:
        def __init__(self, elements, text=False):
            pass

        def write(self, path):
            pass


RANGES = dict(density_min=1.703, density_max=3.871, E_min=3.018, E_max=10.882, nu_min=0.2103, nu_max=0.4493)


def field_inputs(seed, n_occupied=700, D=64, K=8):
    """Sparse 64^3 scene (map_pred_to_ply asserts 64^3): values only at the occupied voxels, zeros elsewhere."""
    rng = np.random.default_rng(seed)
    flat = np.sort(rng.choice(D ** 3, size=n_occupied, replace=False))
    # a coherent blob so that kNN neighbourhoods are meaningful
    idx = np.stack(np.unravel_index(flat, (D, D, D)), axis=1)
    keep = np.linalg.norm(idx - D / 2, axis=1) < D / 2.2
    idx = idx[keep]
    blob = np.argwhere(np.linalg.norm(np.indices((D, D, D)).transpose(1, 2, 3, 0) - D / 2, axis=-1) < 5.5)
    idx = np.unique(np.concatenate([idx, blob]), axis=0)
    vals = np.zeros((len(idx), 3 + K), np.float32)
    vals[:, :3] = rng.uniform(-1.3, 1.3, size=(len(idx), 3))
    vals[:, 3:] = rng.standard_normal((len(idx), K)).astype(np.float32)
    ties = rng.choice(len(idx), size=40, replace=False)                      # exact ties: argmax must take the FIRST maximum
    for t in ties:
        a, b = sorted(rng.choice(K, size=2, replace=False))
        vals[t, 3 + a] = vals[t, 3 + b] = 9.0
    onehot = rng.choice(len(idx), size=len(idx) // 2, replace=False)         # one-hot rows like save_predictions writes
    vals[onehot, 3:] = np.eye(K, dtype=np.float32)[rng.integers(0, K, size=len(onehot))]
    return idx.astype(np.int32), vals


def dense(idx, vals, D=64):
    pred = np.zeros((vals.shape[1], D, D, D), np.float32)
    mask = np.zeros((D, D, D), np.float32)
    pred[:, idx[:, 0], idx[:, 1], idx[:, 2]] = vals.T
    mask[idx[:, 0], idx[:, 1], idx[:, 2]] = 1.0
    return pred, mask


def main():
    blob = {}
    # ---------------------------------------------------------------- f-1a: unscale_prediction + map_pred_to_ply
    ns = {"np": np, "os": os, "logging": logging, "Path": Path, "PlyData": _Capture.PlyData, "PlyElement": _Capture.PlyElement,
          "DictConfig": object}
    extract(REF + "/pixie/voxel/map_pred_to_coords.py", ["unscale_prediction", "get_mat_id", "map_pred_to_ply"], ns)
    cfg = types.SimpleNamespace(training=types.SimpleNamespace(**RANGES))
    idx, vals = field_inputs(seed=5)
    pred, mask = dense(idx, vals)
    lo, hi = np.array([-0.52, -0.41, -0.33]), np.array([0.49, 0.6, 0.71])
    with tempfile.TemporaryDirectory() as td:
        np.save(td + "/pred.npy", pred)
        np.save(td + "/mask.npy", mask)
        np.savez(td + "/grid.npz", min_bounds=lo, max_bounds=hi, grid_shape=np.array([64, 64, 64]))
        ns["map_pred_to_ply"](td + "/pred.npy", td + "/mask.npy", td + "/grid.npz", td + "/out.ply", "obj", cfg=cfg)
    tab = _Capture.table
    un = ns["unscale_prediction"](pred, cfg)
    blob.update({"field/idx": idx, "field/vals": vals, "field/min_bounds": lo, "field/max_bounds": hi,
                 "field/unscaled_at_idx": un[:, idx[:, 0], idx[:, 1], idx[:, 2]].T.copy()})
    for k in ("x", "y", "z", "part_label", "density", "E", "nu", "material_id", "conf"):
        blob[f"field/table/{k}"] = np.asarray(tab[k]).copy()
    print("map_pred_to_ply:", len(tab), "vertices; ids", np.unique(tab["material_id"], return_counts=True))

    # ---------------------------------------------------------------- f-1a': a label-map prediction, (3 + 1, 64, 64, 64):
    # get_mat_id returns the class channel itself and the 'i4' PLY fields truncate it (own RNG: the arrays above are unchanged)
    irng = np.random.default_rng(17)
    iidx, ivals = field_inputs(seed=6)
    ivals = np.concatenate([ivals[:, :3], irng.integers(0, 8, size=(len(iidx), 1)).astype(np.float32)], axis=1)
    odd = irng.choice(len(iidx), size=60, replace=False)
    ivals[odd, 3] = irng.choice(np.array([2.75, -0.5, 7.999, 0.25, 5.5], np.float32), size=60)
    ipred, imask = dense(iidx, ivals)
    with tempfile.TemporaryDirectory() as td:
        np.save(td + "/pred.npy", ipred)
        np.save(td + "/mask.npy", imask)
        np.savez(td + "/grid.npz", min_bounds=lo, max_bounds=hi, grid_shape=np.array([64, 64, 64]))
        ns["map_pred_to_ply"](td + "/pred.npy", td + "/mask.npy", td + "/grid.npz", td + "/out.ply", "obj", cfg=cfg)
    itab = _Capture.table
    blob.update({"field_index/idx": iidx, "field_index/vals": ivals})
    for k in ("x", "y", "z", "part_label", "density", "E", "nu", "material_id", "conf"):
        blob[f"field_index/table/{k}"] = np.asarray(itab[k]).copy()
    print("map_pred_to_ply (class indices):", len(itab), "vertices; ids", np.unique(itab["material_id"], return_counts=True))

    # ---------------------------------------------------------------- f-1b: perform_knn_smoothing
    tns = {"torch": _TorchCPU(), "np": np}
    extract(PG + "/utils/transformation_utils.py",
            ["undotransform2origin", "undoshift2center111", "apply_inverse_rotation", "apply_inverse_rotations", "get_mat_from_upper",
             "get_uppder_from_mat", "apply_cov_rotation", "apply_inverse_cov_rotations", "apply_rotation", "apply_rotations",
             "apply_cov_rotations", "shift2center111"], tns)
    from sklearn.neighbors import NearestNeighbors
    mns = {"np": np, "torch": torch, "Counter": Counter, "NearestNeighbors": NearestNeighbors, "tqdm": lambda it, **kw: it,
           "get_material_name": REFMPM.get_material_name, "save_points_as_ply": lambda *a, **kw: None}
    for k in ("undotransform2origin", "undoshift2center111", "apply_inverse_rotations"):
        mns[k] = tns[k]
    extract(PG + "/material_field.py",
            ["DEFAULT_VALUES", "MaterialProperties", "transform_to_original_coordinates", "scene_bounds", "extract_material_properties",
             "perform_knn_smoothing", "_apply_material_properties_to_solver"], mns)
    assert mns["DEFAULT_VALUES"]["E"] == 5000.0
    blob["knn/DEFAULT_E"] = np.float64(mns["DEFAULT_VALUES"]["E"])

    pos = np.stack([tab["x"], tab["y"], tab["z"]], axis=1).astype(np.float32)
    params = {"pos": pos, "part_labels": np.asarray(tab["part_label"]), "density": np.asarray(tab["density"]), "E": np.asarray(tab["E"]),
              "nu": np.asarray(tab["nu"]), "material_id": np.asarray(tab["material_id"]), "conf": np.asarray(tab["conf"])}
    rng = np.random.default_rng(9)
    n_q = 400
    scale = torch.tensor(1.7)
    mean = torch.tensor([0.03, -0.02, 0.05])
    ang = [0.3, -0.5]
    rots = [torch.tensor([[1, 0, 0], [0, np.cos(ang[0]), -np.sin(ang[0])], [0, np.sin(ang[0]), np.cos(ang[0])]], dtype=torch.float32),
            torch.tensor([[np.cos(ang[1]), 0, np.sin(ang[1])], [0, 1, 0], [-np.sin(ang[1]), 0, np.cos(ang[1])]], dtype=torch.float32)]
    # queries = field points + noise, pushed into the solver's frame (rotate, scale to unit box, shift to (1,1,1))
    base = pos[rng.integers(0, len(pos), size=n_q)] + rng.normal(0, 0.006, size=(n_q, 3)).astype(np.float32)
    base[:25] += 0.5                                                        # 25 of 400 too far (< 10 %): defaults path
    q_sim = tns["shift2center111"](tns["apply_rotations"]((torch.from_numpy(base) - mean) * scale, rots))

    class _Solver:
        n_particles = n_q

        def export_particle_x_to_torch(self):
            return q_sim
    blob.update({"knn/q_sim": q_sim.numpy().copy(), "knn/scale": scale.numpy(), "knn/mean": mean.numpy(),
                 "knn/rots": torch.stack(rots).numpy()})
    q_field = mns["transform_to_original_coordinates"](tns["undoshift2center111"](q_sim), scale, mean, rots).numpy()
    blob["knn/q_field"] = q_field.copy()
    for weighted in (False, True):
        out = mns["perform_knn_smoothing"](_Solver(), dict(params), "cpu", scale, mean, rots, 10, 0.1, weighted, False)
        for name, arr in zip(("part_labels", "density", "E", "nu", "material_id", "conf"), out):
            blob[f"knn/{'weighted' if weighted else 'plain'}/{name}"] = np.asarray(arr).copy()
        print("perform_knn_smoothing weighted =", weighted, "ids", np.unique(out[4], return_counts=True))
    # empty material field: get_defaults falls back to DEFAULT_VALUES (E = 5000.0)
    mp = mns["MaterialProperties"](*(np.zeros(0, np.float32) for _ in range(6)))
    d = mp.get_defaults(3)
    for name in ("density", "E", "nu", "material_id", "part_labels", "conf"):
        blob[f"knn/empty_defaults/{name}"] = np.asarray(d[name])

    # ---------------------------------------------------------------- f-1c: _apply_material_properties_to_solver on the reference solver
    n_p = 48
    x = rng.uniform(0.8, 1.2, size=(n_p, 3)).astype(np.float32)
    x[5] = x[4] + np.float32(4e-4)                                           # inside each other's +-1e-3 box: "last box wins"
    x[20] = x[7] - np.float32(6e-4)
    vol = rng.uniform(1e-4, 2e-4, size=n_p).astype(np.float32)
    s = REFMPM.MPM_Simulator_WARP(n_p, n_grid=16, grid_lim=2.0, device="cpu")
    s.load_initial_data_from_torch(torch.from_numpy(x), torch.from_numpy(vol), None, n_grid=16, grid_lim=2.0, device="cpu")
    s.set_parameters_dict({"material": "jelly", "E": 1e5, "nu": 0.3, "density": 1000.0}, device="cpu")
    dens = rng.uniform(300, 2500, size=n_p).astype(np.float32)
    Ev = (10 ** rng.uniform(4, 6.5, size=n_p)).astype(np.float32)
    nuv = rng.uniform(0.21, 0.45, size=n_p).astype(np.float32)
    ids = rng.integers(0, 7, size=n_p).astype(np.int32)
    mns["_apply_material_properties_to_solver"](s, s.mpm_state.particle_x.numpy(), dens, Ev, nuv, ids, "cpu")
    blob.update({"upload/x": x, "upload/vol": vol, "upload/in_density": dens, "upload/in_E": Ev, "upload/in_nu": nuv, "upload/in_ids": ids,
                 "upload/E": s.mpm_model.E.numpy().copy(), "upload/nu": s.mpm_model.nu.numpy().copy(),
                 "upload/density": s.mpm_state.particle_density.numpy().copy(), "upload/material": s.mpm_state.particle_material.numpy().copy(),
                 "upload/mass": s.mpm_state.particle_mass.numpy().copy(), "upload/mu": s.mpm_model.mu.numpy().copy(),
                 "upload/lam": s.mpm_model.lam.numpy().copy()})
    print("upload: overlapping boxes changed", int((s.mpm_model.E.numpy() != Ev).sum()), "particles")

    # ---------------------------------------------------------------- f-2a: get_particle_volume (Taichi kernels)
    fns = {"ti": _make_ti(), "torch": torch}
    extract(PG + "/particle_filling/filling.py", ["assign_particle_to_grid", "compute_particle_volume", "get_particle_volume"], fns)
    pv = rng.uniform(0.2, 1.8, size=(600, 3)).astype(np.float32)
    pv[:200] = rng.uniform(0.9, 1.1, size=(200, 3)).astype(np.float32)      # dense cluster: many particles per cell
    grid_n, grid_dx = 32, 2.0 / 32
    blob.update({"volume/pos": pv, "volume/grid_n": np.int32(grid_n), "volume/grid_dx": np.float64(grid_dx),
                 "volume/vol": fns["get_particle_volume"](torch.from_numpy(pv), grid_n, grid_dx).numpy().copy(),
                 "volume/vol_uniform": fns["get_particle_volume"](torch.from_numpy(pv), grid_n, grid_dx, unifrom=True).numpy().copy()})

    # ---------------------------------------------------------------- f-2b: per-frame export transform (gs_simulation.py:591-600)
    n_f = 300
    p_sim = torch.from_numpy(rng.uniform(0.6, 1.4, size=(n_f, 3)).astype(np.float32))
    A = rng.standard_normal((n_f, 3, 3)).astype(np.float32) * 0.05
    covm = A @ A.transpose(0, 2, 1)
    cov6 = torch.from_numpy(np.stack([covm[:, 0, 0], covm[:, 0, 1], covm[:, 0, 2], covm[:, 1, 1], covm[:, 1, 2], covm[:, 2, 2]], axis=1).copy())
    z_shift = 0.12
    pos_render = mns["transform_to_original_coordinates"](tns["undoshift2center111"](p_sim, z_shift), scale, mean, rots)
    cov_render = tns["apply_inverse_cov_rotations"](cov6 / (scale ** 2), rots)
    blob.update({"frame/pos": p_sim.numpy().copy(), "frame/cov": cov6.numpy().copy(), "frame/z_shift": np.float64(z_shift),
                 "frame/pos_render": pos_render.numpy().copy(), "frame/cov_render": cov_render.numpy().copy()})

    np.savez_compressed(os.path.join(HERE, "transfer_golden.npz"), **blob)
    print("wrote", os.path.join(HERE, "transfer_golden.npz"), len(blob), "arrays,",
          os.path.getsize(os.path.join(HERE, "transfer_golden.npz")) // 1024, "KiB")


if __name__ == "__main__":
    main()
