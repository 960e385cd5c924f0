"""Generates tests/golden/segmentation_golden.npz by EXECUTING THE REFERENCE'S OWN VLM part segmentation
(pixie/voxel/segmentation.py: get_initial_voxel_grid_from_saved, load_occupancy_grid, run_clip, clip_part_segmentation,
local_post_process_segmentation, save_segmented_point_cloud and the `__main__` block) on the CPU. PIXIE_REFERENCE names a
checkout:

    PIXIE_REFERENCE=<checkout> python tests/golden/make_segmentation_golden.py

The functions are pulled out of the reference file with `ast`, their `device="cuda"` defaults set to "cpu". Only outputs
are stored: the inputs are rebuilt from seeds by `cases()` / `write_inputs()`, which the tests import. Assumed stand-ins for
the modules the reference imports that are not installed here:
  - f3rm's `clip`: `load()` returns a model whose `encode_text` returns the case's seeded (P, C) float32 table, row i for
    query i (`tokenize` returns the query positions); `CLIPArgs.model_name` is a placeholder.
  - `trimesh.load`: a point cloud with `vertices` float64 (N, 3) and `colors` RGBA uint8 with alpha 255, read from the
    binary little-endian PLY (double x y z, uchar red green blue) that Open3D writes for the occupancy grid.
  - `matplotlib.pyplot.colormaps["tab10"]`: matplotlib's ten colours #1f77b4 #ff7f0e #2ca02c #d62728 #9467bd #8c564b
    #e377c2 #7f7f7f #bcbd22 #17becf as hex / 255 in float64 with alpha 1.0, N = 10, called with an int.
  - `plyfile`: the stand-in of make_network_files_golden.py, which writes plyfile's header and the packed rows.
  - `pixie.utils`: the reference's own `str2bool` and `load_json`; `set_logger` does nothing.
  - `tqdm`: the identity.
scikit-learn's KDTree, scipy's mode and cKDTree are the real ones. Cases:
  cli_<name>     the `__main__` block on a case's files: every file it writes in --output_dir (bytes). The smoothing case's
                 seed is one where no vote depends on which of the points tied at the 200th distance scikit-learn keeps
  cache          `__main__` again on cli_plain's part_labels.npy alone (the cached path: coordinates from the PLY)
  clip64_<name>  run_clip's (probabilities, similarities) with torch.float32 read as float64 and `.float()` as `.double()`,
                 i.e. the reference's expressions in fp64; plus the fp32 labels of clip_part_segmentation
  vote_k<k>      local_post_process_segmentation on jittered (tie-free) coordinates for k in (1, 2, 16, 200)
  str2bool       the reference's str2bool on a list of strings (1 / 0, or -1 for ArgumentTypeError)
"""
import argparse
import ast
import io
import json
import logging
import os
import shutil
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

STR2BOOL_INPUTS = ["yes", "true", "True", "t", "y", "1", "no", "false", "False", "f", "n", "0", "TRUE", "Yes", "NO", "F", "2", "", "on"]
VOTE_KS = (1, 2, 16, 200)


def cases():
    """name -> dict(D, C, bounds, feats fp16 (D,D,D,C), mask float32 (D,D,D), table (P,C) fp32, props, wrap, smooth,
    verts float64 (N,3), colors uint8 (N,3))."""
    out = {}

    def make(name, D, C, P, occ, smooth, seed, wrap, bounds):
        rng = np.random.default_rng(seed)
        table = rng.normal(0.0, 1.0, (P, C)).astype(np.float32)
        mask = (rng.uniform(size=(D, D, D)) < occ).astype(np.float32)
        mask[mask > 0] = rng.choice(np.array([1.0, 0.5, np.nan, 3.0], np.float32), int((mask > 0).sum()), p=[0.85, 0.05, 0.05, 0.05])
        # spatially coherent parts: the part of a voxel is set by its position, one part (the last) is never chosen
        ii, jj, kk = np.meshgrid(*(np.arange(D),) * 3, indexing="ij")
        part = ((ii * 2 // D) + 2 * (jj * 2 // D) + (kk * 3 // D)) % (P - 1)
        flip = rng.uniform(size=(D, D, D)) < 0.15
        part = np.where(flip, rng.integers(0, P - 1, (D, D, D)), part)
        feats = 2.5 * table[part] + rng.normal(0.0, 1.0, (D, D, D, C)).astype(np.float32)
        feats = feats.astype(np.float16)
        occupied = np.argwhere(mask.astype(bool))
        if name == "plain":
            feats[tuple(occupied[3])] = 0                          # a zero row: NaN similarities, label 0
        lo, hi = bounds
        axes = [torch.linspace(lo[i], hi[i], D).numpy() for i in range(3)]
        pts = np.stack([axes[0][occupied[:, 0]], axes[1][occupied[:, 1]], axes[2][occupied[:, 2]]], 1).astype(np.float64)
        verts = pts + rng.uniform(-1e-7, 1e-7, pts.shape)          # Open3D's fp64 voxel centres, one per occupied voxel
        colors = rng.integers(0, 256, (len(verts), 3)).astype(np.uint8)
        names = [f"part {i}" for i in range(P)]
        props = {}
        for i, nm in enumerate(names):
            pr = {"density": float(rng.uniform(100, 3000)), "E": float(10 ** rng.uniform(4, 9)), "nu": float(rng.uniform(0.2, 0.45)),
                  "material_id": int(i % 7)}
            if i == 1:
                pr = {"density": 321.5}                            # E, nu and material_id from the defaults
            props[nm] = pr
        out[name] = dict(D=D, C=C, bounds=bounds, feats=feats, mask=mask, table=table, props=props, wrap=wrap, smooth=smooth,
                         verts=verts, colors=colors)

    make("plain", 9, 16, 3, 0.45, False, 101, True, ((-0.4, -0.3, -0.2), (0.5, 0.35, 0.3)))
    make("smooth", 12, 24, 5, 0.65, True, 203, False, ((-1.0, -0.8, -0.5), (1.0, 0.9, 0.6)))
    return out


def ply_bytes(verts, colors):
    """An Open3D-style binary little-endian point cloud: double x y z, uchar red green blue."""
    dt = np.dtype([("x", "<f8"), ("y", "<f8"), ("z", "<f8"), ("red", "u1"), ("green", "u1"), ("blue", "u1")])
    t = np.zeros(len(verts), dt)
    t["x"], t["y"], t["z"] = verts[:, 0], verts[:, 1], verts[:, 2]
    t["red"], t["green"], t["blue"] = colors[:, 0], colors[:, 1], colors[:, 2]
    head = ["ply", "format binary_little_endian 1.0", "comment Created by Open3D", f"element vertex {len(verts)}",
            "property double x", "property double y", "property double z", "property uchar red", "property uchar green",
            "property uchar blue", "end_header"]
    return ("\n".join(head) + "\n").encode("ascii") + t.tobytes()


def write_inputs(c, d):
    """The case's files under d: clip_features.npz (+ _features.npy, _mask.npy), occupancy.ply, materials.json and
    query_embeddings.npy. Returns their paths."""
    os.makedirs(d, exist_ok=True)
    lo, hi = c["bounds"]
    grid = os.path.join(d, "clip_features.npz")
    np.savez(grid, min_bounds=np.array(lo, np.float32), max_bounds=np.array(hi, np.float32), grid_shape=np.array([c["D"]] * 3, np.int64))
    np.save(os.path.join(d, "clip_features_features.npy"), c["feats"])
    np.save(os.path.join(d, "clip_features_mask.npy"), c["mask"])
    occ = os.path.join(d, "occupancy.ply")
    with open(occ, "wb") as f:
        f.write(ply_bytes(c["verts"], c["colors"]))
    mat = os.path.join(d, "materials.json")
    with open(mat, "w") as f:
        json.dump({"material_dict": c["props"], "other": 1} if c["wrap"] else c["props"], f, indent=2)
    emb = os.path.join(d, "query_embeddings.npy")
    np.save(emb, c["table"])
    return dict(grid=grid, occ=occ, mat=mat, emb=emb)


# ------------------------------------------------------------------------------------------------ stand-ins
class _Colormap:
    N = 10
    HEX = ("#1f77b4", "#ff7f0e", "#2ca02c", "#d62728", "#9467bd", "#8c564b", "#e377c2", "#7f7f7f", "#bcbd22", "#17becf")

    def __call__(self, i):
        h = self.HEX[int(i)]
        return tuple(int(h[k:k + 2], 16) / 255 for k in (1, 3, 5)) + (1.0,)


def _trimesh_load(path):
    with open(path, "rb") as f:
        props, count = [], 0
        while True:
            w = f.readline().decode().split()
            if w[0] == "end_header":
                break
            if w[0] == "element":
                count = int(w[2])
            elif w[0] == "property":
                props.append((w[2], {"double": "<f8", "float": "<f4", "uchar": "u1"}[w[1]]))
        t = np.frombuffer(f.read(), dtype=np.dtype(props), count=count)
    colors = np.column_stack([t["red"], t["green"], t["blue"], np.full(count, 255, np.uint8)])
    return types.SimpleNamespace(vertices=np.column_stack([t["x"], t["y"], t["z"]]).astype(np.float64), colors=colors)


class _F64:
    """encode_text's result in the fp64 run: `.float()` gives float64."""

    def __init__(self, t):
        self.t = t

    def float(self):
        return self.t.double()


class _Torch64:
    """torch with float32 read as float64 (run_clip's `.to(torch.float32)`)."""
    float32 = torch.float64

    def __getattr__(self, name):
        return getattr(torch, name)


def _clip(table, f64=False):
    class Model:
        def encode_text(self, tokens):
            t = torch.from_numpy(table)[tokens.cpu()]
            return _F64(t) if f64 else t
    return types.SimpleNamespace(load=lambda name, device=None: (Model(), None),
                                 tokenize=lambda queries: torch.arange(len(queries)))


def extract(path, names, ns):
    tree = ast.parse(open(path).read())
    for node in tree.body:
        if isinstance(node, (ast.FunctionDef, ast.ClassDef)) and node.name in names:
            exec(compile(ast.Module(body=[node], type_ignores=[]), path, "exec"), ns)
    return tree


def ns_from_reference(ref, table, f64=False):
    from make_network_files_golden import PlyData, PlyElement
    from scipy.stats import mode
    from sklearn.neighbors import KDTree
    ns = {"np": np, "torch": _Torch64() if f64 else torch, "os": os, "json": json, "logging": logging, "argparse": argparse,
          "Tuple": tuple, "Dict": dict, "List": list, "PlyData": PlyData, "PlyElement": PlyElement,
          "plt": types.SimpleNamespace(colormaps={"tab10": _Colormap()}), "trimesh": types.SimpleNamespace(load=_trimesh_load),
          "clip": _clip(table, f64), "CLIPArgs": types.SimpleNamespace(model_name="ViT-L/14@336px"), "KDTree": KDTree, "mode": mode,
          "tqdm": lambda it, **kw: it, "set_logger": lambda *a, **k: None}
    extract(os.path.join(ref, "pixie", "utils.py"), {"str2bool", "load_json"}, ns)
    seg = os.path.join(ref, "pixie", "voxel", "segmentation.py")
    tree = extract(seg, {"get_initial_voxel_grid_from_saved", "load_occupancy_grid", "run_clip", "clip_part_segmentation",
                         "local_post_process_segmentation", "save_segmented_point_cloud"}, ns)
    ns["get_initial_voxel_grid_from_saved"].__defaults__ = (None, "cpu")
    ns["load_occupancy_grid"].__defaults__ = ("cpu",)
    ns["clip_part_segmentation"].__defaults__ = (None, "cpu", 0.1)
    main = [n for n in tree.body if isinstance(n, ast.If) and "__main__" in ast.unparse(n.test)][0]
    ns["__main_body__"] = compile(ast.Module(body=main.body, type_ignores=[]), seg, "exec")
    return ns


def run_main(ns, argv):
    old = sys.argv
    sys.argv = ["segmentation.py"] + argv
    try:
        exec(ns["__main_body__"], ns)
    finally:
        sys.argv = old


def main():
    ref = os.environ["PIXIE_REFERENCE"]
    logging.disable(logging.CRITICAL)
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        for name, c in cases().items():
            p = write_inputs(c, os.path.join(tmp, name))
            ns = ns_from_reference(ref, c["table"])
            od = os.path.join(tmp, name, "out")
            os.makedirs(od)                                  # the reference saves part_labels.npy before creating it
            run_main(ns, ["--grid_feature_path", p["grid"], "--occupancy_path", p["occ"], "--output_dir", od, "--material_dict_path",
                          p["mat"], "--use_spatial_smoothing", "true" if c["smooth"] else "false"])
            for f in sorted(os.listdir(od)):
                out[f"cli_{name}/{f}"] = np.frombuffer(open(os.path.join(od, f), "rb").read(), np.uint8)
            queries = list(c["props"].keys())
            coords, labels, scores, _ = ns["clip_part_segmentation"](p["grid"], queries)
            out[f"clip64_{name}/labels32"] = labels.numpy()
            out[f"clip64_{name}/scores32"] = scores.numpy()
            ns64 = ns_from_reference(ref, c["table"], f64=True)
            feats, _, _ = ns64["get_initial_voxel_grid_from_saved"](p["grid"])
            probs, sims = ns64["run_clip"](queries, feats, 0.1, device="cpu")
            out[f"clip64_{name}/probs"] = probs.numpy()
            out[f"clip64_{name}/sims"] = sims.numpy()
            if name == "plain":                              # the cached path: only part_labels.npy is kept
                for f in os.listdir(od):
                    if f != "part_labels.npy":
                        os.remove(os.path.join(od, f))
                run_main(ns, ["--grid_feature_path", p["grid"], "--occupancy_path", p["occ"], "--output_dir", od,
                              "--material_dict_path", p["mat"], "--overwrite", "False"])
                for f in sorted(os.listdir(od)):
                    out[f"cache/{f}"] = np.frombuffer(open(os.path.join(od, f), "rb").read(), np.uint8)
                shutil.rmtree(od)
        c = cases()["smooth"]
        ns = ns_from_reference(ref, c["table"])
        coords, labels = vote_inputs()
        for k in VOTE_KS:
            out[f"vote_k{k}"] = ns["local_post_process_segmentation"](torch.from_numpy(coords), torch.from_numpy(labels), k=k).numpy()
        res = []
        for v in STR2BOOL_INPUTS:
            try:
                res.append(int(ns["str2bool"](v)))
            except argparse.ArgumentTypeError:
                res.append(-1)
        out["str2bool"] = np.array(res, np.int64)
    buf = io.BytesIO()
    np.savez_compressed(buf, **dict(sorted(out.items())))
    path = os.path.join(HERE, "segmentation_golden.npz")
    with open(path, "wb") as f:
        f.write(buf.getvalue())
    print(f"wrote {path} ({os.path.getsize(path)} bytes, {len(out)} arrays)")


def vote_inputs():
    """Jittered (tie-free) float32 coordinates of 1500 points and spatially coherent labels in [0, 5)."""
    rng = np.random.default_rng(303)
    pts = rng.uniform(-1.0, 1.0, (1500, 3)).astype(np.float32)
    labels = ((pts[:, 0] > 0).astype(np.int64) + 2 * (pts[:, 1] > 0.3)) % 5
    flip = rng.uniform(size=1500) < 0.25
    labels = np.where(flip, rng.integers(0, 5, 1500), labels).astype(np.int64)
    return pts, labels


if __name__ == "__main__":
    main()
