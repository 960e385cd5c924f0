"""Generates tests/golden/scene_files_golden.npz by EXECUTING THE REFERENCE'S OWN scene-loading code on the CPU:
GaussianModel.load_ply (gaussian-splatting/scene/gaussian_model.py:215-260) with build_rotation / build_scaling_rotation /
strip_symmetric (utils/general_utils.py:64-110), the sigmoid / exp activations and get_features, the opacity mask of
gs_simulation.py:405, decode_param_json (utils/decode_param.py), generate_rotation_matrices
(utils/transformation_utils.py:23-51), load_point_cloud and load_e_field_from_ply (gs_simulation.py:108-202, :246-250) and
searchForMaxIteration (utils/system_utils.py:26-28). PIXIE_REFERENCE names a checkout of the reference:

    PIXIE_REFERENCE=<checkout> python tests/golden/make_scene_files_golden.py

The functions are pulled out of the reference files with `ast` and exec'd with a `torch` that ignores device="cuda" (and
`.cuda()`) and a plyfile stand-in that parses the header the way PlyData.read does (binary little-endian, scalar
properties). Each file the reference reads is stored as bytes. Cases:
  ckpt_k{1,4,9,16}     random checkpoints in save_ply's property order (40 rows)
  ckpt_perm            K = 4, properties shuffled, with extra float / int32 properties (a 63-word row)
  ckpt_edge            K = 16: logits in a band of float32 ulps around the logits of 0.02 and 0.05, NaN / +-Inf logits,
                       zero, 1e-30 and 1e20 quaternions, log scales at +-89 and +-100
  for each: pos, shs, opacity, cov and the masks at 0.02 and 0.05
  configs              the 22 shipped physics configs and the edge configs as JSON text, and what decode_param_json returns
                       (JSON text, key order kept) or the exception it raises
  rot_*                generate_rotation_matrices for every config's lists and for negative, 360 and multi-rotation lists
  cloud / cloud_noconf / efield   load_point_cloud and load_e_field_from_ply on map_pred_to_ply-layout files
  iters                searchForMaxIteration on iteration_100 / 7000 / 30000
"""
import ast
import glob
import io
import json
import os
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ["PIXIE_REFERENCE"]
PG = os.path.join(REF, "third_party", "PhysGaussian")
GS = os.path.join(PG, "gaussian-splatting")
TYPES = {"f4": "float", "i4": "int", "u1": "uchar"}


def extract(path, names, ns, cls=None):
    for node in ast.parse(open(path).read()).body:
        body = node.body if cls and isinstance(node, ast.ClassDef) and node.name == cls else [node]
        for m in body:
            if isinstance(m, (ast.FunctionDef, ast.ClassDef)) and m.name in names:
                exec(compile(ast.Module(body=[m], type_ignores=[]), path, "exec"), ns)


class _CpuTorch(types.ModuleType):
    def __getattr__(self, name):
        return getattr(torch, name)

    @staticmethod
    def tensor(*a, device=None, **k):
        return torch.tensor(*a, **k)

    @staticmethod
    def zeros(*a, device=None, **k):
        return torch.zeros(*a, **k)

    @staticmethod
    def ones(*a, device=None, **k):
        return torch.ones(*a, **k)


class _Prop:
    def __init__(self, name):
        self.name = name


class _Element:
    def __init__(self, data):
        self.data = data
        self.properties = [_Prop(n) for n in data.dtype.names]

    def __getitem__(self, k):
        return self.data[k]

    def __contains__(self, k):
        return k in self.data.dtype.names


class PlyData:
    """plyfile.PlyData.read for binary little-endian files with scalar properties."""
    _NP = {"float": "<f4", "int": "<i4", "uchar": "u1", "double": "<f8"}

    def __init__(self, elements):
        self.elements = elements

    def __getitem__(self, name):
        return self.elements[0]

    @classmethod
    def read(cls, path):
        with open(path, "rb") as f:
            assert f.readline() == b"ply\n"
            props, count = [], 0
            while True:
                w = f.readline().decode().split()
                if w[0] == "end_header":
                    break
                if w[0] == "format":
                    assert w[1] == "binary_little_endian"
                elif w[0] == "element":
                    count = int(w[2])
                elif w[0] == "property":
                    props.append((w[2], cls._NP[w[1]]))
            data = np.frombuffer(f.read(), dtype=np.dtype(props), count=count)
        return cls([_Element(data)])


def ply_bytes(arr: np.ndarray, comment=True) -> bytes:
    head = ["ply", "format binary_little_endian 1.0"] + (["comment made for the scene-files tests"] if comment else []) + \
           [f"element vertex {len(arr)}"] + [f"property {TYPES[arr.dtype[n].str[1:]]} {n}" for n in arr.dtype.names] + ["end_header"]
    return ("\n".join(head) + "\n").encode() + arr.tobytes()


def namespace():
    ns = {"np": np, "torch": _CpuTorch("torch"), "os": os, "json": json, "PlyData": PlyData, "nn": torch.nn}
    extract(os.path.join(GS, "utils", "general_utils.py"), {"build_rotation", "build_scaling_rotation", "strip_lowerdiag", "strip_symmetric"}, ns)
    extract(os.path.join(GS, "scene", "gaussian_model.py"), {"load_ply"}, ns, cls="GaussianModel")
    extract(os.path.join(GS, "utils", "system_utils.py"), {"searchForMaxIteration"}, ns)
    extract(os.path.join(PG, "utils", "decode_param.py"), {"decode_param_json"}, ns)
    extract(os.path.join(PG, "utils", "transformation_utils.py"), {"generate_rotation_matrix", "generate_rotation_matrices"}, ns)
    extract(os.path.join(PG, "gs_simulation.py"), {"load_point_cloud", "load_e_field_from_ply"}, ns)
    return ns


def checkpoint_array(rng, n, K, order=None, extra=()):
    names = ["x", "y", "z", "nx", "ny", "nz", "f_dc_0", "f_dc_1", "f_dc_2"] + [f"f_rest_{i}" for i in range(3 * K - 3)] + \
            ["opacity", "scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3"]
    dt = [(nm, "<f4") for nm in names] + list(extra)
    if order is not None:
        dt = [dt[i] for i in order]
    a = np.zeros(n, dtype=dt)
    for nm in a.dtype.names:
        if nm.startswith("n"):
            continue
        if a.dtype[nm] == np.int32:
            a[nm] = rng.integers(-5, 5, n)
        elif nm.startswith("scale"):
            a[nm] = rng.uniform(-7, -1, n)
        elif nm == "opacity":
            a[nm] = rng.normal(-2.5, 2.5, n)
        else:
            a[nm] = rng.normal(0, 1, n)
    return a


def run_load(ns, blob, K):
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "point_cloud.ply")
        open(p, "wb").write(blob)
        g = types.SimpleNamespace(max_sh_degree=int(round(K ** 0.5)) - 1)
        ns["load_ply"](g, p)
    L = ns["build_scaling_rotation"](torch.exp(g._scaling), g._rotation)
    cov = ns["strip_symmetric"](L @ L.transpose(1, 2))
    opacity = torch.sigmoid(g._opacity)
    out = {"pos": g._xyz.detach(), "shs": torch.cat((g._features_dc, g._features_rest), dim=1).detach(), "opacity": opacity.detach(),
           "cov": cov.detach()}
    out = {k: v.numpy() for k, v in out.items()}
    for thr in (0.02, 0.05):
        out[f"mask_{thr}"] = (opacity[:, 0] > thr).numpy()
    return out


def edge_rows(rng, K):
    a = checkpoint_array(rng, 0, K)
    rows = []
    for target in (0.02, 0.05):
        base = np.float32(np.log(target / (1 - target)))
        for d in range(-12, 13):
            rows.append(("opacity", np.float32(base + np.float32(d) * np.spacing(base))))
    for v in (np.nan, np.inf, -np.inf):
        rows.append(("opacity", np.float32(v)))
    for q in ((0, 0, 0, 0), (1e-30, 0, 0, 0), (1e-30, 1e-30, 1e-30, 1e-30), (1e20, 0, 0, 0), (1e20, 1e20, -1e20, 1e20), (0, 0, 0, 1e-30)):
        rows.append(("rot", np.float32(q)))
    for s in ((89, -3, -3), (-89, -3, -3), (100, 0, 0), (-100, -100, -100), (88, 88, 88)):
        rows.append(("scale", np.float32(s)))
    a = checkpoint_array(rng, len(rows), K)
    a["opacity"] = 1.0
    for i, (kind, v) in enumerate(rows):
        if kind == "opacity":
            a["opacity"][i] = v
        elif kind == "rot":
            for j in range(4):
                a[f"rot_{j}"][i] = v[j]
        else:
            for j in range(3):
                a[f"scale_{j}"][i] = v[j]
    return a


def to_json(obj):
    return json.dumps(obj, allow_nan=True)


def main():
    torch.Tensor.cuda = lambda self, *a, **k: self          # generate_rotation_matrix ends in .cuda(); stay on the CPU
    ns = namespace()
    rng = np.random.default_rng(2026)
    out = {}
    cases = {f"ckpt_k{K}": (checkpoint_array(rng, 40, K), K) for K in (1, 4, 9, 16)}
    order = list(rng.permutation(14 + 3 * 4 + 2))
    cases["ckpt_perm"] = (checkpoint_array(rng, 40, 4, order=order, extra=[("extra_a", "<f4"), ("label", "<i4")]), 4)
    cases["ckpt_edge"] = (edge_rows(rng, 16), 16)
    for name, (arr, K) in cases.items():
        blob = ply_bytes(arr)
        out[f"{name}/file"] = np.frombuffer(blob, dtype=np.uint8)
        out[f"{name}/K"] = np.int32(K)
        for k, v in run_load(ns, blob, K).items():
            out[f"{name}/{k}"] = v

    configs = sorted(glob.glob(os.path.join(PG, "config", "*", "custom_*_config.json")))
    texts = {os.path.basename(p): open(p).read() for p in configs}
    texts["empty.json"] = "{}"
    texts["nu_high.json"] = json.dumps({"nu": 0.6})
    texts["nu_negative.json"] = json.dumps({"nu": -0.1})
    for k in ("point", "size", "E", "nu"):
        entry = {"point": [1, 1, 1], "size": [0.1, 0.1, 0.1], "E": 1e4, "nu": 0.3}
        del entry[k]
        texts[f"additional_no_{k}.json"] = json.dumps({"additional_material_params": [entry]})
    texts["additional_density.json"] = json.dumps({"density": 300.0, "additional_material_params": [
        {"point": [1, 1, 1], "size": [0.1, 0.1, 0.1], "E": 1e4, "nu": 0.3}, {"point": [0, 1, 1], "size": [0.2, 0.1, 0.1], "E": 1e3, "nu": 0.2, "density": 50}]})
    texts["filling_defaults.json"] = json.dumps({"n_grid": 32, "particle_filling": {"visualize": True}})
    decoded, rot_lists = {}, {}
    with tempfile.TemporaryDirectory() as d:
        for name, text in texts.items():
            p = os.path.join(d, name)
            open(p, "w").write(text)
            try:
                decoded[name] = {"result": list(ns["decode_param_json"](p))}
            except Exception as e:                                              # noqa: BLE001
                decoded[name] = {"error": type(e).__name__, "message": str(e)}
            if "result" in decoded[name]:
                pre = decoded[name]["result"][3]
                rot_lists[name] = (pre["rotation_degree"], pre["rotation_axis"])
    out["configs/text"] = np.array(to_json(texts))
    out["configs/decoded"] = np.array(to_json(decoded))
    rot_lists.update({"neg": ([-90, -45.5], [0, 2]), "full": ([360], [1]), "multi": ([30, 45.0, 60], [0, 1, 2]),
                      "float_int": ([90.0, 180], [2, 1]), "none": ([], [])})
    out["rot/lists"] = np.array(to_json(rot_lists))
    for name, (deg, ax) in rot_lists.items():
        ms = ns["generate_rotation_matrices"](torch.tensor(deg), ax)
        out[f"rot/{name}"] = np.stack([m.numpy() for m in ms]) if ms else np.zeros((0, 3, 3), np.float32)

    n = 50
    cloud = np.zeros(n, dtype=[("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("part_label", "<i4"), ("density", "<f4"), ("E", "<f4"),
                               ("nu", "<f4"), ("material_id", "<i4"), ("conf", "<f4")])
    for k in cloud.dtype.names:
        cloud[k] = rng.integers(0, 7, n) if cloud.dtype[k] == np.int32 else rng.uniform(0, 2, n)
    noconf = np.zeros(n, dtype=[(k, cloud.dtype[k]) for k in cloud.dtype.names if k not in ("conf", "part_label")])
    for k in noconf.dtype.names:
        noconf[k] = cloud[k]
    with tempfile.TemporaryDirectory() as d:
        for name, arr in (("cloud", cloud), ("cloud_noconf", noconf)):
            blob = ply_bytes(arr)
            p = os.path.join(d, name + ".ply")
            open(p, "wb").write(blob)
            r = ns["load_point_cloud"](p)
            out[f"{name}/file"] = np.frombuffer(blob, dtype=np.uint8)
            out[f"{name}/pos"] = r["pos"].numpy()
            for k in ("density", "E", "nu", "material_id", "part_labels", "conf"):
                out[f"{name}/{k}"] = np.asarray(r[k])
        e = np.zeros(n, dtype=[("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("E", "<f4")])
        e["E"] = rng.uniform(0.01, 1, n)
        blob = ply_bytes(e)
        p = os.path.join(d, "E_field_epoch_07.ply")
        open(p, "wb").write(blob)
        out["efield/file"] = np.frombuffer(blob, dtype=np.uint8)
        out["efield/E"] = ns["load_e_field_from_ply"](p, device="cpu").numpy()
        for it in (100, 7000, 30000):
            os.makedirs(os.path.join(d, "point_cloud", f"iteration_{it}"))
        out["iters/max"] = np.int64(ns["searchForMaxIteration"](os.path.join(d, "point_cloud")))

    buf = io.BytesIO()
    np.savez_compressed(buf, **dict(sorted(out.items())))
    path = os.path.join(HERE, "scene_files_golden.npz")
    with open(path, "wb") as f:
        f.write(buf.getvalue())
    print(f"wrote {path} ({os.path.getsize(path)} bytes, {len(out)} arrays)")


if __name__ == "__main__":
    main()
