"""Generates tests/golden/network_files_golden.npz by EXECUTING THE REFERENCE'S OWN evaluation and mapping code on the CPU:
compute_accuracy / masked_mean (pixie/training_utils.py:68-87), process_batch / save_predictions / load_test_dataset
(WG/trainer/inference_combined.py:48-217), MaterialVoxelDataset (WG/data_utils/my_data.py:19-224), InferenceMetrics /
save_metrics_file / generate_metrics_report (pixie/metrics.py, print_table=False) and unscale_prediction / get_mat_id /
map_pred_to_ply / transform_nerf_to_world (pixie/voxel/map_pred_to_coords.py). PIXIE_REFERENCE names a checkout:

    PIXIE_REFERENCE=<checkout> python tests/golden/make_network_files_golden.py

The functions are pulled out of the reference files with `ast`; the networks are stubs that return the seeded logits and
predictions of `metric_cases()` (which the tests rebuild, so only outputs are stored), and plyfile is a stand-in that
writes the header plyfile writes. Cases:
  batch_<name>   D in (8, 13, 64), N in (1, 3, 4): empty and all-foreground masks, tied and NaN logits, a NaN prediction
                 outside the mask, densities / E at 0 and +-1e-6, ids at background_id. Per batch: the batch metrics, the
                 per-sample metrics, counts, and every saved .npy (bytes for D < 64, sha256 at D = 64)
  dataset        a render_outputs tree with a problematic, an out-of-range, a shape-mismatched and a mask-inconsistent
                 object: the discovered ids and what __getitem__ does with each
  split_*        obj_id, saved test_set.json and random_split selection
  report_*       metrics.json / evaluated_obj_ids.json for one and several samples per object, SE and STD
  cloud_*        mapped_preds.ply and world_mapped_preds.ply (non-unit scale) from a seeded 64^3 prediction
"""
import ast
import hashlib
import io
import json
import logging
import math
import os
import tempfile
import types
from collections import defaultdict
from pathlib import Path

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
RANGES = {"density_min": 1.7031893730163574, "density_max": 3.871432304382324, "E_min": 3.0183002948760986, "E_max": 10.881680488586426,
          "nu_min": 0.21027633547782898, "nu_max": 0.4492689371109009}
BG = 7


def raw_material(rng, D, n_classes=8, bg_frac=0.4):
    """A (D, D, D, 4) material_grid.npy: density, E, nu in and around the normalisation ranges, ids with background."""
    mat = np.zeros((D, D, D, 4), np.float32)
    mat[..., 0] = 10.0 ** rng.uniform(1.0, 4.5, (D, D, D))
    mat[..., 1] = 10.0 ** rng.uniform(2.5, 11.5, (D, D, D))
    mat[..., 2] = rng.uniform(0.15, 0.5, (D, D, D))
    ids = rng.integers(0, n_classes - 1, (D, D, D))
    ids[rng.uniform(size=(D, D, D)) < bg_frac] = BG
    mat[..., 3] = ids
    return mat


def metric_cases():
    """name -> dict(mats [N] raw grids, masks [N], logits (N, 8, D, D, D), cont (N, 3, D, D, D)), all float32."""
    rng = np.random.default_rng(20261018)
    out = {}

    def make(D, N):
        mats = [raw_material(rng, D) for _ in range(N)]
        masks = [(m[..., 3] != BG).astype(np.float32) for m in mats]
        logits = rng.normal(0, 1, (N, 8, D, D, D)).astype(np.float32)
        cont = rng.uniform(-1.2, 1.2, (N, 3, D, D, D)).astype(np.float32)
        return dict(mats=mats, masks=masks, logits=logits, cont=cont)

    out["d8_n1"] = make(8, 1)
    c = make(13, 3)
    c["mats"][0][..., 3] = BG                                   # empty mask: accuracy 0, MSE through clamp + eps
    c["masks"][0][:] = 0
    c["mats"][1][..., 3] = np.where(c["mats"][1][..., 3] == BG, 2, c["mats"][1][..., 3])     # all foreground
    c["masks"][1][:] = 1
    lg = c["logits"][2]
    lg[:, 0, :, :] = 0.5                                         # all classes tied
    lg[3, 1, :, :] = 2.0
    lg[5, 1, :, :] = 2.0                                         # ties on the max
    lg[2, 2, ::2, :] = np.nan                                    # NaN logits
    lg[6, 2, 1::3, :] = np.nan
    out["d13_n3_edges"] = c
    c = make(8, 4)
    m = c["mats"][0]
    flat = m.reshape(-1, 4)
    for k, v in enumerate((0.0, 1e-6, -1e-6, np.float32(1e-6) * np.float32(1.0000001), 0.0, -0.0)):
        flat[k, 0] = v
        flat[k + 8, 1] = v
    flat[:16, 3] = 1                                             # foreground, so the zeros enter the MSE
    c["masks"][0] = (m[..., 3] != BG).astype(np.float32)
    c["mats"][3][0, 0, 0, 3] = BG
    c["masks"][3][0, 0, 0] = 0
    c["cont"][3, 1, 0, 0, 0] = np.nan                            # NaN outside the mask: the reference's MSE is NaN
    out["d8_n4_zero_nan"] = c
    out["d64_n1"] = make(64, 1)
    return out


def cloud_case():
    rng = np.random.default_rng(7)
    pred = np.zeros((11, 64, 64, 64), np.float32)
    pred[:3] = rng.uniform(-1.3, 1.3, (3, 64, 64, 64))
    seg = rng.integers(0, 8, (64, 64, 64))
    pred[3:] = (np.arange(8)[:, None, None, None] == seg[None]).astype(np.float32)
    mask = np.zeros((64, 64, 64), np.float32)
    mask.reshape(-1)[rng.choice(64 ** 3, 300, replace=False)] = 1.0
    meta = dict(min_bounds=np.array([-0.7, -0.4, -0.2]), max_bounds=np.array([0.6, 0.5, 0.9]), grid_shape=np.array([64, 64, 64]))
    dataparser = {"transform": [[0.9, -0.1, 0.05, 0.3], [0.1, 0.95, -0.2, -0.1], [-0.03, 0.2, 0.97, 0.4]], "scale": 0.37}
    return pred, mask, meta, dataparser


# ------------------------------------------------------------------------------------------------------------ generator
TYPES = {"f4": "float", "i4": "int", "u1": "uchar"}


class PlyElement:
    def __init__(self, data):
        self.data = data

    @staticmethod
    def describe(data, name):
        return PlyElement(data)


class PlyData:
    """plyfile's PlyData for one binary little-endian vertex element: write() emits plyfile's header and the rows."""

    def __init__(self, elements, text=False):
        self.elements = elements

    def __getitem__(self, name):
        return self.elements[0]

    def write(self, path):
        d = self.elements[0].data
        lines = ["ply", "format binary_little_endian 1.0", f"element vertex {len(d)}"] + \
                [f"property {TYPES[d.dtype[n].str[1:]]} {n}" for n in d.dtype.names] + ["end_header"]
        with open(path, "wb") as f:
            f.write(("\n".join(lines) + "\n").encode("ascii"))
            f.write(d.astype(d.dtype.newbyteorder("<")).tobytes())

    @classmethod
    def read(cls, path):
        with open(path, "rb") as f:
            props, count = [], 0
            while True:
                w = f.readline().decode().split()
                if w[0] == "end_header":
                    break
                if w[0] == "element":
                    count = int(w[2])
                elif w[0] == "property":
                    props.append((w[2], {"float": "<f4", "int": "<i4", "uchar": "u1"}[w[1]]))
            data = np.frombuffer(f.read(), dtype=np.dtype(props), count=count).copy()
        return cls([PlyElement(data)])


def extract(path, names, ns, cls=None):
    for node in ast.parse(open(path).read()).body:
        body = node.body if cls and isinstance(node, ast.ClassDef) and node.name == cls else [node]
        for m in body:
            if isinstance(m, (ast.FunctionDef, ast.ClassDef)) and m.name in names:
                exec(compile(ast.Module(body=[m], type_ignores=[]), path, "exec"), ns)


def ns_from_reference(ref):
    wg = os.path.join(ref, "third_party", "Wavelet-Generation")
    ns = {"np": np, "torch": torch, "os": os, "json": json, "math": math, "logging": logging, "Path": Path, "defaultdict": defaultdict,
          "PlyData": PlyData, "PlyElement": PlyElement, "get_obj_class_for_id": lambda obj_id, cfg: "UNKNOWN",
          "Subset": torch.utils.data.Subset, "DictConfig": object, "Tuple": tuple, "Dict": dict, "List": list, "Optional": object}
    extract(os.path.join(ref, "pixie", "utils.py"), {"load_json", "save_json"}, ns)
    extract(os.path.join(ref, "pixie", "training_utils.py"), {"masked_mean", "compute_accuracy"}, ns)
    extract(os.path.join(ref, "pixie", "metrics.py"), {"InferenceMetrics", "save_metrics_file", "generate_metrics_report"}, ns)
    extract(os.path.join(wg, "trainer", "inference_combined.py"), {"process_batch", "save_predictions", "load_test_dataset"}, ns)
    extract(os.path.join(wg, "data_utils", "my_data.py"), {"MaterialVoxelDataset"}, ns)
    extract(os.path.join(ref, "pixie", "voxel", "map_pred_to_coords.py"),
            {"unscale_prediction", "get_mat_id", "map_pred_to_ply", "transform_nerf_to_world"}, ns)
    return ns


def config(root, stats_dir, D=8, seg_ckpt=""):
    S = types.SimpleNamespace
    tr = S(to_normalize=True, feature_type="clip", target_obj_classes=None, default_grid_size=D, feature_channels=4, in_material_channels=4,
           num_material_classes=8, sample_id=0, background_id=BG, enforce_mask_consistency=True,
           inference=S(use_saved_test_split=False), training=S(train_size=0.9), **RANGES)
    return S(training=tr, paths=S(render_outputs_dir=root, normalization_stats_dir=stats_dir), _seg=seg_ckpt)


def write_scene(root, obj, mat, mask, C_feat=4, feat_D=None):
    D = mat.shape[0] if feat_D is None else feat_D
    os.makedirs(os.path.join(root, obj, "sample_0"), exist_ok=True)
    np.save(os.path.join(root, obj, "clip_features_features.npy"), np.zeros((D, D, D, C_feat), np.float16))
    np.save(os.path.join(root, obj, "clip_features_mask.npy"), mask)
    np.save(os.path.join(root, obj, "sample_0", "material_grid.npy"), mat)


def sha(b):
    return hashlib.sha256(b).hexdigest()


def run_batch(ns, name, c, out, tmp):
    N, D = c["logits"].shape[0], c["logits"].shape[2]
    root = os.path.join(tmp, name)
    for i in range(N):
        write_scene(root, f"obj{i}", c["mats"][i], c["masks"][i])
    cfg = config(root, os.path.join(tmp, "nostats"), D)
    ds = ns["MaterialVoxelDataset"](cfg)
    order = [ds.obj_ids.index(f"obj{i}") for i in range(N)]
    batch = torch.utils.data.default_collate([ds[k] for k in order])
    seg = lambda x: torch.from_numpy(c["logits"])                                        # noqa: E731
    cont = lambda x: torch.from_numpy(c["cont"])                                         # noqa: E731
    m = ns["InferenceMetrics"]()
    od = os.path.join(tmp, name + "_out")
    ns["process_batch"](seg, cont, batch, cfg, "cpu", m, od)
    out[f"batch_{name}/batch"] = np.array([m.seg_accuracies[0], m.cont_mse_values[0], m.density_mse_values[0], m.youngs_mse_values[0],
                                           m.poisson_mse_values[0]], np.float64)
    keys = ["seg_acc", "cont_mse", "density_mse", "youngs_mse", "poisson_mse"]
    out[f"batch_{name}/samples"] = np.array([[m.obj_metrics[f"obj{i}"][k][0] for k in keys] for i in range(N)], np.float64)
    mat_id, mask = batch[2], batch[3]
    pred = torch.from_numpy(c["logits"]).argmax(1)
    out[f"batch_{name}/counts"] = np.array([[int(mask[i].bool().sum()), int(((pred[i] == mat_id[i]) & mask[i].bool()).sum())]
                                            for i in range(N)], np.int64)
    for i in range(N):
        for kind in ("pred", "gt", "mask", "info"):
            b = open(os.path.join(od, f"obj{i}", f"sample_0_{kind}.npy"), "rb").read()
            if D < 64 or kind == "info":
                out[f"batch_{name}/{i}/{kind}"] = np.frombuffer(b, np.uint8)
            else:
                out[f"batch_{name}/{i}/{kind}_sha256"] = np.array(sha(b))
        out[f"batch_{name}/{i}/info_paths"] = np.array(json.dumps(
            {k: ds.__getitem__(order[i])[4][k] for k in ("data_path", "feature_path", "mask_path")}))


def build_dataset_tree(tmp):
    """render_outputs/ (objects a..h), stats/problematic_objects.json and ckpt/test_set.json under `tmp`."""
    rng = np.random.default_rng(5)
    root = os.path.join(tmp, "render_outputs")
    stats = os.path.join(tmp, "stats")
    os.makedirs(stats)
    for obj in ("a", "b", "c", "d", "e", "f", "g"):
        mat = raw_material(rng, 8)
        mask = (mat[..., 3] != BG).astype(np.float32)
        if obj == "c":
            mat[0, 0, 0, 3] = 8                                   # id out of range
        if obj == "e":
            mask[1, 1, 1] = 1.0 - mask[1, 1, 1]                   # mask inconsistent with the ids
        write_scene(root, obj, mat, mask, feat_D=9 if obj == "d" else None)     # d: shape mismatch
    os.makedirs(os.path.join(root, "h"))                          # no files at all
    json.dump(["b"], open(os.path.join(stats, "problematic_objects.json"), "w"))
    ckdir = os.path.join(tmp, "ckpt")
    os.makedirs(ckdir)
    json.dump(["f", "a", "zz"], open(os.path.join(ckdir, "test_set.json"), "w"))
    return root, stats, ckdir


def run_dataset(ns, out, tmp):
    root, stats, ckdir = build_dataset_tree(tmp)
    cfg = config(root, stats, 8)
    ds = ns["MaterialVoxelDataset"](cfg)
    out["dataset/obj_ids"] = np.array(json.dumps(ds.obj_ids))
    res = {}
    for k, o in enumerate(ds.obj_ids):
        try:
            ds[k]
            res[o] = "ok"
        except AssertionError:
            res[o] = "AssertionError"
    out["dataset/getitem"] = np.array(json.dumps(res))

    ns["get_checkpoint_paths"] = lambda c: (c._seg, "")
    cfg._seg = os.path.join(ckdir, "epoch_10.pth")
    sub, _ = ns["load_test_dataset"](cfg, "g")
    out["split_obj/ids"] = np.array(json.dumps([ds.obj_ids[i] for i in sub.indices]))
    cfg.training.inference.use_saved_test_split = True
    sub, _ = ns["load_test_dataset"](cfg, None)
    out["split_saved/ids"] = np.array(json.dumps([ds.obj_ids[i] for i in sub.indices]))
    cfg.training.inference.use_saved_test_split = False
    for n, ts in ((10, 0.9), (10, 0.5), (7, 0.7)):
        sub = torch.utils.data.random_split(list(range(n)), [int(ts * n), n - int(ts * n)], generator=torch.Generator().manual_seed(42))[1]
        out[f"split_random/n{n}_t{int(ts * 10)}"] = np.array(sub.indices, np.int64)
    sub, _ = ns["load_test_dataset"](cfg, None)
    out["split_random/dataset"] = np.array(json.dumps([ds.obj_ids[i] for i in sub.indices]))


def report_inputs():
    """Per-rank metric lists as gather_all_metrics returns them: one and several samples per object, two ranks."""
    rng = np.random.default_rng(11)
    ranks = []
    for r, objs in enumerate((["o1", "o2", "o1"], ["o3", "o2", "o4"])):
        m = {"seg": [], "cont": [], "dens": [], "young": [], "pois": [], "ids": [], "obj": {}}
        for o in objs:
            s = {"seg_acc": float(np.float32(rng.uniform())), "density_mse": float(np.float32(rng.uniform(0, 0.3))),
                 "youngs_mse": float(np.float32(rng.uniform(0, 0.3))), "poisson_mse": float(np.float32(rng.uniform(0, 0.3)))}
            s["cont_mse"] = (s["density_mse"] + s["youngs_mse"] + s["poisson_mse"]) / 3.0
            m["obj"].setdefault(o, {k: [] for k in s})
            for k, v in s.items():
                m["obj"][o][k].append(v)
            m["ids"].append(o)
        for k in ("seg", "cont", "dens", "young", "pois"):
            m[k].append(float(np.float32(rng.uniform())))
        ranks.append(m)
    return ranks


def as_all_metrics(ranks, world=2):
    ranks = ranks[:world]
    return [[m[k] for m in ranks] for k in ("seg", "cont", "dens", "young", "pois", "ids")] + \
           [[{o: defaultdict(list, {k: list(v) for k, v in d.items()}) for o, d in m["obj"].items()} for m in ranks]]


def run_report(ns, out, tmp):
    ranks = report_inputs()
    for world in (1, 2):
        for disp in ("sem", "std"):
            od = os.path.join(tmp, f"report_{world}_{disp}")
            os.makedirs(od)
            ns["generate_metrics_report"](None, as_all_metrics(ranks, world), od, "seg.pth", "cont.pth", disp, False)
            for f in ("metrics.json", "evaluated_obj_ids.json"):
                out[f"report_w{world}_{disp}/{f}"] = np.frombuffer(open(os.path.join(od, f), "rb").read(), np.uint8)


def run_cloud(ns, out, tmp):
    pred, mask, meta, dp = cloud_case()
    d = os.path.join(tmp, "cloud")
    os.makedirs(d)
    np.save(os.path.join(d, "pred.npy"), pred)
    np.save(os.path.join(d, "mask.npy"), mask)
    np.savez(os.path.join(d, "clip_features.npz"), **meta)
    json.dump(dp, open(os.path.join(d, "dataparser_transforms.json"), "w"))
    cfg = types.SimpleNamespace(training=types.SimpleNamespace(**RANGES))
    for variant, dp_path in (("heuristic", None), ("explicit", os.path.join(d, "dataparser_transforms.json"))):
        o, w = os.path.join(d, f"mapped_{variant}.ply"), os.path.join(d, f"world_{variant}.ply")
        ns["map_pred_to_ply"](os.path.join(d, "pred.npy"), os.path.join(d, "mask.npy"), os.path.join(d, "clip_features.npz"), o, "obj",
                              world_output_path=w, dataparser_path=dp_path, cfg=cfg)
        out[f"cloud_{variant}/mapped"] = np.frombuffer(open(o, "rb").read(), np.uint8)
        out[f"cloud_{variant}/world"] = np.frombuffer(open(w, "rb").read(), np.uint8)
    o = os.path.join(d, "mapped_only.ply")
    ns["map_pred_to_ply"](os.path.join(d, "pred.npy"), os.path.join(d, "mask.npy"), os.path.join(d, "clip_features.npz"), o, "obj", cfg=cfg)
    out["cloud_nodp/mapped"] = np.frombuffer(open(o, "rb").read(), np.uint8)
    out["cloud/dataparser"] = np.array(json.dumps(dp))


def main():
    ns = ns_from_reference(os.environ["PIXIE_REFERENCE"])
    logging.disable(logging.CRITICAL)
    out = {}
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        os.chdir(tmp)                  # relative paths: the pickled info dicts do not depend on where this runs
        try:
            for name, c in metric_cases().items():
                run_batch(ns, name, c, out, "")
            run_dataset(ns, out, "")
            run_report(ns, out, "")
            run_cloud(ns, out, "")
        finally:
            os.chdir(cwd)
    buf = io.BytesIO()
    np.savez_compressed(buf, **dict(sorted(out.items())))
    path = os.path.join(HERE, "network_files_golden.npz")
    with open(path, "wb") as f:
        f.write(buf.getvalue())
    print(f"wrote {path} ({os.path.getsize(path)} bytes, {len(out)} arrays)")


if __name__ == "__main__":
    main()
