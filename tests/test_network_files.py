"""CPU tests of pixie_b200.network_files against tests/golden/network_files_golden.npz, which the reference's own
process_batch, save_predictions, MaterialVoxelDataset, load_test_dataset, generate_metrics_report and map_pred_to_ply
produced (make_network_files_golden.py). The per-voxel counts and sums come from the fp64 oracle
(oracle/network_files_ref.py), which the device kernel is held to in test_gpu_material_metrics.py."""
import hashlib
import json
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import make_network_files_golden as G  # noqa: E402
from oracle import network_files_ref as O  # noqa: E402
from pixie_b200 import network_files as NF  # noqa: E402
from pixie_b200 import scene_files  # noqa: E402

GOLD = np.load(os.path.join(ROOT, "tests", "golden", "network_files_golden.npz"))
CASES = G.metric_cases()


def oracle_batch(c, mask=True):
    gts = [O.normalize_gt(m, G.RANGES) for m in c["mats"]]
    cs = [O.sample_counts_sums(gts[i], c["masks"][i] if mask else None, c["logits"][i], c["cont"][i], G.BG) for i in range(len(gts))]
    return gts, np.array([x[0] for x in cs], np.int64), np.array([x[1] for x in cs], np.float64)


def packed(c, i):
    """save_predictions' combined_pred from the logits: cont, then the one-hot of torch.argmax."""
    pred = torch.from_numpy(c["logits"][i]).argmax(0).numpy()
    return np.concatenate([c["cont"][i], (np.arange(8)[:, None, None, None] == pred[None]).astype(np.float32)])


@pytest.mark.parametrize("name", list(CASES))
def test_counts_and_accuracies_match_the_reference(name):
    _, counts, sums = oracle_batch(CASES[name])
    assert np.array_equal(counts, GOLD[f"batch_{name}/counts"])
    batch, samples = NF.batch_metrics(counts, sums)
    ref_b, ref_s = GOLD[f"batch_{name}/batch"], GOLD[f"batch_{name}/samples"]
    assert batch[0] == ref_b[0]                                                     # bit for bit
    assert [s["seg_acc"] for s in samples] == list(ref_s[:, 0])
    keys = ["cont_mse", "density_mse", "youngs_mse", "poisson_mse"]
    mine = np.array([[s[k] for k in keys] for s in samples])
    np.testing.assert_allclose(np.array(batch[1:]), ref_b[1:], rtol=1e-6, equal_nan=True)
    np.testing.assert_allclose(mine, ref_s[:, 1:], rtol=1e-6, equal_nan=True)


def test_edge_cases_take_the_reference_paths():
    b, s = NF.batch_metrics(*oracle_batch(CASES["d13_n3_edges"])[1:])
    assert s[0]["seg_acc"] == 0.0 and s[0]["density_mse"] == 0.0                  # total == 0, den clamped to 1
    assert s[1]["seg_acc"] == GOLD["batch_d13_n3_edges/samples"][1, 0]
    b, s = NF.batch_metrics(*oracle_batch(CASES["d8_n4_zero_nan"])[1:])
    assert np.isnan(s[3]["youngs_mse"]) and np.isnan(b[1]) and not np.isnan(s[3]["density_mse"])


def test_empty_mask_uses_clamp_and_eps():
    counts = np.array([[0, 0]], np.int64)
    sums = np.array([[0.5, 0.0, 0.0, 0.0]])
    b, s = NF.batch_metrics(counts, sums)
    assert s[0]["density_mse"] == np.float32(0.5) / (np.float32(1) + np.float32(1e-8))
    assert b[0] == 0.0


def test_argmax_oracle_follows_torch():
    x = np.array([[1, np.nan, 3, 3], [1, 2, np.nan, 3], [1, np.nan, 3, 1]], np.float32)
    assert np.array_equal(O.argmax_torch(x), torch.from_numpy(x).argmax(0).numpy())


@pytest.mark.parametrize("name", list(CASES))
def test_saved_files_equal_the_reference_bytes(tmp_path, name, monkeypatch):
    c = CASES[name]
    gts, _, _ = oracle_batch(c)
    monkeypatch.chdir(tmp_path)
    for i in range(len(gts)):
        paths = json.loads(str(GOLD[f"batch_{name}/{i}/info_paths"]))
        info = dict(obj_id=f"obj{i}", sample_id="0", **paths)
        NF.save_predictions("out", info, packed(c, i), gts[i], c["masks"][i])
        for kind in ("pred", "gt", "mask", "info"):
            b = (tmp_path / "out" / f"obj{i}" / f"sample_0_{kind}.npy").read_bytes()
            key = f"batch_{name}/{i}/{kind}"
            if key in GOLD:
                assert b == GOLD[key].tobytes(), kind
            else:
                assert hashlib.sha256(b).hexdigest() == str(GOLD[key + "_sha256"]), kind


def test_dataset_discovery_and_getitem(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    root, stats, ckdir = G.build_dataset_tree("")
    ds = NF.MaterialVoxelDataset(root, grid_size=8, feature_channels=4, problematic_objects=os.path.join(stats, "problematic_objects.json"))
    ref = json.loads(str(GOLD["dataset/obj_ids"]))
    assert set(ds.obj_ids) == set(ref)
    assert ds.obj_ids == [o for o in os.listdir(root) if o in set(ref)]            # os.listdir order
    for k, o in enumerate(ds.obj_ids):
        expect = json.loads(str(GOLD["dataset/getitem"]))[o]
        if expect == "ok":
            mat, mask = ds.load_labels(k)
            assert mat.shape == (8, 8, 8, 4) and mask.dtype == np.float32
        else:
            with pytest.raises(AssertionError):
                ds.load_labels(k)
    seg = os.path.join(ckdir, "epoch_10.pth")
    ids = lambda idx: [ds.obj_ids[i] for i in idx]                                   # noqa: E731
    assert ids(NF.load_test_dataset(ds, "g")) == json.loads(str(GOLD["split_obj/ids"]))
    assert ids(NF.load_test_dataset(ds, None, True, seg)) == json.loads(str(GOLD["split_saved/ids"]))
    assert ids(NF.load_test_dataset(ds, None)) == json.loads(str(GOLD["split_random/dataset"]))
    with pytest.raises(ValueError):
        NF.load_test_dataset(ds, "nope")
    with pytest.raises(AssertionError):
        NF.load_test_dataset(ds, None, True, os.path.join(stats, "x.pth"))


@pytest.mark.parametrize("n,t", [(10, 0.9), (10, 0.5), (7, 0.7)])
def test_random_split(n, t):
    class DS:
        obj_ids = [str(i) for i in range(n)]

        def __len__(self):
            return n
    assert NF.load_test_dataset(DS(), None, train_size=t) == list(GOLD[f"split_random/n{n}_t{int(t * 10)}"])


@pytest.mark.parametrize("world", [1, 2])
@pytest.mark.parametrize("disp", ["sem", "std"])
def test_metrics_report_equals_the_reference(tmp_path, world, disp):
    NF.generate_metrics_report(G.as_all_metrics(G.report_inputs(), world), str(tmp_path), "seg.pth", "cont.pth", disp)
    for f in ("metrics.json", "evaluated_obj_ids.json"):
        assert (tmp_path / f).read_bytes() == GOLD[f"report_w{world}_{disp}/{f}"].tobytes(), f


def test_checkpoint_and_ranges(tmp_path):
    sd = {"a": torch.ones(2)}
    for wrap in ({"model_state_dict": sd, "epoch": 3}, {"state_dict": sd}, sd):
        torch.save(wrap, tmp_path / "c.pth")
        assert NF.load_network_checkpoint(str(tmp_path / "c.pth")).keys() == sd.keys()
    assert NF.load_network_checkpoint(str(tmp_path / "missing.pth")) is None
    (tmp_path / "r.yaml").write_text(json.dumps({"density_p1": 1.5, "density_p99": 3.5, "E_p1": 3.0, "E_p99": 10.0, "nu_p1": 0.2,
                                                 "nu_p99": 0.45, "density_min": 0.0}))
    assert NF.load_normalization_ranges(str(tmp_path / "r.yaml")) == {"density_min": 1.5, "density_max": 3.5, "E_min": 3.0,
                                                                      "E_max": 10.0, "nu_min": 0.2, "nu_max": 0.45}


@pytest.mark.parametrize("variant", ["heuristic", "explicit", "nodp"])
def test_point_cloud_writer_and_world_transform(tmp_path, variant):
    src = tmp_path / "in.ply"
    src.write_bytes(GOLD[f"cloud_{variant}/mapped"].tobytes())
    el = scene_files.read_ply(str(src))
    assert el.dtype == NF.CLOUD_DTYPE                                                   # the reference's property order
    NF.write_material_point_cloud(str(tmp_path / "out.ply"), el.read())
    assert (tmp_path / "out.ply").read_bytes() == GOLD[f"cloud_{variant}/mapped"].tobytes()
    if variant == "nodp":
        return
    dp = tmp_path / "dataparser_transforms.json"
    dp.write_text(str(GOLD["cloud/dataparser"]))
    NF.transform_nerf_to_world(str(src), str(dp), str(tmp_path / "world.ply"))
    assert (tmp_path / "world.ply").read_bytes() == GOLD[f"cloud_{variant}/world"].tobytes()


def test_map_pred_to_ply_rejects_bad_shapes(tmp_path):
    pred, mask, meta, _ = G.cloud_case()
    np.save(tmp_path / "mask.npy", mask[:32, :32, :32])
    np.save(tmp_path / "pred.npy", pred)
    np.savez(tmp_path / "g.npz", **meta)
    with pytest.raises(AssertionError):
        NF.map_pred_to_ply(str(tmp_path / "pred.npy"), str(tmp_path / "mask.npy"), str(tmp_path / "g.npz"), str(tmp_path / "o.ply"))
    np.save(tmp_path / "mask.npy", mask)
    np.save(tmp_path / "pred.npy", pred[:, :32])
    with pytest.raises(ValueError):
        NF.map_pred_to_ply(str(tmp_path / "pred.npy"), str(tmp_path / "mask.npy"), str(tmp_path / "g.npz"), str(tmp_path / "o.ply"))
