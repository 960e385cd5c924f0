"""GPU tests of csrc/material_metrics.cu and the neural-mode command lines: the kernel against the fp64 oracle, the
reference's torch expressions on the same device and the reference fixture (tests/golden/network_files_golden.npz); then
inference_combined -> map_pred_to_coords -> gs_simulation end to end on labelled 64^3 scenes."""
import json
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import make_network_files_golden as G  # noqa: E402
from oracle import network_files_ref as O  # noqa: E402
from pixie_b200 import network_files as NF  # noqa: E402

DEV = "cuda:0"
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "network_files_golden.npz"))
CASES = G.metric_cases()
pytestmark = pytest.mark.gpu


def _run(c, mask=True, offset=0):
    """The kernel on a case; offset > 0 moves every input off 16 B alignment (the scalar path)."""
    def dev(a):
        a = torch.from_numpy(np.ascontiguousarray(a))
        if not offset:
            return a.to(DEV)
        buf = torch.empty(a.numel() + offset, dtype=a.dtype, device=DEV)
        v = buf[offset:].view(a.shape)
        v.copy_(a)
        return v
    mats = dev(np.stack(c["mats"]))
    masks = dev(np.stack(c["masks"])) if mask else None
    return NF.material_metrics(mats, masks, dev(c["logits"]), dev(c["cont"]), G.RANGES, G.BG)


def _torch_reference(c, gt):
    """masked_mean as the reference writes it, on the device, per sample and channel."""
    cont = torch.from_numpy(c["cont"]).to(DEV)
    mask = torch.from_numpy(np.stack(c["masks"])).to(DEV).unsqueeze(1)
    diff_sq = (cont - gt[:, :3]) ** 2
    return ((diff_sq * mask).sum((2, 3, 4)) / ((mask.sum((2, 3, 4)).clamp(min=1)) + 1e-8)).cpu().numpy()


def _ulp_log_bound(raw, lo, hi):
    """|d gt| allowed for a log10 channel: 2 ulp32 of log10(x + 1e-6), carried through 2 (x - lo) / (hi - lo) - 1, plus
    one rounding of the result."""
    with np.errstate(divide="ignore", invalid="ignore"):
        lg = np.log10(raw + np.float32(1e-6))
    lg = np.where(np.isfinite(lg), lg, 0).astype(np.float32)
    return 2 * np.spacing(np.abs(lg)) * 2 / (hi - lo) + 2 * np.spacing(np.float32(1))


@pytest.mark.parametrize("offset", [0, 1])
@pytest.mark.parametrize("name", list(CASES))
def test_kernel_against_oracle_and_reference(name, offset):
    c = CASES[name]
    gt, counts, sums = _run(c, offset=offset)
    gts, o_counts, o_sums = [], [], []
    for i, m in enumerate(c["mats"]):
        g = O.normalize_gt(m, G.RANGES)
        gts.append(g)
        (t, k), s = O.sample_counts_sums(g, c["masks"][i], c["logits"][i], c["cont"][i], G.BG)
        o_counts.append((t, k))
        o_sums.append(s)
    assert np.array_equal(counts, np.array(o_counts)) and np.array_equal(counts, GOLD[f"batch_{name}/counts"])
    g_dev = gt.cpu().numpy()
    worst = 0.0
    for i, g in enumerate(gts):
        raw = c["mats"][i]
        for ch, (lo, hi) in ((0, ("density_min", "density_max")), (1, ("E_min", "E_max"))):
            bound = _ulp_log_bound(raw[..., ch], np.float32(G.RANGES[lo]), np.float32(G.RANGES[hi]))
            err = np.abs(g_dev[i, ch] - g[ch])
            assert np.all(err <= bound), (ch, err.max())
            worst = max(worst, float((err / bound).max()))
        assert np.array_equal(g_dev[i, 2:], g[2:])                        # nu and id: same float32 ops, bit for bit
    print(f"[gt] {name}: worst |gt - numpy| / bound = {worst:.3f}")
    batch, samples = NF.batch_metrics(counts, sums)
    o_batch, o_samples = NF.batch_metrics(np.array(o_counts), np.array(o_sums))
    ref_b, ref_s = GOLD[f"batch_{name}/batch"], GOLD[f"batch_{name}/samples"]
    assert batch[0] == ref_b[0] and [s["seg_acc"] for s in samples] == list(ref_s[:, 0])
    keys = ["density_mse", "youngs_mse", "poisson_mse"]
    mine = np.array([[s[k] for k in keys] for s in samples], np.float32)
    orac = np.array([[s[k] for k in keys] for s in o_samples], np.float32)
    assert np.array_equal(np.isnan(mine), np.isnan(orac))
    ok = ~np.isnan(orac)
    ulps = np.abs(mine[ok].view(np.int32).astype(np.int64) - orac[ok].view(np.int32).astype(np.int64))
    assert ulps.max(initial=0) <= 2
    tref = _torch_reference(c, gt)
    assert np.array_equal(np.isnan(tref), np.isnan(mine))
    np.testing.assert_allclose(mine[ok], tref[ok], rtol=1e-6, atol=0)


def _check_sums(dev, oracle):
    """nu's squared errors and the mask sum come from identical float32 terms, so only the fp64 summation order differs;
    the density and E terms also carry the last-bit log10 differences of the gt."""
    np.testing.assert_allclose(dev[2:], oracle[2:], rtol=1e-13)
    np.testing.assert_allclose(dev[:2], oracle[:2], rtol=1e-6)


def test_no_mask_branch():
    c = CASES["d13_n3_edges"]
    _, counts, sums = _run(c, mask=False)
    for i, m in enumerate(c["mats"]):
        (t, k), s = O.sample_counts_sums(O.normalize_gt(m, G.RANGES), None, c["logits"][i], c["cont"][i], G.BG)
        assert (counts[i] == (t, k)).all()
        _check_sums(sums[i], s)


def test_repeat_is_bit_identical_and_paths_agree():
    rng = np.random.default_rng(3)
    for D, N in ((64, 4), (37, 2)):
        c = dict(mats=[G.raw_material(rng, D) for _ in range(N)], logits=rng.normal(0, 1, (N, 8, D, D, D)).astype(np.float32),
                 cont=rng.uniform(-1, 1, (N, 3, D, D, D)).astype(np.float32))
        c["masks"] = [(m[..., 3] != G.BG).astype(np.float32) for m in c["mats"]]
        a = _run(c)
        b = _run(c)
        assert torch.equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and np.array_equal(a[2].view(np.int64), b[2].view(np.int64))
        s = _run(c, offset=1)
        assert torch.equal(a[0], s[0]) and np.array_equal(a[1], s[1])
        np.testing.assert_allclose(a[2], s[2], rtol=1e-13)
        for i in range(N):
            (t, k), o = O.sample_counts_sums(O.normalize_gt(c["mats"][i], G.RANGES), c["masks"][i], c["logits"][i], c["cont"][i])
            _check_sums(a[2][i], o)


# ------------------------------------------------------------------------------------------------------------ end to end
def _labelled_scenes(root, C, n=3, D=64):
    rng = np.random.default_rng(99)
    ids = []
    for k in range(n):
        obj = f"scene{k}"
        mat = G.raw_material(rng, D)
        mat[:8] = 0.0
        mat[:8, ..., 3] = G.BG
        mask = (mat[..., 3] != G.BG).astype(np.float32)
        d = os.path.join(root, obj)
        os.makedirs(os.path.join(d, "sample_0"))
        np.save(os.path.join(d, "clip_features_features.npy"), (0.05 * rng.standard_normal((D, D, D, C))).astype(np.float16))
        np.save(os.path.join(d, "clip_features_mask.npy"), mask)
        np.save(os.path.join(d, "sample_0", "material_grid.npy"), mat)
        np.savez(os.path.join(d, "clip_features.npz"), min_bounds=np.array([-0.5] * 3), max_bounds=np.array([0.5] * 3),
                 grid_shape=np.array([D, D, D]))
        ids.append(obj)
    return ids


def test_inference_map_and_simulate_end_to_end(tmp_path):
    from pixie_b200 import gs_simulation, inference_combined as IC, map_pred_to_coords as MP, scene_files as SF
    from pixie_b200.inference import MaterialFieldPredictor
    from pixie_b200.material_transfer import extract_material_points
    from pixie_b200.synthetic import seeded_state_dict
    from pixie_b200.unet import _expected_keys
    C, D = 64, 64
    root = tmp_path / "render_outputs"
    ids = _labelled_scenes(str(root), C)
    stats = tmp_path / "stats"
    stats.mkdir()
    ranges_yaml = {"density_p1": G.RANGES["density_min"], "density_p99": G.RANGES["density_max"], "E_p1": G.RANGES["E_min"],
                   "E_p99": G.RANGES["E_max"], "nu_p1": G.RANGES["nu_min"], "nu_p99": G.RANGES["nu_max"]}
    (stats / "normalization_ranges.yaml").write_text(json.dumps(ranges_yaml))
    cfg = IC.UNET_CFG
    keys = lambda out: _expected_keys(C, cfg["cond_dim"], cfg["model_channels"], cfg["num_res_blocks"], cfg["channel_mult"], D, out)  # noqa: E731
    seg_sd, cont_sd = seeded_state_dict(keys(8), 0), seeded_state_dict(keys(3), 1)
    torch.save({"model_state_dict": seg_sd, "epoch": 5}, tmp_path / "seg.pth")
    torch.save(cont_sd, tmp_path / "cont.pth")
    out = tmp_path / "out"
    args = ["--render_outputs_dir", str(root), "--seg_checkpoint", str(tmp_path / "seg.pth"), "--cont_checkpoint", str(tmp_path / "cont.pth"),
            "--normalization_ranges", str(stats / "normalization_ranges.yaml"), "--output_dir", str(out), "--feature_channels", str(C),
            "--batch_size", "1", "--train_size", "0.0", "--precision", "fp16x3"]
    assert IC.main(args, device=DEV) == 0
    report = json.loads((out / "metrics.json").read_text())
    assert json.loads((out / "evaluated_obj_ids.json").read_text()) == sorted(ids)

    # oracle: the same networks one scene at a time, the fp64 counts / sums and the reference's float32 arithmetic
    pred = MaterialFieldPredictor(C, grid_size=D, device=DEV, max_batch=1, precision="fp16x3", **cfg).load_state_dicts(seg_sd, cont_sd, strict=False)
    for obj in ids:
        d = root / obj
        feat = torch.from_numpy(np.load(d / "clip_features_features.npy")).to(DEV)[None]
        seg, cont = pred.predict(feat)
        packed = pred.pack(seg, cont).cpu().numpy()[0]
        mat, mask = np.load(d / "sample_0" / "material_grid.npy"), np.load(d / "clip_features_mask.npy")
        g = O.normalize_gt(mat, G.RANGES)
        cs = O.sample_counts_sums(g, mask, seg[0].cpu().numpy(), cont[0].cpu().numpy())
        _, (s,) = NF.batch_metrics(np.array([cs[0]]), np.array([cs[1]]))
        got = report["per_object_metrics"][obj]
        # two forwards of the same networks agree to the last bits only (the kernel tests above are exact), so the
        # command line is compared with a second run at the networks' tolerance
        assert abs(got["seg_acc"] - s["seg_acc"]) <= 1e-4
        for k in ("density_mse", "youngs_mse", "poisson_mse"):
            assert abs(got[k] - s[k]) <= 1e-5 * abs(s[k])
        o = out / obj
        saved = np.load(o / "sample_0_pred.npy")
        assert saved.shape == packed.shape and saved.dtype == np.float32
        np.testing.assert_allclose(saved[:3], packed[:3], rtol=0, atol=1e-5)
        assert np.mean(saved[3:].argmax(0) == packed[3:].argmax(0)) > 0.999 and set(np.unique(saved[3:])) <= {0.0, 1.0}
        assert np.array_equal(np.load(o / "sample_0_mask.npy"), mask)
        gd = np.load(o / "sample_0_gt.npy")
        assert gd.shape == (4, D, D, D) and np.array_equal(gd[2:], g[2:])
        for ch, (lo, hi) in ((0, ("density_min", "density_max")), (1, ("E_min", "E_max"))):
            assert np.all(np.abs(gd[ch] - g[ch]) <= _ulp_log_bound(mat[..., ch], np.float32(G.RANGES[lo]), np.float32(G.RANGES[hi])))
        info = np.load(o / "sample_0_info.npy", allow_pickle=True).item()
        assert info == {"obj_id": obj, "sample_id": "0", "data_path": f"{root}/{obj}/sample_0/material_grid.npy",
                        "feature_path": f"{root}/{obj}/clip_features_features.npy", "mask_path": f"{root}/{obj}/clip_features_mask.npy"}

    # map_pred_to_coords on the first scene's prediction, read back as gs_simulation reads it
    obj = ids[0]
    ply = tmp_path / "mapped_preds.ply"
    assert MP.main(["--pred_path", str(out / obj / "sample_0_pred.npy"), "--mask_path", str(root / obj / "clip_features_mask.npy"),
                    "--grid_feature_path", str(root / obj / "clip_features.npz"), "--output_path", str(ply),
                    "--normalization_ranges", str(stats / "normalization_ranges.yaml")], device=DEV) == 0
    cloud = SF.load_point_cloud(str(ply), DEV)
    want = extract_material_points(torch.from_numpy(np.load(out / obj / "sample_0_pred.npy")).to(DEV),
                                   torch.from_numpy(np.load(root / obj / "clip_features_mask.npy")).to(DEV), [-0.5] * 3, [0.5] * 3, G.RANGES)
    assert set(cloud) == set(want)
    for k in want:
        assert torch.equal(cloud[k], want[k]), k

    # gs_simulation runs one scene from that file
    from test_scene_files import BASE_CONFIG, _model_dir
    model, _, _ = _model_dir(tmp_path, np.random.default_rng(11))
    (tmp_path / "config.json").write_text(json.dumps(dict(BASE_CONFIG, frame_num=2)))
    assert gs_simulation.main(["--model_path", model, "--config", str(tmp_path / "config.json"), "--point_cloud_path", str(ply)], device=DEV) == 0
