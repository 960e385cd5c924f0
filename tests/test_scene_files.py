"""Scenes from files: the PLY reader, the device checkpoint decoder (pixie_gaussian_checkpoint_decode), the physics-config
and rotation decoders, the material-cloud / E-field loaders, Scene.from_files and the gs_simulation command line.

CPU tests hold the oracle and the host-side loaders to tests/golden/scene_files_golden.npz (the reference's own code,
make_scene_files_golden.py). GPU tests hold the decoder to the reference's torch expressions run on the same device
(oracle/gaussian_model_ref.torch_reference) and to the fp64 oracle, and the command line to the scene driver."""
import json
import os
import re
import struct
import zlib

import numpy as np
import pytest
import torch

from oracle import gaussian_model_ref as GM
from pixie_b200 import gs_simulation as CLI
from pixie_b200 import scene_files as SF

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = np.load(os.path.join(HERE, "golden", "scene_files_golden.npz"))
CKPTS = ("ckpt_k1", "ckpt_k4", "ckpt_k9", "ckpt_k16", "ckpt_perm", "ckpt_edge")
PLY_TYPE = {"f4": "float", "f8": "double", "i4": "int", "u1": "uchar"}


def ply_bytes(arr: np.ndarray, fmt="binary_little_endian") -> bytes:
    head = ["ply", f"format {fmt} 1.0", "comment a test file", "obj_info none", f"element vertex {len(arr)}"] + \
           [f"property {PLY_TYPE[arr.dtype[n].str[1:]]} {n}" for n in arr.dtype.names] + ["end_header"]
    return ("\n".join(head) + "\n").encode() + arr.tobytes()


def checkpoint(rng, n, K, extra=(), opacity=None):
    """A checkpoint vertex table in save_ply's property order (+ `extra` properties at the end)."""
    names = ["x", "y", "z", "nx", "ny", "nz", "f_dc_0", "f_dc_1", "f_dc_2"] + [f"f_rest_{i}" for i in range(3 * K - 3)] + \
            ["opacity", "scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3"]
    a = np.zeros(n, dtype=[(nm, "<f4") for nm in names] + list(extra))
    for nm in a.dtype.names:
        if nm.startswith("n"):
            continue
        a[nm] = rng.uniform(-6, -3, n) if nm.startswith("scale") else rng.normal(-2.0, 2.5, n) if nm == "opacity" else rng.normal(0, 1, n)
    if opacity is not None:
        a["opacity"] = opacity
    return a


def raw_columns(arr: np.ndarray, K: int):
    rest = sorted([n for n in arr.dtype.names if n.startswith("f_rest_")], key=lambda s: int(s.split("_")[-1]))
    col = lambda names: np.stack([arr[n] for n in names], axis=1).astype(np.float32)          # noqa: E731
    return {"xyz": col("xyz"), "f_dc": col(["f_dc_0", "f_dc_1", "f_dc_2"]),
            "f_rest": col(rest) if rest else np.zeros((len(arr), 0), np.float32), "opacity": arr["opacity"].astype(np.float32),
            "scale": col(["scale_0", "scale_1", "scale_2"]), "rot": col(["rot_0", "rot_1", "rot_2", "rot_3"])}


def f32_norm_ok(rot: np.ndarray) -> np.ndarray:
    """Rows whose quaternion's float32 squared norm neither overflows nor vanishes: elsewhere build_rotation's float32
    normalisation gives a different (or no) rotation than the fp64 oracle's."""
    with np.errstate(over="ignore", under="ignore"):
        n2 = (rot.astype(np.float32) ** 2).sum(axis=1, dtype=np.float32)
    return np.isfinite(n2) & (n2 >= np.finfo(np.float32).tiny)


def golden_file(tmp_path, name) -> str:
    p = tmp_path / f"{name}.ply"
    p.write_bytes(GOLD[f"{name}/file"].tobytes())
    return str(p)


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("name", CKPTS)
def test_oracle_matches_golden(tmp_path, name):
    K = int(GOLD[f"{name}/K"])
    raw = raw_columns(SF.read_ply(golden_file(tmp_path, name)).read(), K)
    o = GM.decode_f64(raw)
    np.testing.assert_array_equal(o["pos"].astype(np.float32), GOLD[f"{name}/pos"])
    np.testing.assert_array_equal(o["shs"].astype(np.float32), GOLD[f"{name}/shs"])
    g_op = GOLD[f"{name}/opacity"]
    np.testing.assert_allclose(o["opacity"], g_op, rtol=1e-6, atol=1e-7)
    for thr in (0.02, 0.05):
        np.testing.assert_array_equal(GM.keep_mask(g_op, thr), GOLD[f"{name}/mask_{thr}"])
    fin = np.isfinite(o["cov"]).all(1) & np.isfinite(GOLD[f"{name}/cov"]).all(1) & (o["s_max"] < 1e18) & f32_norm_ok(raw["rot"])
    tol = 1e-6 * o["s_max"][fin, None] ** 2
    assert np.all(np.abs(o["cov"][fin] - GOLD[f"{name}/cov"][fin]) <= tol + 1e-30)


def test_edge_rows_straddle_the_thresholds():
    m02, m05 = GOLD["ckpt_edge/mask_0.02"], GOLD["ckpt_edge/mask_0.05"]
    assert 0 < m02[:25].sum() < 25 and 0 < m05[25:50].sum() < 25


@pytest.mark.parametrize("name", CKPTS + ("cloud", "cloud_noconf", "efield"))
def test_reader_accepts_golden_files(tmp_path, name):
    el = SF.read_ply(golden_file(tmp_path, name))
    assert el.name == "vertex" and el.count > 0
    rows = el.read()
    if name.startswith("ckpt"):
        np.testing.assert_array_equal(np.stack([rows[c] for c in "xyz"], 1), GOLD[f"{name}/pos"])


def test_reader_rejects(tmp_path):
    a = checkpoint(np.random.default_rng(0), 4, 1)
    cases = {"ascii": ply_bytes(a, "ascii"), "big": ply_bytes(a, "binary_big_endian")}
    lst = ply_bytes(a).replace(b"property float nx\n", b"property list uchar int nx\n")
    cases["list"] = lst
    for name, blob in cases.items():
        p = tmp_path / f"{name}.ply"
        p.write_bytes(blob)
        with pytest.raises(ValueError):
            SF.read_ply(str(p))
    d = np.zeros(4, dtype=[("x", "<f8")] + [(n, a.dtype[n]) for n in a.dtype.names if n != "x"])
    p = tmp_path / "f64.ply"
    p.write_bytes(ply_bytes(d))
    with pytest.raises(ValueError, match="float32"):
        SF.decode_checkpoint_ply(str(p), sh_degree=0)
    p = tmp_path / "rest.ply"
    p.write_bytes(ply_bytes(checkpoint(np.random.default_rng(0), 4, 4)))
    with pytest.raises(AssertionError):
        SF.decode_checkpoint_ply(str(p), sh_degree=3)


def test_search_for_max_iteration(tmp_path):
    for it in (100, 7000, 30000):
        (tmp_path / "point_cloud" / f"iteration_{it}").mkdir(parents=True)
    assert SF.search_for_max_iteration(str(tmp_path / "point_cloud")) == int(GOLD["iters/max"]) == 30000
    assert SF.checkpoint_path(str(tmp_path)).endswith(os.path.join("iteration_30000", "point_cloud.ply"))
    (tmp_path / "point_cloud" / "notes.txt").write_text("x")
    with pytest.raises(ValueError):
        SF.search_for_max_iteration(str(tmp_path / "point_cloud"))


def test_decode_param_json_matches_reference(tmp_path):
    texts = json.loads(str(GOLD["configs/text"]))
    decoded = json.loads(str(GOLD["configs/decoded"]))
    assert sum(n.startswith("custom_") for n in texts) == 22
    for name, text in texts.items():
        p = tmp_path / name
        p.write_text(text)
        want = decoded[name]
        if "error" in want:
            with pytest.raises({"ValueError": ValueError, "TypeError": TypeError}[want["error"]], match=re.escape(want["message"])):
                SF.decode_param_json(str(p))
            continue
        got = SF.decode_param_json(str(p))
        assert json.dumps(list(got)) == json.dumps(want["result"]), name          # values and key order


def test_rotation_matrices_bit_identical():
    lists = json.loads(str(GOLD["rot/lists"]))
    assert len(lists) > 22
    for name, (deg, ax) in lists.items():
        ms = SF.generate_rotation_matrices(deg, ax, device="cpu")
        got = np.stack([m.numpy() for m in ms]) if ms else np.zeros((0, 3, 3), np.float32)
        assert got.dtype == np.float32
        np.testing.assert_array_equal(got.view(np.uint32), GOLD[f"rot/{name}"].view(np.uint32), err_msg=name)
    with pytest.raises(ValueError):
        SF.generate_rotation_matrices([10], [3], device="cpu")
    with pytest.raises(AssertionError):
        SF.generate_rotation_matrices([10, 20], [0], device="cpu")


@pytest.mark.parametrize("name", ("cloud", "cloud_noconf"))
def test_load_point_cloud(tmp_path, name):
    c = SF.load_point_cloud(golden_file(tmp_path, name), device="cpu")
    np.testing.assert_array_equal(c["pos"].numpy(), GOLD[f"{name}/pos"])
    for k in ("density", "E", "nu", "material_id", "part_labels", "conf"):
        np.testing.assert_array_equal(c[k].numpy(), GOLD[f"{name}/{k}"].astype(c[k].numpy().dtype), err_msg=k)
    assert c["material_id"].dtype == torch.int32 and c["part_labels"].dtype == torch.int32 and c["conf"].dtype == torch.float32


def test_e_field(tmp_path):
    d = tmp_path / "opt"
    d.mkdir()
    for ep in (3, 7):
        (d / f"E_field_epoch_{ep:02d}.ply").write_bytes(GOLD["efield/file"].tobytes())
    (d / "E_field_epoch_x.ply").write_text("not an epoch")
    assert SF.find_e_field_epoch(str(d)).endswith("E_field_epoch_07.ply")
    assert SF.find_e_field_epoch(str(d), 3).endswith("E_field_epoch_03.ply")
    np.testing.assert_array_equal(SF.load_e_field_from_ply(str(d / "E_field_epoch_07.ply"), "cpu").numpy(), GOLD["efield/E"])
    np.testing.assert_array_equal(SF.load_optimized_e_field(str(d), device="cpu").numpy(), (torch.from_numpy(GOLD["efield/E"]) * 1e7).numpy())
    with pytest.raises(FileNotFoundError):
        SF.find_e_field_epoch(str(tmp_path / "missing"))
    with pytest.raises(FileNotFoundError):
        SF.find_e_field_epoch(str(tmp_path))


def test_grid_metadata(tmp_path):
    from pixie_b200 import voxel_io
    p = tmp_path / "clip_features.npz"
    np.savez(p, min_bounds=np.array([-1.0, -2, -3]), max_bounds=np.array([1.0, 2, 3]), grid_shape=np.array([64, 64, 64]))
    lo, hi, shape = voxel_io.load_grid_metadata(str(p))
    assert lo.tolist() == [-1, -2, -3] and hi.tolist() == [1, 2, 3] and shape.tolist() == [64, 64, 64]


def _cli_dir(tmp_path, config):
    (tmp_path / "model" / "point_cloud" / "iteration_1").mkdir(parents=True, exist_ok=True)
    cfg = tmp_path / "config.json"
    cfg.write_text(json.dumps(config))
    return ["--model_path", str(tmp_path / "model"), "--config", str(cfg), "--point_cloud_path", str(tmp_path / "none.ply"),
            "--output_path", str(tmp_path / "out")]


def test_cli_rejects_before_device_work(tmp_path, monkeypatch):
    touched = []
    monkeypatch.setattr(SF, "decode_checkpoint_ply", lambda *a, **k: touched.append(1))
    base = _cli_dir(tmp_path, {})
    with pytest.raises(NotImplementedError, match="compile_video"):
        CLI.main(base + ["--render_img", "--compile_video"])
    with pytest.raises(NotImplementedError, match="debug"):
        CLI.main(base + ["--debug"])
    smooth = _cli_dir(tmp_path, {"particle_filling": {"smooth": True, "visualize": True}})
    with pytest.raises(NotImplementedError, match="smooth"):
        CLI.main(smooth + ["--render_img"])
    with pytest.raises(SystemExit):
        CLI.main(["--config", "x.json", "--point_cloud_path", "p.ply"])                  # --model_path is required
    assert not touched and not (tmp_path / "out").exists()


def _png_decode(path):
    """A minimal PNG reader (8-bit RGB, filter 0 rows) with the stdlib."""
    data = open(path, "rb").read()
    assert data[:8] == b"\x89PNG\r\n\x1a\n"
    pos, idat, w, h = 8, b"", None, None
    while pos < len(data):
        n, = struct.unpack(">I", data[pos:pos + 4])
        kind, body = data[pos + 4:pos + 8], data[pos + 8:pos + 8 + n]
        assert zlib.crc32(kind + body) & 0xFFFFFFFF == struct.unpack(">I", data[pos + 8 + n:pos + 12 + n])[0]
        if kind == b"IHDR":
            w, h, depth, ctype = struct.unpack(">IIBB", body[:10])
            assert depth == 8 and ctype == 2
        elif kind == b"IDAT":
            idat += body
        pos += 12 + n
    rows = np.frombuffer(zlib.decompress(idat), np.uint8).reshape(h, 1 + 3 * w)
    assert (rows[:, 0] == 0).all()
    return rows[:, 1:].reshape(h, w, 3)


def _special_image():
    vals = np.array([0, 0.5 / 255, 1.5 / 255, 2.5 / 255, 127.5 / 255, 254.5 / 255, 1, 1.2, -0.3, np.nan, np.inf, -np.inf, 1e8, -1e8,
                     2147483520 / 255, 2147483648 / 255], np.float32)
    rng = np.random.default_rng(3)
    img = rng.uniform(-0.2, 1.2, (7, 16, 3)).astype(np.float32)
    img[0, :, 0], img[1, :, 1], img[2, :, 2] = vals, vals[::-1], vals * 0.5
    return img


def test_png_writer_round_trip(tmp_path):
    img = _special_image()
    px = CLI.png_pixels(img)
    CLI.write_png(str(tmp_path / "a.png"), px)
    np.testing.assert_array_equal(_png_decode(str(tmp_path / "a.png")), px)
    assert px[0, :4, 0].tolist() == [0, 0, 2, 2] and px[0, 4, 0] == 128 and px[0, 9, 0] == 0


def test_png_pixels_match_cv2(tmp_path):
    cv2 = pytest.importorskip("cv2")
    img = _special_image()
    p = str(tmp_path / "cv.png")
    cv2.imwrite(p, 255 * cv2.cvtColor(img, cv2.COLOR_BGR2RGB))
    np.testing.assert_array_equal(cv2.cvtColor(cv2.imread(p), cv2.COLOR_BGR2RGB), CLI.png_pixels(img))
    CLI.write_png(str(tmp_path / "ours.png"), CLI.png_pixels(img))
    np.testing.assert_array_equal(cv2.imread(str(tmp_path / "ours.png")), cv2.imread(p))


# ------------------------------------------------------------------------------------------------ GPU: decoder
DEV = "cuda:0"


def _u32(t):
    return t.detach().cpu().contiguous().numpy().view(np.uint32)


def _same_bits(a, b):
    a, b = _u32(a), _u32(b)
    both_nan = np.isnan(a.view(np.float32)) & np.isnan(b.view(np.float32))
    np.testing.assert_array_equal(np.where(both_nan, 0, a), np.where(both_nan, 0, b))


def _check_decode(path, arr, K, threshold=None):
    raw = raw_columns(arr, K)
    d = SF.decode_checkpoint_ply(path, int(round(K ** 0.5)) - 1, threshold, DEV)
    ref = GM.torch_reference(raw, DEV)
    keep = torch.ones(len(arr), dtype=torch.bool, device=DEV) if threshold is None else ref["opacity"][:, 0] > threshold
    assert d["pos"].shape[0] == int(keep.sum())
    for k in ("pos", "shs", "opacity"):
        assert d[k].shape == ref[k][keep].shape
        _same_bits(d[k], ref[k][keep])
    got, want, L = d["cov"].cpu().numpy(), ref["cov"][keep].cpu().numpy(), ref["L"][keep].cpu().double().numpy()
    np.testing.assert_array_equal(np.isnan(got), np.isnan(want))
    np.testing.assert_array_equal(np.isinf(got), np.isinf(want))
    fin = np.isfinite(want)
    absL = np.abs(L)
    bound = np.einsum("nik,njk->nij", absL, absL)[:, [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]]
    with np.errstate(invalid="ignore", over="ignore"):
        err = np.abs(got.astype(np.float64) - want)
        assert np.all(err[fin] <= 3 * np.spacing(bound.astype(np.float32))[fin] + 1e-45)
    o = GM.decode_f64({k: v[keep.cpu().numpy()] for k, v in raw.items()})
    rows = np.isfinite(o["cov"]).all(1) & (o["s_max"] < 1e18) & np.isfinite(got).all(1) & f32_norm_ok(raw["rot"][keep.cpu().numpy()])
    # 2e-6 s_max^2: the reference's float32 build_rotation alone (several roundings per entry of R, which the kernel
    # reproduces bit for bit) already reaches 0.9e-6 s_max^2 from the fp64 value on random quaternions
    assert np.all(np.abs(got[rows] - o["cov"][rows]) <= 2e-6 * o["s_max"][rows, None] ** 2 + 1e-37)
    return d


@pytest.mark.gpu
@pytest.mark.parametrize("name", CKPTS)
@pytest.mark.parametrize("threshold", (None, 0.02, 0.05))
def test_decoder_golden_files(tmp_path, name, threshold):
    path = golden_file(tmp_path, name)
    K = int(GOLD[f"{name}/K"])
    _check_decode(path, SF.read_ply(path).read(), K, threshold)


@pytest.mark.gpu
@pytest.mark.parametrize("K", (1, 4, 9, 16))
@pytest.mark.parametrize("n", (1, 127, 128, 129, 3001))
def test_decoder_ragged(tmp_path, K, n):
    rng = np.random.default_rng(K * 10000 + n)
    a = checkpoint(rng, n, K, extra=[("extra", "<f4")] if n % 2 else ())           # odd n: a 1-word longer, unaligned row
    p = tmp_path / "c.ply"
    p.write_bytes(ply_bytes(a))
    _check_decode(str(p), a, K)
    _check_decode(str(p), a, K, 0.1)


@pytest.mark.gpu
def test_decoder_threshold_ulps(tmp_path):
    """Opacities in a band of float32 ulps around float32(0.02): rows with sigmoid == threshold are dropped, the others
    are kept or dropped exactly as torch's mask says, in file order."""
    x0 = np.float32(np.log(0.02 / 0.98))
    logits = (x0 + np.arange(-300, 300, dtype=np.float32) * np.spacing(x0)).astype(np.float32)
    a = checkpoint(np.random.default_rng(1), len(logits), 16, opacity=logits)
    p = tmp_path / "t.ply"
    p.write_bytes(ply_bytes(a))
    op = torch.sigmoid(torch.tensor(logits, device=DEV))
    thr = np.float32(0.02)
    assert bool((op == float(thr)).any()) or bool((op < float(thr)).any() and (op > float(thr)).any())
    d = _check_decode(str(p), a, 16, 0.02)
    assert d["pos"].shape[0] == int((op > 0.02).sum())


@pytest.mark.gpu
def test_decoder_empty_and_none_kept(tmp_path):
    a = checkpoint(np.random.default_rng(2), 300, 4)
    p = tmp_path / "c.ply"
    p.write_bytes(ply_bytes(a))
    d = SF.decode_checkpoint_ply(str(p), 1, 1.0, DEV)                               # sigmoid < 1 for these logits
    assert d["pos"].shape == (0, 3) and d["shs"].shape == (0, 4, 3) and d["cov"].shape == (0, 6)
    p.write_bytes(ply_bytes(a[:0]))
    for thr in (None, 0.02):
        d = SF.decode_checkpoint_ply(str(p), 1, thr, DEV)
        assert d["opacity"].shape == (0, 1)


@pytest.mark.gpu
def test_decoder_one_million(tmp_path):
    a = checkpoint(np.random.default_rng(5), 1_000_000, 16)
    p = tmp_path / "big.ply"
    p.write_bytes(ply_bytes(a))
    _check_decode(str(p), a, 16, 0.02)


@pytest.mark.gpu
def test_load_checkpoint_interface(tmp_path):
    a = checkpoint(np.random.default_rng(8), 500, 16)
    d = tmp_path / "model" / "point_cloud" / "iteration_30000"
    d.mkdir(parents=True)
    (d / "point_cloud.ply").write_bytes(ply_bytes(a))
    (tmp_path / "model" / "point_cloud" / "iteration_7000").mkdir()
    g = SF.load_checkpoint(str(tmp_path / "model"))
    assert g.active_sh_degree == g.max_sh_degree == 3 and not hasattr(g, "get_scaling")
    ref = GM.torch_reference(raw_columns(a, 16), DEV)
    _same_bits(g.get_xyz, ref["pos"])
    _same_bits(g.get_features, ref["shs"])
    _same_bits(g.get_opacity, ref["opacity"])
    p_all = SF.load_params_from_gs(g)
    p_thr = SF.load_params_from_gs(g, 0.05)
    fused = SF.load_gaussians(str(tmp_path / "model"), 0.05)
    mask = ref["opacity"][:, 0] > 0.05
    assert p_all["cov3D_precomp"] is g.get_covariance()
    for k in ("pos", "shs", "opacity", "cov3D_precomp", "screen_points"):
        _same_bits(p_thr[k], fused[k])
    _same_bits(fused["pos"], ref["pos"][mask])


# ------------------------------------------------------------------------------------------------ GPU: end to end
CAMERAS = [{"id": 0, "img_name": "c0", "width": 160, "height": 120, "position": [0.0, 0.0, 0.0], "rotation": np.eye(3).tolist(),
            "fx": 140.0, "fy": 140.0}]
BASE_CONFIG = {"material": "jelly", "n_grid": 32, "grid_lim": 2.0, "g": [0.0, 0.0, -9.8], "density": 1000.0, "E": 1e5, "nu": 0.3,
               "boundary_conditions": [{"type": "bounding_box"}], "substep_dt": 1e-4, "frame_dt": 2e-3, "frame_num": 3,
               "nn_distance_threshold": 0.2, "opacity_threshold": 0.02, "default_camera_index": -1, "init_azimuthm": 30.0,
               "init_elevation": 10.0, "init_radius": 2.0, "move_camera": True, "delta_a": 5.0, "delta_e": 1.0, "delta_r": 0.02}


def _model_dir(tmp_path, rng, n=3000):
    """A trained-model directory: a shell of Gaussians (radius 0.3) and a slab beside it, in save_ply's layout, and a
    cameras.json; plus a map_pred_to_ply-layout material cloud around them."""
    v = rng.standard_normal((n, 3))
    shell = np.array([0.0, -0.1, 0.0]) + 0.3 * v / np.linalg.norm(v, axis=1, keepdims=True)
    slab = np.stack([rng.uniform(-0.45, 0.45, n // 3), rng.uniform(0.3, 0.45, n // 3), rng.uniform(-0.45, 0.45, n // 3)], axis=1)
    pos = np.concatenate([shell, slab]).astype(np.float32)
    a = checkpoint(rng, len(pos), 16, opacity=rng.normal(0.5, 2.0, len(pos)).astype(np.float32))
    for i, c in enumerate("xyz"):
        a[c] = pos[:, i]
    for j in range(3):
        a[f"scale_{j}"] = np.log(rng.uniform(0.01, 0.02, len(pos)))
    a["f_dc_0"] *= 0.4
    d = tmp_path / "model"
    (d / "point_cloud" / "iteration_30000").mkdir(parents=True)
    (d / "point_cloud" / "iteration_30000" / "point_cloud.ply").write_bytes(ply_bytes(a))
    (d / "cameras.json").write_text(json.dumps(CAMERAS))
    g = np.stack(np.meshgrid(*[np.linspace(-0.5, 0.5, 12)] * 3, indexing="ij"), -1).reshape(-1, 3).astype(np.float32)
    cloud = np.zeros(len(g), dtype=[("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("part_label", "<i4"), ("density", "<f4"), ("E", "<f4"),
                                     ("nu", "<f4"), ("material_id", "<i4"), ("conf", "<f4")])
    cloud["x"], cloud["y"], cloud["z"] = g.T
    cloud["material_id"] = cloud["part_label"] = np.where(g[:, 2] < -0.3, 6, 0)
    cloud["density"], cloud["E"], cloud["nu"], cloud["conf"] = 1000.0, rng.uniform(5e4, 2e5, len(g)), 0.3, 1.0
    (tmp_path / "mapped_preds.ply").write_bytes(ply_bytes(cloud))
    return str(d), str(tmp_path / "mapped_preds.ply"), a


def _run_cli_and_driver(tmp_path, config, extra=()):
    from pixie_b200 import scene_driver as SD
    model, cloud_path, a = _model_dir(tmp_path, np.random.default_rng(11))
    cfg = tmp_path / "config.json"
    cfg.write_text(json.dumps(config))
    out = tmp_path / "out"
    assert CLI.main(["--model_path", model, "--config", str(cfg), "--point_cloud_path", cloud_path, "--output_path", str(out),
                     "--render_img", "--save_ply", *extra]) == 0
    sc = SD.Scene.from_files("model", model, str(cfg), save_ply=True)
    images = {}
    ref_ply = tmp_path / "ref_ply"
    rec = SD.SceneBatchDriver.physics_only(DEV).run_physics_simulation(
        sc, SF.load_point_cloud(cloud_path), on_image=lambda f, im: images.__setitem__(f, im.permute(1, 2, 0).cpu().numpy()),
        ply_dir=str(ref_ply))
    n_frames = config["frame_num"]
    assert sorted(os.listdir(out / "frames")) == [f"{f:05d}.png" for f in range(n_frames)]
    assert sorted(os.listdir(out / "ply_files")) == [f"frame_{f:05d}.ply" for f in range(n_frames)]
    # frame 0 precedes every substep, so both runs must write the same bytes; later frames carry the last-bit differences
    # of the substeps' float atomics between two rollouts, so they are compared by value
    assert (out / "ply_files" / "frame_00000.ply").read_bytes() == (ref_ply / "frame_00000.ply").read_bytes()
    np.testing.assert_array_equal(_png_decode(str(out / "frames" / "00000.png")), CLI.png_pixels(images[0]))
    for f in range(1, n_frames):
        got, want = (SF.read_ply(str(d / f"frame_{f:05d}.ply")) for d in (out / "ply_files", ref_ply))
        assert got.dtype == want.dtype and got.count == want.count
        g, w = got.read(), want.read()
        for name in g.dtype.names:
            if name in "xyz":
                np.testing.assert_allclose(g[name], w[name], rtol=0, atol=1e-4)
            elif not name.startswith(("scale_", "rot_")):
                np.testing.assert_array_equal(g[name], w[name])
        px, ref_px = _png_decode(str(out / "frames" / f"{f:05d}.png")).astype(int), CLI.png_pixels(images[f]).astype(int)
        assert np.mean(np.abs(px - ref_px) > 2) < 0.01
    assert _png_decode(str(out / "frames" / "00000.png")).max() > 0
    return sc, rec, a, out


@pytest.mark.gpu
def test_cli_end_to_end(tmp_path):
    sc, rec, a, out = _run_cli_and_driver(tmp_path, BASE_CONFIG)
    op = torch.sigmoid(torch.tensor(a["opacity"], device=DEV))
    keep = (op > 0.02).cpu().numpy()
    assert rec["n_gaussians"] == int(keep.sum()) < len(a)
    frame0 = SF.read_ply(str(out / "ply_files" / "frame_00000.ply")).read()
    xyz = np.stack([frame0[c] for c in "xyz"], 1)
    want = np.stack([a[c] for c in "xyz"], 1)[keep]
    np.testing.assert_allclose(xyz, want, rtol=0, atol=1e-6)


@pytest.mark.gpu
def test_cli_real_scene_style(tmp_path):
    config = dict(BASE_CONFIG, rotation_degree=[90.0, -30], rotation_axis=[2, 0], sim_area=[-0.25, 0.5, -0.5, 0.5, -0.5, 0.5],
                  opacity_threshold=0.05, z_shift_value=0.1)
    sc, rec, a, out = _run_cli_and_driver(tmp_path, config)
    assert rec["n_unselected"] > 0 and len(sc.rotation_matrices) == 2


@pytest.mark.gpu
def test_cli_filled_visualize(tmp_path):
    config = dict(BASE_CONFIG, particle_filling={"n_grid": 40, "density_threshold": 0.5, "search_threshold": 0.2, "visualize": True})
    sc, rec, a, out = _run_cli_and_driver(tmp_path, config)
    assert rec["n_filled"] > 0 and rec["n_particles"] == rec["n_gaussians"] + rec["n_filled"]
    assert SF.read_ply(str(out / "ply_files" / "frame_00000.ply")).count == rec["n_particles"]        # visualize exports every particle


@pytest.mark.gpu
def test_cli_e_field_replay(tmp_path):
    from pixie_b200 import scene_driver as SD
    model, cloud_path, a = _model_dir(tmp_path, np.random.default_rng(12))
    cfg = tmp_path / "config.json"
    cfg.write_text(json.dumps(BASE_CONFIG))
    sc = SD.Scene.from_files("m", model, str(cfg))
    n = sc.particles.shape[0]
    sc.e_field = torch.full((n,), 3e5, device=DEV)
    rec = SD.SceneBatchDriver.physics_only(DEV).run_physics_simulation(sc, SF.load_point_cloud(cloud_path), on_frame=lambda *x: None)
    assert rec["substeps"] == 60
    sc.e_field = torch.full((n + 1,), 3e5, device=DEV)
    with pytest.raises(ValueError, match="E field"):
        SD.SceneBatchDriver.physics_only(DEV).run_physics_simulation(sc, SF.load_point_cloud(cloud_path), on_frame=lambda *x: None)
