"""Dataset-view rendering (pixie_b200.gs_dataset_render): the host readers, cameras and argument merge on the CPU; the
scale/rotation checkpoint decode, the scale/rotation rasterizer against the reference's rasterizer binary and the fp64
oracle, and the command line end to end on the GPU."""
from __future__ import annotations

import json
import math
import os
import struct
import sys

import numpy as np
import pytest
import torch
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import gs_render_ref as R  # noqa: E402
from oracle import gs_scale_rot_ref as SR  # noqa: E402
from pixie_b200 import gs_dataset_render as D  # noqa: E402
from pixie_b200 import gs_render as GR  # noqa: E402
from pixie_b200 import scene_files as SF  # noqa: E402
from gs_views_fixtures import (reference_rasterizer, ref_render_scale_rot, seeded_gaussians, tree_snapshot,  # noqa: E402
                              write_blender, write_checkpoint, write_colmap)

GOLDEN = os.path.join(ROOT, "tests", "golden", "gs_views_golden.npz")


# ------------------------------------------------------------------------------------------------ host (CPU)
@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def rebuild(golden, prefix, dst):
    """The dataset tree stored under file/<prefix>/ in the golden file, written to dst."""
    for k in golden.files:
        if k.startswith(f"file/{prefix}/"):
            p = os.path.join(dst, k[len(f"file/{prefix}/"):])
            os.makedirs(os.path.dirname(p), exist_ok=True)
            with open(p, "wb") as f:
                f.write(golden[k].tobytes())
    return dst


def check_cams(golden, key, cams):
    names = json.loads(golden[key + "_names"].tobytes())
    assert [os.path.basename(c.image_path) for c in cams] == names
    if not cams:
        return
    np.testing.assert_allclose(np.array([c.R for c in cams]), golden[key + "_R"], rtol=0, atol=1e-12)
    np.testing.assert_allclose(np.array([c.T for c in cams]), golden[key + "_T"], rtol=0, atol=1e-12)
    np.testing.assert_allclose(np.array([[c.FovX, c.FovY] for c in cams]), golden[key + "_fov"], rtol=0, atol=1e-12)
    assert np.array_equal(np.array([[c.width, c.height] for c in cams]), golden[key + "_wh"])


def test_cfg_args_merge_matches_reference(golden, tmp_path):
    m = tmp_path / "model"
    m.mkdir()
    (m / "cfg_args").write_text(golden["args_cfg"].tobytes().decode())
    for argv, want in zip(json.loads(golden["args_cases"].tobytes()), json.loads(golden["args_merged"].tobytes())):
        got = vars(D.get_combined_args(["-m", str(m)] + argv))
        got["model_path"] = "<model>"
        assert got == want, argv


def test_cfg_args_rejections(tmp_path):
    m = tmp_path / "model"
    m.mkdir()
    with pytest.raises(FileNotFoundError):                 # as the reference's get_combined_args, which only catches TypeError
        D.get_combined_args(["-m", str(m), "-s", "/x"])
    for bad in ("__import__('os').system('true')", "Namespace(a=open('x'))", "dict(a=1)", "Namespace(1)", "Namespace(**{'a': 1})",
                "Namespace(a=1); x", "Namespace(a=[f for f in ()])"):
        (m / "cfg_args").write_text(bad)
        with pytest.raises(ValueError):
            D.get_combined_args(["-m", str(m)])


def test_rejections_before_any_device_call(tmp_path, monkeypatch):
    def boom(*a, **k):
        raise AssertionError("device work started")
    monkeypatch.setattr(SF, "decode_checkpoint_ply_scale_rot", boom)
    monkeypatch.setattr(GR, "rasterize_scale_rot", boom)
    m = tmp_path / "model"
    (m / "point_cloud" / "iteration_100").mkdir(parents=True)
    for flag in ("--convert_SHs_python", "--compute_cov3D_python", "--debug"):
        with pytest.raises(ValueError, match="not supported"):
            D.main(["-m", str(m), "-s", str(tmp_path), flag])
    (m / "cfg_args").write_text("Namespace(source_path='" + str(tmp_path / "nothing") + "')")
    with pytest.raises(ValueError, match="scene type"):
        D.main(["-m", str(m)])
    # a view loadCam cannot take is found before the checkpoint is decoded, and nothing is written
    src = str(tmp_path / "src")
    write_blender(src, np.random.default_rng(0), 2, 0, 8, 8)
    Image.fromarray(np.zeros((4, 8, 4), np.uint8), "RGBA").save(os.path.join(src, "train", "r_1.png"))
    (m / "cfg_args").write_text(f"Namespace(source_path={src!r})")
    with pytest.raises(ValueError, match="4-pixel-high"):
        D.main(["-m", str(m), "--quiet"])
    assert not (m / "train").exists()


@pytest.mark.parametrize("white", [False, True])
@pytest.mark.parametrize("evaluate", [False, True])
def test_blender_cameras_match_reference(golden, tmp_path, white, evaluate):
    """Frames with and without ".png", partial alpha with values where 255 times the composite lands just below an
    integer; R, T, FovX, FovY to 1e-12 and the composited pixels equal."""
    src = rebuild(golden, "blender", str(tmp_path / "src"))
    before = tree_snapshot(src)
    tr, te = D.readNerfSyntheticInfo(src, white, evaluate)
    key = f"blender_{int(white)}_{int(evaluate)}"
    check_cams(golden, key + "_train", tr)
    check_cams(golden, key + "_test", te)
    np.testing.assert_array_equal(np.stack([np.array(c.image) for c in tr + te]), golden[key + "_images"])
    assert tree_snapshot(src) == before and not os.path.exists(os.path.join(src, "points3d.ply"))


def test_trunc_differs_from_rounding_somewhere(golden):
    """The composite keeps trunc(255 c) (the reference's int8 cast), which is not round(255 c) on the golden frames."""
    rgba = np.array([[[255, 255, 255, 128], [10, 200, 3, 77]]], np.uint8)
    out = D._composite_trunc(rgba, True)
    norm = rgba / 255.0
    arr = norm[:, :, :3] * norm[:, :, 3:4] + (1 - norm[:, :, 3:4])
    assert (out != np.round(arr * 255.0).astype(np.uint8)).any()


@pytest.mark.parametrize("case", ["pinhole_bin", "simple_bin", "pinhole_txt"])
@pytest.mark.parametrize("evaluate", [False, True])
def test_colmap_cameras_match_reference(golden, tmp_path, case, evaluate):
    """PINHOLE and SIMPLE_PINHOLE binary models, a PINHOLE text model, unsorted image names, the llffhold split."""
    src = rebuild(golden, case, str(tmp_path / "src"))
    before = tree_snapshot(src)
    tr, te = D.readColmapSceneInfo(src, None, evaluate)
    check_cams(golden, f"colmap_{case}_{int(evaluate)}_train", tr)
    check_cams(golden, f"colmap_{case}_{int(evaluate)}_test", te)
    assert tree_snapshot(src) == before and not os.path.exists(os.path.join(src, "sparse", "0", "points3D.ply"))


def test_colmap_text_reader_takes_pinhole_only(golden, tmp_path):
    """The reference's text camera reader asserts PINHOLE; a SIMPLE_PINHOLE text model is refused likewise."""
    src = rebuild(golden, "pinhole_txt", str(tmp_path / "src"))
    path = os.path.join(src, "sparse", "0", "cameras.txt")
    lines = open(path).read().splitlines()
    e = lines[1].split()
    lines[1] = " ".join([e[0], "SIMPLE_PINHOLE"] + e[2:5] + e[6:])
    open(path, "w").write("\n".join(lines) + "\n")
    with pytest.raises(ValueError, match="PINHOLE"):
        D.readColmapSceneInfo(src, None, False)


def test_colmap_rejects_distorted_models(tmp_path):
    rng = np.random.default_rng(0)
    src = str(tmp_path / "src")
    write_colmap(src, rng, ["a.png"], [(8, 6)])
    with open(os.path.join(src, "sparse", "0", "cameras.bin"), "wb") as f:
        f.write(struct.pack("<Q", 1) + struct.pack("<iiQQ", 1, 2, 8, 6) + struct.pack("<dddd", 5, 4, 3, 0.1))
    with pytest.raises(ValueError, match="SIMPLE_RADIAL"):
        D.readColmapSceneInfo(src, None, False)


def test_load_cam_matches_reference(golden):
    """Resolution -1 at widths 1600, 1601 and 3203; 1, 2, 4, 8; explicit widths; odd sizes. The gt image equals the
    reference's original_image and the camera its float32 matrices."""
    for k, (W, H, res) in enumerate(golden["loadcam_cases"]):
        info = D.CameraInfo(k, golden[f"loadcam_{k}_R"], golden[f"loadcam_{k}_T"], 0.5, 0.6, Image.fromarray(golden[f"loadcam_{k}_in"]),
                            "x.png", "x", int(W), int(H))
        cam, gt = D.loadCam(int(res), info)
        want = golden[f"loadcam_{k}_gt"]
        assert gt.shape == (want.shape[1], want.shape[2], 3), k
        np.testing.assert_array_equal((torch.from_numpy(gt).permute(2, 0, 1) / 255.0).numpy(), want)
        np.testing.assert_allclose(cam.world_view_transform.numpy(), golden[f"loadcam_{k}_world_view"], rtol=2e-7, atol=1e-7)
        np.testing.assert_allclose(cam.full_proj_transform.numpy(), golden[f"loadcam_{k}_full_proj"], rtol=2e-7, atol=1e-7)
        np.testing.assert_allclose(cam.camera_center.numpy(), golden[f"loadcam_{k}_center"], rtol=2e-7, atol=1e-6)


def test_load_cam_drops_alpha_and_rejects_height_4():
    rng = np.random.default_rng(5)
    rgba = rng.integers(0, 256, (7, 9, 4), dtype=np.uint8)
    info = D.CameraInfo(0, np.eye(3), np.array([0.0, 0.0, 3.0]), 0.5, 0.6, Image.fromarray(rgba, "RGBA"), "x.png", "x", 9, 7)
    cam, gt = D.loadCam(1, info)
    np.testing.assert_array_equal(gt, rgba[:, :, :3])
    assert (cam.image_width, cam.image_height) == (9, 7)
    for res in (2, 1):           # 9 x 7 at resolution 2 is 4 x 4 (round(4.5), round(3.5))
        img = info.image if res == 2 else Image.fromarray(rgba[:4], "RGBA")
        with pytest.raises(ValueError, match="4-pixel-high"):
            D.check_views([D.CameraInfo(0, np.eye(3), np.zeros(3), 0.5, 0.6, img, "y.png", "y", 9, 7)], res)


def test_png_bytes_match_save_image(golden, tmp_path):
    """save_image's files: the ground truth (pixels equal the decoded image) and an unclamped float render."""
    info = D.CameraInfo(0, np.eye(3), np.zeros(3), 0.5, 0.6, Image.fromarray(golden["png_gt_in"]), "x.png", "x", 33, 17)
    _, u8 = D.loadCam(2, info)                       # the golden file is save_image of this view's original_image
    q = D.quantize(torch.from_numpy(u8).permute(2, 0, 1) / 255.0).numpy()
    np.testing.assert_array_equal(q, u8)
    D.save_png(q, str(tmp_path / "gt.png"))
    assert (tmp_path / "gt.png").read_bytes() == golden["png_gt"].tobytes()
    D.save_png(D.quantize(torch.from_numpy(golden["png_render_in"])).numpy(), str(tmp_path / "r.png"))
    assert (tmp_path / "r.png").read_bytes() == golden["png_render"].tobytes()


def test_empty_splits_create_directories(tmp_path, monkeypatch):
    src, m = str(tmp_path / "src"), tmp_path / "model"
    write_blender(src, np.random.default_rng(0), 0, 0, 8, 8)
    (m / "point_cloud" / "iteration_30000").mkdir(parents=True)
    (m / "point_cloud" / "iteration_500").mkdir(parents=True)
    (m / "cfg_args").write_text(f"Namespace(source_path={src!r})")
    monkeypatch.setattr(SF, "decode_checkpoint_ply_scale_rot", lambda *a, **k: {})
    before = tree_snapshot(src)
    out = D.render_sets(D.get_combined_args(["-m", str(m), "--quiet"]))
    assert out == {"train": 0, "test": 0}
    for split in ("train", "test"):
        for kind in ("renders", "gt"):
            d = m / split / "ours_30000" / kind
            assert d.is_dir() and not any(d.iterdir())
    assert tree_snapshot(src) == before


def test_oracle_cov_from_scale_rot_closed_form():
    q = np.array([[1.0, 0.0, 0.0, 0.0], [math.cos(0.3), 0.0, 0.0, math.sin(0.3)]])
    s = np.array([[0.1, 0.2, 0.3], [0.5, 0.1, 0.2]])
    cov = SR.cov3d_from_scale_rot(s, q)
    np.testing.assert_allclose(cov[0], [0.01, 0, 0, 0.04, 0, 0.09], atol=1e-15)
    c, si = math.cos(0.6), math.sin(0.6)                 # rotation by 0.6 about z
    Q = np.array([[c, -si, 0], [si, c, 0], [0, 0, 1]])
    S = Q @ np.diag([0.25, 0.01, 0.04]) @ Q.T
    np.testing.assert_allclose(cov[1], [S[0, 0], S[0, 1], S[0, 2], S[1, 1], S[1, 2], S[2, 2]], atol=1e-15)


# ------------------------------------------------------------------------------------------------ device (GPU)
def _ref_module():
    mod = reference_rasterizer()
    if mod is None:
        pytest.skip("the reference rasterizer binary was not built (oracle/build_gs_rasterizer_ref.py)")
    return mod


def _ceil_args(pos, scales, rots, cam):
    from test_gs_render import _cam_dict
    def f(idx):
        idx = idx.numpy()
        cov = SR.cov3d_from_scale_rot(scales[idx].cpu().numpy(), rots[idx].cpu().numpy())
        pre = R.preprocess(pos[idx].cpu().numpy(), cov, _cam_dict(cam))
        return np.array([p["r_arg"] if p is not None else 0.0 for p in pre])
    return f


@pytest.mark.gpu
def test_decode_scale_rot_matches_torch(built_lib, cuda_dev, tmp_path):
    rng = np.random.default_rng(1)
    for K in (1, 4, 16):
        model = str(tmp_path / f"m{K}")
        a = write_checkpoint(model, rng, 3001, K)
        a["rot_0"][:3] = 0.0; a["rot_1"][:3] = 0.0; a["rot_2"][:3] = 0.0; a["rot_3"][:3] = 0.0   # zero norm: clamp at 1e-12
        a["rot_1"][3] = 1e-30
        ply = SF.checkpoint_path(model)
        with open(ply, "rb") as f:
            head = f.read().split(b"end_header\n")[0] + b"end_header\n"
        with open(ply, "wb") as f:
            f.write(head + a.tobytes())
        d = SF.decode_checkpoint_ply_scale_rot(ply, int(round(K ** 0.5)) - 1, cuda_dev)
        col = lambda *ns: torch.from_numpy(np.stack([a[n] for n in ns], 1).astype(np.float32)).to(cuda_dev)
        assert torch.equal(d["pos"], col("x", "y", "z"))
        assert torch.equal(d["opacity"], torch.sigmoid(col("opacity")))
        assert torch.equal(d["scales"], torch.exp(col("scale_0", "scale_1", "scale_2")))
        r = col("rot_0", "rot_1", "rot_2", "rot_3")
        # the decode's arithmetic, one torch op (one rounding) per operation: the squares summed in index order
        sq = r * r
        norm = torch.sqrt(((sq[:, 0] + sq[:, 1]) + sq[:, 2]) + sq[:, 3]).clamp_min(1e-12)
        assert torch.equal(d["rotations"], r / norm[:, None])
        # torch's norm reduction spreads the four squares over threads and adds them in another order, so its norm may
        # differ in the last bit, and the quotient then by up to 2 ulp
        want = torch.nn.functional.normalize(r)
        ulp = (d["rotations"].view(torch.int32).long() - want.view(torch.int32).long()).abs()
        assert int(ulp.max()) <= 2, int(ulp.max())
        old = SF.decode_checkpoint_ply(ply, int(round(K ** 0.5)) - 1, None, cuda_dev)
        assert torch.equal(old["shs"], d["shs"]) and torch.equal(old["opacity"], d["opacity"])


@pytest.mark.gpu
@pytest.mark.parametrize("n", [2000, 200000])
@pytest.mark.parametrize("wh", [(800, 800), (801, 577)])
def test_scale_rot_matches_reference_binary(built_lib, cuda_dev, n, wh):
    from test_gs_render import compare, look_at_camera
    mod = _ref_module()
    W, H = wh
    cam = look_at_camera(W, H)
    pos, sc, rot, op, shs = seeded_gaussians(n, seed=n + W, dev=cuda_dev)
    for deg in range(4):
        for bg in ([0.0, 0.0, 0.0], [1.0, 1.0, 1.0]):
            img, radii = GR.rasterize_scale_rot(pos, sc, rot, op, cam, bg, shs, deg)
            img_r, radii_r = ref_render_scale_rot(mod, pos, sc, rot, op, cam, bg, shs, deg)
            compare(img, radii, img_r, radii_r, _ceil_args(pos, sc, rot, cam), f"scale/rot n={n} {W}x{H} deg={deg} bg={bg[0]}")
    assert int((radii == 0).sum()) > 0 and int((radii > 0).sum()) > n // 2


@pytest.mark.gpu
def test_scale_rot_matches_oracle_small(built_lib, cuda_dev):
    from test_gs_render import _cam_dict, compare, look_at_camera
    cam = look_at_camera(53, 37, radius=3.0)
    pos, sc, rot, op, shs = seeded_gaussians(300, seed=7, dev=cuda_dev)
    img, radii = GR.rasterize_scale_rot(pos, sc, rot, op, cam, [0.3, 0.2, 0.1], shs, 3)
    cd = _cam_dict(cam)
    cov = SR.cov3d_from_scale_rot(sc.cpu().numpy(), rot.cpu().numpy())
    col = R.eval_sh_colors(3, shs.cpu().numpy(), pos.cpu().numpy(), cd["campos"])
    img_o, radii_o, _ = R.rasterize(pos.cpu().numpy(), cov, op.cpu().numpy(), col, cd, [0.3, 0.2, 0.1])
    compare(img, radii, torch.from_numpy(img_o).float().to(cuda_dev), torch.from_numpy(radii_o).to(cuda_dev),
            _ceil_args(pos, sc, rot, cam), "scale/rot oracle 53x37")


def _check_split(mod, model, split, it, infos, g, sh_degree, bg, resolution, cuda_dev):
    rdir, gdir = os.path.join(model, split, f"ours_{it}", "renders"), os.path.join(model, split, f"ours_{it}", "gt")
    assert sorted(os.listdir(rdir)) == sorted(os.listdir(gdir)) == [f"{i:05d}.png" for i in range(len(infos))]
    for i, info in enumerate(infos):
        cam, gt = D.loadCam(resolution, info)
        np.testing.assert_array_equal(np.array(Image.open(os.path.join(gdir, f"{i:05d}.png"))), gt)
        png = torch.from_numpy(np.array(Image.open(os.path.join(rdir, f"{i:05d}.png")))).to(cuda_dev)
        img_r, _ = ref_render_scale_rot(mod, g["pos"], g["scales"], g["rotations"], g["opacity"], cam, bg, g["shs"], sh_degree)
        img, _ = GR.rasterize_scale_rot(g["pos"], g["scales"], g["rotations"], g["opacity"], cam, bg, g["shs"], sh_degree)
        want = D.quantize(img_r)
        assert torch.equal(png, D.quantize(img)), "the PNG is not the device render quantised"
        differ = (png != want).any(2)
        flip = (img - img_r).abs().amax(0) > 1e-4
        # a pixel the two rasterizers agree on to 1e-4 may still round the other way at a .5 boundary
        v = img_r.permute(1, 2, 0) * 255 + 0.5
        edge = ((v - v.round()).abs() < 255 * 1e-4 + 1e-3).any(2) | ((v - v.floor()) < 255 * 1e-4 + 1e-3).any(2)
        assert int(flip.sum()) < 1e-4 * flip.numel()
        assert bool((~differ | flip | edge).all()), f"{split} view {i}: {int((differ & ~flip & ~edge).sum())} unexplained pixels"


@pytest.mark.gpu
def test_cli_blender_end_to_end(built_lib, cuda_dev, tmp_path):
    mod = _ref_module()
    rng = np.random.default_rng(21)
    src, model = str(tmp_path / "src"), str(tmp_path / "model")
    write_blender(src, rng, 4, 3, 96, 80, alpha_values=[0, 40, 128, 255])
    write_checkpoint(model, rng, 20000, 16, iteration=30000, extent=0.5)
    write_checkpoint(model, rng, 10, 16, iteration=7000)
    with open(os.path.join(model, "cfg_args"), "w") as f:
        f.write(f"Namespace(sh_degree=3, source_path={src!r}, model_path={model!r}, images='images', resolution=-1, "
                "white_background=True, data_device='cuda', eval=True)")
    before = tree_snapshot(src)
    assert D.main(["-m", model, "--quiet"]) == 0
    assert tree_snapshot(src) == before
    tr, te = D.readNerfSyntheticInfo(src, True, True)
    g = SF.decode_checkpoint_ply_scale_rot(SF.checkpoint_path(model), 3, cuda_dev)
    _check_split(mod, model, "train", 30000, tr, g, 3, [1.0, 1.0, 1.0], -1, cuda_dev)
    _check_split(mod, model, "test", 30000, te, g, 3, [1.0, 1.0, 1.0], -1, cuda_dev)


@pytest.mark.gpu
def test_cli_colmap_end_to_end(built_lib, cuda_dev, tmp_path):
    mod = _ref_module()
    rng = np.random.default_rng(22)
    src, model = str(tmp_path / "src"), str(tmp_path / "model")
    names = [f"img_{k}.png" for k in (3, 1, 2, 0, 4)]
    write_colmap(src, rng, names, [(1700, 40), (64, 48), (65, 47), (64, 48), (80, 60)], binary=True, model="PINHOLE")
    write_checkpoint(model, rng, 5000, 4, iteration=500, extent=0.4)
    with open(os.path.join(model, "cfg_args"), "w") as f:
        f.write(f"Namespace(sh_degree=3, source_path={src!r}, white_background=False)")
    before = tree_snapshot(src)
    assert D.main(["-m", model, "-s", src, "--sh_degree", "1", "--quiet"]) == 0
    assert tree_snapshot(src) == before
    tr, te = D.readColmapSceneInfo(src, None, False)
    assert te == [] and os.path.isdir(os.path.join(model, "test", "ours_500", "renders"))
    g = SF.decode_checkpoint_ply_scale_rot(SF.checkpoint_path(model), 1, cuda_dev)
    _check_split(mod, model, "train", 500, tr, g, 1, [0.0, 0.0, 0.0], -1, cuda_dev)
    wide = np.array(Image.open(os.path.join(model, "train", "ours_500", "gt", "00003.png")))
    assert wide.shape == (37, 1600, 3)        # img_3: 1700 wide, downscaled to 1600 by PIL
