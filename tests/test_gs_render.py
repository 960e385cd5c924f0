"""Frame rendering (pixie_b200.gs_render): cameras and SH against the reference's own Python (tests/golden/render_golden.npz),
the fp64 brute-force rasterizer (oracle/gs_render_ref.py) against closed forms, and the device rasterizer against the
reference's rasterizer binary (built into oracle/_ref/ by oracle/build_gs_rasterizer_ref.py) and the oracle."""
from __future__ import annotations

import importlib.machinery
import importlib.util
import json
import math
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import gs_render_ref as R  # noqa: E402
from pixie_b200 import gs_render as GR  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "render_golden.npz")


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def _cam_dict(cam: GR.Camera):
    return {"view": cam.world_view_transform.numpy().astype(np.float64), "proj": cam.full_proj_transform.numpy().astype(np.float64),
            "campos": cam.camera_center.numpy(), "tan_fovx": math.tan(cam.FoVx * 0.5), "tan_fovy": math.tan(cam.FoVy * 0.5),
            "W": cam.image_width, "H": cam.image_height}


def _check_pose(golden, prefix, pose):
    Rm, T, fx, fy, w, h = pose
    np.testing.assert_allclose(Rm, golden[prefix + "_R"], rtol=0, atol=1e-12)
    np.testing.assert_allclose(T, golden[prefix + "_T"], rtol=0, atol=1e-12)
    np.testing.assert_allclose([fx, fy], golden[prefix + "_fov"], rtol=0, atol=1e-12)
    assert [w, h] == list(golden[prefix + "_wh"])
    cam = GR.make_camera(*pose)
    # float32 matrices of float64 values that agree to 1e-12: equal up to the last float32 bit
    np.testing.assert_allclose(cam.world_view_transform.numpy().T, golden[prefix + "_world_view"], rtol=2e-7, atol=1e-7)
    np.testing.assert_allclose(cam.projection_matrix.numpy().T, golden[prefix + "_proj"], rtol=2e-7, atol=0)


# ------------------------------------------------------------------------------------------------ cameras and SH (CPU)
def test_cameras_json_entries_match_reference(golden):
    cams = json.loads(bytes(golden["cameras_json"]).decode())
    for k in range(len(cams)):
        _check_pose(golden, f"cam_index_{k}", GR.camera_pose(cams, k))


def test_view_centre_and_orbit_cameras_match_reference(golden):
    cams = json.loads(bytes(golden["cameras_json"]).decode())
    for name in ("center_a", "center_b"):
        vc, oc = GR.get_center_view_worldspace_and_observant_coordinate(
            golden[name + "_in_center"], golden[name + "_in_up"], list(torch.from_numpy(golden[name + "_in_rots"])),
            torch.from_numpy(golden[name + "_in_scale"]), torch.from_numpy(golden[name + "_in_mean"]))
        np.testing.assert_allclose(vc, golden[name + "_view_center"], rtol=0, atol=1e-12)
        np.testing.assert_allclose(oc, golden[name + "_observant"], rtol=0, atol=1e-12)
    a, e, r, da, de, dr = golden["orbit_params"]
    vc, oc = golden["center_b_view_center"], golden["center_b_observant"]
    for f in range(6):
        kw = dict(init_azimuthm=a, init_elevation=e, init_radius=r, move_camera=True, current_frame=f, delta_a=da, delta_e=de, delta_r=dr)
        _check_pose(golden, f"orbit_{f}", GR.camera_pose(cams, -1, vc, oc, **kw))
        _check_pose(golden, f"orbit_roll_{f}", GR.camera_pose(cams, -1, vc, oc, init_roll=12.0, delta_roll=2.5, **kw))


def test_oracle_sh_matches_reference(golden):
    for deg in range(4):
        got = R.eval_sh_colors(deg, golden["sh_in_shs"], golden["sh_in_pos"], golden["sh_in_campos"])
        np.testing.assert_allclose(got, golden[f"sh_{deg}"], rtol=0, atol=1e-12)


def test_decode_camera_params_defaults_and_rejections():
    p = GR.decode_camera_params({})
    assert p["mpm_space_viewpoint_center"] == [1.0, 1.0, 1.0] and p["mpm_space_vertical_upward_axis"] == [0, 0, 1]
    assert p["default_camera_index"] == 0 and p["move_camera"] is False and p["init_roll"] == 0.0 and p["delta_a"] is None
    assert GR.decode_camera_params(p) == p
    with pytest.raises(ValueError, match="show_hint"):
        GR.decode_camera_params({"show_hint": True})
    with pytest.raises(ValueError, match="init_azimuthm"):
        GR.decode_camera_params({"default_camera_index": -1})
    with pytest.raises(ValueError, match="delta"):
        GR.decode_camera_params({"move_camera": True, "delta_a": 1.0})
    with pytest.raises(ValueError, match="3 numbers"):
        GR.decode_camera_params({"mpm_space_viewpoint_center": [1.0, 2.0]})
    with pytest.raises(TypeError):
        GR.decode_camera_params([1, 2])
    with pytest.raises(ValueError, match="show_hint"):
        GR.get_camera_view([_simple_camera_json(32, 32)], 0, show_hint=True)
    with pytest.raises(ValueError, match="out of range"):
        GR.get_camera_view([_simple_camera_json(32, 32)], 3)


# ------------------------------------------------------------------------------------------------ oracle hand cases (CPU)
def _simple_camera_json(W, H, f=None):
    """Camera at the origin looking down +z (identity rotation), focal length f (default W)."""
    f = float(W if f is None else f)
    return {"width": W, "height": H, "position": [0.0, 0.0, 0.0], "rotation": np.eye(3).tolist(), "fx": f, "fy": f}


def _simple_cam(W, H, f=None):
    return GR.get_camera_view([_simple_camera_json(W, H, f)], 0)


def _iso_cov(s2, n=1):
    return np.tile([s2, 0.0, 0.0, s2, 0.0, s2], (n, 1))


def _centre_of(W, H):
    """The pixel the image centre maps to: ndc 0 -> ((0 + 1) W - 1) / 2."""
    return (W - 1) / 2.0, (H - 1) / 2.0


def test_oracle_single_isotropic_gaussian():
    W = H = 32
    cam = _cam_dict(_simple_cam(W, H, f=32.0))
    z, s2, o = 2.0, 0.01, 0.7
    img, radii, _ = R.rasterize([[0.0, 0.0, z]], _iso_cov(s2), [o], [[1.0, 0.5, 0.25]], cam, [0.0, 0.0, 0.0])
    # 2D variance: (f / z)^2 s2 + 0.3 on both axes, centred on the image centre
    v = (32.0 / z) ** 2 * s2 + 0.3
    assert radii[0] == math.ceil(3 * math.sqrt(v + math.sqrt(0.1)))
    cx, cy = _centre_of(W, H)
    for (y, x) in ((16, 16), (15, 15), (20, 13)):
        a = min(0.99, o * math.exp(-0.5 * ((x - cx) ** 2 + (y - cy) ** 2) / v))
        want = a if a >= 1 / 255 else 0.0
        np.testing.assert_allclose(img[:, y, x], np.array([1.0, 0.5, 0.25]) * want, rtol=1e-9, atol=1e-12)


def test_oracle_alpha_clamp_and_faint_gaussian():
    W = H = 16
    cam = _cam_dict(_simple_cam(W, H))
    cx, cy = _centre_of(W, H)
    img, _, _ = R.rasterize([[0.0, 0.0, 1.0]], _iso_cov(1.0), [1.0], [[1.0, 1.0, 1.0]], cam, [0.0, 0.0, 1.0])
    # opacity 1 at the centre: alpha clamped to 0.99, T = 0.01 over the blue background
    y, x = int(cy), int(cx)
    a = min(0.99, math.exp(-0.5 * ((x - cx) ** 2 + (y - cy) ** 2) / ((16.0 ** 2) + 0.3)))
    assert a == 0.99
    np.testing.assert_allclose(img[:, y, x], [0.99, 0.99, 0.99 + 0.01], rtol=1e-12)
    # opacity 1/300: alpha below 1/255 everywhere, the background stays
    img, _, contrib = R.rasterize([[0.0, 0.0, 1.0]], _iso_cov(1.0), [1.0 / 300], [[1.0, 1.0, 1.0]], cam, [0.2, 0.3, 0.4])
    assert np.all(img == np.array([0.2, 0.3, 0.4])[:, None, None]) and all(len(c) == 0 for c in contrib.values())


def test_oracle_early_stop_on_opaque_stack():
    W = H = 16
    cam = _cam_dict(_simple_cam(W, H))
    n = 5
    means = [[0.0, 0.0, 1.0 + 0.1 * k] for k in range(n)]
    cols = np.eye(3)[np.arange(n) % 3]
    img, _, contrib = R.rasterize(means, _iso_cov(1.0, n), [1.0] * n, cols, cam, [0.0, 0.0, 0.0])
    y, x = 7, 7
    # alpha 0.99 each: T 1 -> 0.01 -> 1e-4 (not < 1e-4, kept) -> the third would give 1e-6 < 1e-4: stop before it
    a = [min(0.99, math.exp(-0.5 * ((x - 7.5) ** 2 + (y - 7.5) ** 2) / (16.0 ** 2 / (1.0 + 0.1 * k) ** 2 + 0.3))) for k in range(n)]
    T, C, used = 1.0, np.zeros(3), []
    for k in range(n):
        if T * (1 - a[k]) < 1e-4:
            break
        C += cols[k] * a[k] * T
        T *= 1 - a[k]
        used.append(k)
    assert len(used) < n and contrib[(y, x)] == tuple(used)
    np.testing.assert_allclose(img[:, y, x], C, rtol=1e-12)


def test_oracle_culls_behind_near_plane_and_off_screen():
    W = H = 16
    cam = _cam_dict(_simple_cam(W, H))
    means = [[0.0, 0.0, 0.15], [0.0, 0.0, -1.0], [50.0, 0.0, 1.0], [0.0, 0.0, 1.0]]
    img, radii, _ = R.rasterize(means, _iso_cov(0.001, 4), [0.9] * 4, np.ones((4, 3)), cam, [0.0, 0.0, 0.0])
    assert list(radii[:3]) == [0, 0, 0] and radii[3] > 0
    _, radii_alone, _ = R.rasterize(means[3:], _iso_cov(0.001), [0.9], np.ones((1, 3)), cam, [0.0, 0.0, 0.0])
    assert radii[3] == radii_alone[0]


def test_oracle_equal_depths_composite_lower_index_first():
    W = H = 16
    cam = _cam_dict(_simple_cam(W, H))
    means = [[0.0, 0.0, 1.0]] * 2
    img, _, contrib = R.rasterize(means, _iso_cov(0.01, 2), [0.5, 0.5], [[1.0, 0.0, 0.0], [0.0, 1.0, 0.0]], cam, [0.0, 0.0, 0.0])
    y = x = 7
    assert contrib[(y, x)] == (0, 1)
    a = img[0, y, x]
    assert img[1, y, x] == pytest.approx(a * (1 - a), rel=1e-12)   # index 1 behind index 0


def test_oracle_image_size_not_multiple_of_16():
    W, H = 37, 21
    cam = _cam_dict(_simple_cam(W, H))
    rng = np.random.default_rng(0)
    n = 12
    means = np.c_[rng.uniform(-0.5, 0.5, (n, 2)), rng.uniform(1.0, 2.0, n)]
    op, col = rng.uniform(0.3, 0.9, n), rng.uniform(0, 1, (n, 3))
    img, radii, contrib = R.rasterize(means, _iso_cov(0.002, n), op, col, cam, [0.1, 0.1, 0.1])
    assert img.shape == (3, H, W) and len(contrib) == W * H
    # a pixel of the ragged last tile row and column composites exactly its list (closed form from the 2D Gaussians)
    pre = R.preprocess(means, _iso_cov(0.002, n), cam)
    ragged = [(y, x) for (y, x) in contrib if y >= 16 or x >= 32]
    y, x = max(ragged, key=lambda k: len(contrib[k]))
    assert len(contrib[(y, x)]) >= 2
    T, C = 1.0, np.zeros(3)
    for i in contrib[(y, x)]:
        a_, b_, c_ = pre[i]["conic"]
        dx, dy = pre[i]["xy"][0] - x, pre[i]["xy"][1] - y
        al = min(0.99, op[i] * math.exp(-0.5 * (a_ * dx * dx + c_ * dy * dy) - b_ * dx * dy))
        C, T = C + col[i] * al * T, T * (1 - al)
    np.testing.assert_allclose(img[:, y, x], C + 0.1 * T, rtol=1e-12)


# ------------------------------------------------------------------------------------------------ interface (CPU)
def test_capi_symbols_present(built_lib):
    for name in ("pixie_gs_renderer_create", "pixie_gs_render", "pixie_gs_renderer_destroy"):
        assert hasattr(built_lib, name)


def test_rasterize_argument_validation():
    cam = _simple_cam(16, 16)
    n = 4
    m, c, o = torch.zeros(n, 3), torch.zeros(n, 6), torch.ones(n)
    shs = torch.zeros(n, 16, 3)
    bad = [
        dict(means3D=torch.zeros(n, 4)),
        dict(cov3D=torch.zeros(n, 3, 3)),
        dict(opacity=torch.ones(n, 2)),
        dict(shs=torch.zeros(n, 4, 3), sh_degree=2),
        dict(sh_degree=4),
        dict(shs=None),
        dict(colors=torch.zeros(n, 3)),
    ]
    for b in bad:
        kw = dict(means3D=m, cov3D=c, opacity=o, camera=cam, bg=[0, 0, 0], shs=shs, sh_degree=3)
        kw.update(b)
        with pytest.raises(ValueError):
            GR.rasterize(**kw)
    from pixie_b200 import _lib
    with pytest.raises(_lib.PixieError, match="CPU fallback"):
        GR.rasterize(m, c, o, cam, [0, 0, 0], shs=shs, sh_degree=3)


def test_scene_defaults_leave_rendering_off():
    from pixie_b200 import scene_driver as SD
    sc = SD.Scene(name="x", grid=None, mask=None, min_bounds=[0] * 3, max_bounds=[1] * 3, particles=torch.zeros(1, 3))
    assert sc.shs is None and sc.camera_params is None and sc.cameras is None and sc.white_bg is False


# ------------------------------------------------------------------------------------------------ device (GPU)
def _ref_module():
    from oracle import build_gs_rasterizer_ref as B
    path = B.artefact()
    if path is None:
        pytest.skip("the reference rasterizer binary was not built (oracle/build_gs_rasterizer_ref.py)")
    loader = importlib.machinery.ExtensionFileLoader(B.NAME, path)
    spec = importlib.util.spec_from_file_location(B.NAME, path, loader=loader)
    mod = importlib.util.module_from_spec(spec)
    loader.exec_module(mod)
    return mod


def ref_render(mod, means, cov, opacity, cam: GR.Camera, bg, shs=None, deg=0, colors=None):
    dev = means.device
    empty = torch.empty(0, device=dev)
    out = mod.rasterize_gaussians(
        torch.as_tensor(bg, dtype=torch.float32, device=dev), means, colors if colors is not None else empty,
        opacity.reshape(-1, 1).contiguous(), empty, empty, 1.0, cov, cam.world_view_transform.to(dev), cam.full_proj_transform.to(dev),
        math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5), cam.image_height, cam.image_width,
        shs if shs is not None else empty, deg, cam.camera_center.to(dev), False, False)
    return out[1], out[2]


def look_at_camera(W, H, az=30.0, el=20.0, radius=4.0, f_scale=1.0):
    pos, Rm = GR.orbit_camera_pose(az, el, radius, 0.0, np.zeros(3), np.eye(3))
    return GR.get_camera_view([{"width": W, "height": H, "position": pos.tolist(), "rotation": Rm.tolist(), "fx": f_scale * W,
                                "fy": f_scale * W}], 0)


def seeded_scene(n, seed, dev, near_cam=None):
    """Gaussians in a unit ball with anisotropic covariances (axis ratios up to 1e3), opacities across (0, 1], 16 SH
    coefficients; a share straddles the camera's near plane or lies off screen, and a share duplicates others' means
    (exact depth ties)."""
    g = torch.Generator().manual_seed(seed)
    pos = torch.randn(n, 3, generator=g) * 0.6
    k = n // 20
    if near_cam is not None:          # around and behind the near plane (view z 0.2)
        c = near_cam.camera_center
        fwd = -c / c.norm()
        t = torch.rand(k, 1, generator=g) * 0.5 - 0.1
        pos[:k] = c + fwd * t + torch.randn(k, 3, generator=g) * 0.05
    pos[k:2 * k] = torch.randn(k, 3, generator=g) * 8.0                  # mostly off screen
    pos[2 * k:3 * k] = pos[3 * k:4 * k]                                  # exact depth ties
    s = torch.exp(torch.rand(n, 3, generator=g) * math.log(1e3)) * 2e-4  # 2e-4 .. 0.2
    q, _ = torch.linalg.qr(torch.randn(n, 3, 3, generator=g))
    m = q @ torch.diag_embed(s ** 2) @ q.transpose(1, 2)
    cov = torch.stack([m[:, 0, 0], m[:, 0, 1], m[:, 0, 2], m[:, 1, 1], m[:, 1, 2], m[:, 2, 2]], 1)
    opacity = torch.rand(n, 1, generator=g) * 0.98 + 0.02
    shs = torch.randn(n, 16, 3, generator=g) * 0.4
    colors = torch.rand(n, 3, generator=g)
    return [t.to(dev, torch.float32).contiguous() for t in (pos, cov, opacity, shs, colors)]


def compare(img, radii, img_ref, radii_ref, ceil_args=None, label=""):
    """Radii equal (a +-1 step only where the ceil argument is within 1e-5 of an integer); pixels off by more than 1e-4
    (a threshold decision flipped) fewer than 0.01 % of the image. Returns the numbers for the log."""
    d = (radii.long() - radii_ref.long()).cpu()
    bad = torch.nonzero(d).flatten()
    n_step = 0
    if len(bad):
        assert d[bad].abs().max() <= 1, f"{label}: radii differ by more than 1"
        assert ceil_args is not None, f"{label}: {len(bad)} radii differ"
        frac = ceil_args(bad)
        assert np.all(np.abs(frac - np.round(frac)) <= 1e-5), f"{label}: radius step away from an integer ceil argument"
        n_step = len(bad)
    err = (img - img_ref).abs().amax(0)
    n_pix = err.numel()
    n_flip = int((err > 1e-4).sum())
    ok = err[err <= 1e-4]
    print(f"[gs_render] {label}: radii +-1 steps {n_step}, max|err| (agreeing pixels) {float(ok.max()) if ok.numel() else 0:.2e}, "
          f"pixels > 1e-4: {n_flip} / {n_pix}, max|err| {float(err.max()):.2e}")
    assert n_flip < 1e-4 * n_pix, f"{label}: {n_flip} of {n_pix} pixels differ by more than 1e-4"
    return n_step, n_flip


def _ceil_args(means, cov, cam):
    def f(idx):
        idx = idx.numpy()
        pre = R.preprocess(means[idx].cpu().numpy(), cov[idx].cpu().numpy(), _cam_dict(cam))
        return np.array([p["r_arg"] if p is not None else 0.0 for p in pre])
    return f


@pytest.mark.gpu
@pytest.mark.parametrize("n", [2000, 200000])
@pytest.mark.parametrize("wh", [(800, 800), (801, 577)])
def test_device_matches_reference_binary(built_lib, cuda_dev, n, wh):
    mod = _ref_module()
    W, H = wh
    cam = look_at_camera(W, H)
    pos, cov, op, shs, colors = seeded_scene(n, seed=n + W, dev=cuda_dev, near_cam=cam)
    for deg in range(4):
        for bg in ([0.0, 0.0, 0.0], [1.0, 1.0, 1.0]):
            img, radii = GR.rasterize(pos, cov, op, cam, bg, shs=shs, sh_degree=deg)
            img_r, radii_r = ref_render(mod, pos, cov, op, cam, bg, shs=shs, deg=deg)
            compare(img, radii, img_r, radii_r, _ceil_args(pos, cov, cam), f"n={n} {W}x{H} deg={deg} bg={bg[0]}")
    img, radii = GR.rasterize(pos, cov, op, cam, [0.0, 0.0, 0.0], colors=colors)
    img_r, radii_r = ref_render(mod, pos, cov, op, cam, [0.0, 0.0, 0.0], colors=colors)
    compare(img, radii, img_r, radii_r, _ceil_args(pos, cov, cam), f"n={n} {W}x{H} colours")
    assert int((radii == 0).sum()) > 0 and int((radii > 0).sum()) > n // 2


@pytest.mark.gpu
def test_device_matches_oracle_small(built_lib, cuda_dev):
    W, H = 53, 37
    cam = look_at_camera(W, H, radius=3.0)
    pos, cov, op, shs, colors = seeded_scene(300, seed=7, dev=cuda_dev, near_cam=cam)
    img, radii = GR.rasterize(pos, cov, op, cam, [0.3, 0.2, 0.1], shs=shs, sh_degree=3)
    cd = _cam_dict(cam)
    col = R.eval_sh_colors(3, shs.cpu().numpy(), pos.cpu().numpy(), cd["campos"])
    img_o, radii_o, _ = R.rasterize(pos.cpu().numpy(), cov.cpu().numpy(), op.cpu().numpy(), col, cd, [0.3, 0.2, 0.1])
    compare(img, radii, torch.from_numpy(img_o).float().to(cuda_dev), torch.from_numpy(radii_o).to(cuda_dev), _ceil_args(pos, cov, cam),
            "oracle 53x37")


@pytest.mark.gpu
def test_device_renders_are_deterministic(built_lib, cuda_dev):
    cam = look_at_camera(801, 577)
    pos, cov, op, shs, _ = seeded_scene(200000, seed=11, dev=cuda_dev, near_cam=cam)
    a = GR.rasterize(pos, cov, op, cam, [0, 0, 0], shs=shs, sh_degree=3)
    b = GR.rasterize(pos, cov, op, cam, [0, 0, 0], shs=shs, sh_degree=3)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


@pytest.mark.gpu
def test_mpm_rollout_covariances_match_reference_binary(built_lib, cuda_dev):
    """50 frames of the covariances the solver exports (export_particle_cov_to_torch), rendered by both rasterizers."""
    from oracle import mpm_ref
    from pixie_b200.mpm_solver_warp import MPM_Simulator_WARP
    mod = _ref_module()
    dev = cuda_dev
    n, ng = 4000, 32
    sc = mpm_ref.synthetic_scene(n, ng, seed=3)
    g = torch.Generator().manual_seed(3)
    s0 = torch.rand(n, 3, generator=g) * 0.01 + 0.002
    q, _ = torch.linalg.qr(torch.randn(n, 3, 3, generator=g))
    m = q @ torch.diag_embed(s0 ** 2) @ q.transpose(1, 2)
    cov0 = torch.stack([m[:, 0, 0], m[:, 0, 1], m[:, 0, 2], m[:, 1, 1], m[:, 1, 2], m[:, 2, 2]], 1).float().to(dev)
    s = MPM_Simulator_WARP(10)
    s.load_initial_data_from_torch(torch.from_numpy(sc["x"]).to(dev), torch.from_numpy(sc["vol"]).to(dev), cov0, n_grid=ng, grid_lim=2.0)
    s.set_parameters_dict({"material": "jelly", "g": [0.0, 0.0, -9.8], "density": 1000.0, "E": 2e4, "nu": 0.3})
    s.add_bounding_box()
    pos_cam, Rm = GR.orbit_camera_pose(20.0, 25.0, 2.5, 0.0, np.ones(3), np.eye(3))
    cam = GR.get_camera_view([{"width": 801, "height": 577, "position": pos_cam.tolist(), "rotation": Rm.tolist(), "fx": 900.0,
                               "fy": 900.0}], 0)
    op = torch.rand(n, 1, generator=g).to(dev) * 0.9 + 0.1
    shs = (torch.randn(n, 16, 3, generator=g) * 0.4).to(dev)
    steps = flips = 0
    for frame in range(50):
        x = s.export_particle_x_to_torch().contiguous()
        c = s.export_particle_cov_to_torch().view(-1, 6).contiguous()
        img, radii = GR.rasterize(x, c, op, cam, [1, 1, 1], shs=shs, sh_degree=3)
        img_r, radii_r = ref_render(mod, x, c, op, cam, [1, 1, 1], shs=shs, deg=3)
        a, b = compare(img, radii, img_r, radii_r, _ceil_args(x, c, cam), f"MPM frame {frame}")
        steps, flips = steps + a, flips + b
        s.p2g2p_n(10, 2e-4)
    print(f"[gs_render] MPM rollout: {steps} radius steps, {flips} flipped pixels over 50 frames")


@pytest.mark.gpu
def test_scene_driver_renders_frames(built_lib, cuda_dev):
    from oracle import unet_ref as O
    from pixie_b200 import material_transfer as MT
    from pixie_b200 import scene_driver as SD
    mod = _ref_module()
    dev = cuda_dev
    C, G = 64, 16
    seg, reg = O.build_pair(C, G, seed=3)
    drv = SD.SceneBatchDriver(feature_channels=C, grid_size=G, device=dev, seg_state_dict=seg.state_dict(), cont_state_dict=reg.state_dict(),
                              **O.DEFAULT_CFG)
    rng = np.random.default_rng(4)
    K = 8
    pred = np.zeros((3 + K, G, G, G), np.float32)
    pred[:3] = rng.uniform(-0.2, 0.2, size=(3, G, G, G))
    pred[3 + rng.integers(0, K, size=(G, G, G)), np.arange(G)[:, None, None], np.arange(G)[None, :, None], np.arange(G)[None, None, :]] = 1.0
    ranges = dict(density_min=2.95, density_max=3.05, E_min=4.4, E_max=4.6, nu_min=0.29, nu_max=0.31)
    cloud = MT.extract_material_points(torch.from_numpy(pred).to(dev), torch.ones((G, G, G)).to(dev), [-0.5] * 3, [0.5] * 3, ranges)
    # a solid ball of Gaussians: filling (dense cells) adds interior particles
    n = 6000
    v = rng.standard_normal((n, 3))
    pos = (0.4 * v / np.linalg.norm(v, axis=1, keepdims=True) * rng.uniform(0.8, 1.0, (n, 1)) ** (1 / 3)).astype(np.float32)
    s = rng.uniform(0.005, 0.02, size=(n, 3))
    Q, _ = np.linalg.qr(rng.standard_normal((n, 3, 3)))
    m = Q @ (s[:, :, None] ** 2 * np.eye(3)) @ Q.transpose(0, 2, 1)
    cov = np.stack([m[:, 0, 0], m[:, 0, 1], m[:, 0, 2], m[:, 1, 1], m[:, 1, 2], m[:, 2, 2]], axis=1).astype(np.float32)
    opacity = rng.uniform(0.3, 1.0, size=(n, 1)).astype(np.float32)
    shs = (rng.standard_normal((n, 16, 3)) * 0.4).astype(np.float32)
    cameras = [_simple_camera_json(801, 577, 700.0)]
    camera_params = {"default_camera_index": -1, "init_azimuthm": 30.0, "init_elevation": 10.0, "init_radius": 2.0, "move_camera": True,
                     "delta_a": 5.0, "delta_e": 1.0, "delta_r": 0.02, "mpm_space_vertical_upward_axis": [0, 0, 1]}
    mp = {"n_grid": 32, "grid_lim": 2.0, "material": "jelly", "g": [0.0, 0.0, -9.8], "density": 1000.0, "E": 1e5, "nu": 0.3}
    filling = {"n_grid": 40, "density_threshold": 0.5, "search_threshold": 0.2, "max_particles_num": 2000000}
    tp = {"substep_dt": 1e-4, "frame_dt": 2e-3, "frame_num": 3}
    base = dict(name="ball", grid=None, mask=None, min_bounds=[-0.5] * 3, max_bounds=[0.5] * 3, particles=torch.from_numpy(pos),
                cov=torch.from_numpy(cov), opacity=torch.from_numpy(opacity), material_params=mp, bc_params=[{"type": "bounding_box"}],
                time_params=tp, nn_distance_threshold=0.2, particle_filling=filling)
    sc = SD.Scene(**base, shs=torch.from_numpy(shs), sh_degree=3, camera_params=camera_params, cameras=cameras, white_bg=True)
    rec = drv.run_physics_simulation(sc, cloud)
    assert rec["n_particles"] > rec["n_gaussians"] == n and len(rec["frames_rgb"]) == 3
    # the record's frames are rasterize() of its own frames, with the camera of each frame index
    t, scale, mean = SD.transform2origin(torch.from_numpy(pos).to(dev))
    cp = GR.decode_camera_params(camera_params)
    vc, oc = GR.get_center_view_worldspace_and_observant_coordinate(cp["mpm_space_viewpoint_center"], cp["mpm_space_vertical_upward_axis"],
                                                                   [], scale, mean)
    op_d, shs_d = torch.from_numpy(opacity).to(dev), torch.from_numpy(shs).to(dev)
    for f in range(3):
        cam = GR.get_camera_view(cameras, -1, vc, oc, False, 30.0, 10.0, 2.0, None, True, f, 5.0, 1.0, 0.02)
        img, radii = GR.rasterize(rec["frames_pos"][f], rec["frames_cov"][f], op_d, cam, [1, 1, 1], shs=shs_d, sh_degree=3)
        assert torch.equal(img, rec["frames_rgb"][f]), f
        img_r, radii_r = ref_render(mod, rec["frames_pos"][f], rec["frames_cov"][f], op_d, cam, [1, 1, 1], shs=shs_d, deg=3)
        compare(img, radii, img_r, radii_r, _ceil_args(rec["frames_pos"][f], rec["frames_cov"][f], cam), f"driver frame {f}")
    # on_image receives the same frames; the record then has none
    seen = {}
    rec2 = drv.run_physics_simulation(sc, cloud, on_image=lambda f, im: seen.__setitem__(f, im.clone()))
    assert sorted(seen) == [0, 1, 2] and rec2["frames_rgb"] == []
    # the same scene without shs renders nothing and simulates the same frames
    plain = drv.run_physics_simulation(SD.Scene(**base), cloud)
    assert "frames_rgb" not in plain
    for f in range(3):
        assert (plain["frames_pos"][f] - rec["frames_pos"][f]).abs().max() < 2e-5
