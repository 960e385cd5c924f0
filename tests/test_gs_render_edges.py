"""Edges of the Gaussian rasterizer (pixie_b200.gs_render, csrc/gs_render.cu): the blend's 256-record batch boundaries,
tile-rectangle edges, sort widths at powers of two, one-tile and sub-tile images, projection limits, empty and fully
culled frames, the pair-count guard, the persistent renderer's buffer reuse, and frames drawn on several streams and
host threads.

Every device frame is compared three ways:
  - with the fp64 oracle (oracle/gs_render_ref.py): radii equal, except a ±1 step where the ceil argument lies within
    1e-5 of an integer; every pixel whose threshold margin exceeds 1e-5 within 1e-5;
  - with the reference's rasterizer binary (oracle/_ref/): radii identical, |Δpixel| <= 1e-5 except at small-margin pixels;
  - with itself: bit-identical across repeated calls.
The CPU tests hold the oracle's threshold margin and its vectorised compositor to the per-pixel loop on hand cases.
"""
from __future__ import annotations

import math
import threading

import numpy as np
import pytest
import torch

from oracle import gs_render_ref as R
from pixie_b200 import _lib
from pixie_b200 import gs_render as GR
from test_gs_render import _cam_dict, _iso_cov, _ref_module, _simple_cam, look_at_camera, ref_render, seeded_scene

TOL = 1e-5           # pixel bound against both references, and the margin below which a pixel may legitimately differ
F32_NEAR = float(np.float32(0.2))


# ------------------------------------------------------------------------------------------------ scene helpers
def _world(px, py, Z, W, H, f):
    """World point (camera at the origin looking down +z, focal f) that projects to pixel (px, py) at depth Z."""
    px, py, Z = np.broadcast_arrays(*(np.atleast_1d(np.asarray(v, np.float64)) for v in (px, py, Z)))
    return np.stack([(px - (W - 1) / 2.0) * Z / f, (py - (H - 1) / 2.0) * Z / f, Z], 1)


def _iso_cov_for(v2d, Z, f):
    """Covariances flat along the view axis whose 2D covariance at depth Z is v2d I wherever the mean projects (the
    +0.3 dilation included), for the camera of _world with equal focal lengths."""
    s2 = (np.asarray(v2d, np.float64) - 0.3) * (np.asarray(Z, np.float64) / f) ** 2
    s2 = np.atleast_1d(np.broadcast_to(s2, np.broadcast_shapes(np.shape(s2), np.shape(Z))))
    z = np.zeros_like(s2)
    return np.stack([s2, z, z, s2, z, z], 1)


def _v_for_radius(r):
    """2D variance of an isotropic splat whose ceil argument 3 sqrt(v + sqrt(0.1)) is r - 0.5, i.e. radius r."""
    return (r - 0.5) ** 2 / 9.0 - math.sqrt(0.1)


def _dev(*arrays, dev):
    return [torch.as_tensor(np.asarray(a), dtype=torch.float32).to(dev).contiguous() for a in arrays]


def _colors(n, seed):
    return np.random.default_rng(seed).uniform(0.0, 1.0, (n, 3))


@pytest.fixture(scope="module")
def ref_mod():
    return _ref_module()


@pytest.fixture
def fresh_renderers(monkeypatch):
    """A renderer of its own for the test: the shared one's buffers are whatever earlier tests left."""
    monkeypatch.setattr(GR, "_RENDERERS", {})


def three_way(mod, pos, cov, op, cam, bg, shs=None, deg=0, colors=None, label=""):
    """Device vs itself, vs the reference binary and vs the fp64 oracle (see the module docstring). Returns the stats."""
    n = pos.shape[0]
    img, radii = GR.rasterize(pos, cov, op, cam, bg, shs=shs, sh_degree=deg, colors=colors)
    img2, radii2 = GR.rasterize(pos, cov, op, cam, bg, shs=shs, sh_degree=deg, colors=colors)
    assert torch.equal(img, img2) and torch.equal(radii, radii2), f"{label}: repeated calls differ"

    cd = _cam_dict(cam)
    P, Cv, O = (t.detach().cpu().double().numpy() for t in (pos, cov, op))
    col = (R.eval_sh_colors(deg, shs.cpu().double().numpy(), P, cd["campos"]) if shs is not None
           else colors.cpu().double().numpy())
    img_o, radii_o, marg = R.rasterize_tiles(P, Cv, O, col, cd, bg)
    small = marg <= TOL
    d_img = img.cpu().double().numpy()
    r_dev = radii.cpu().numpy().astype(np.int64)

    # the fp64 oracle: a radius may step by one where the ceil argument is within 1e-5 of an integer, and a Gaussian may
    # be kept or culled where its tile rectangle is empty or not under a last-bit change of its screen position
    step = np.nonzero(r_dev != radii_o)[0]
    for i, g in zip(step, R.preprocess(P[step], Cv[step], cd)):
        assert g is not None, f"{label}: Gaussian {i} has radius {r_dev[i]}, the oracle culls it"
        ceils = {math.ceil(g["r_arg"] - R.R_ARG_TOL), math.ceil(g["r_arg"] + R.R_ARG_TOL)}
        ix0, iy0, ix1, iy1 = g["inner"]
        if r_dev[i] == 0 or radii_o[i] == 0:
            ok = (ix1 - ix0) * (iy1 - iy0) == 0 and max(r_dev[i], radii_o[i]) in ceils
        else:
            ok = len(ceils) == 2 and {r_dev[i], radii_o[i]} == ceils
        assert ok, f"{label}: Gaussian {i} has radius {r_dev[i]}, the oracle {radii_o[i]} (ceil argument {g['r_arg']:.7f})"
    e_or = np.abs(d_img - img_o).max(0)
    worst_or = float(e_or[~small].max()) if (~small).any() else 0.0
    assert worst_or <= TOL, (f"{label}: {int((e_or[~small] > TOL).sum())} pixels with margin > {TOL} differ from the oracle "
                             f"by up to {worst_or:.3e}; first at (y, x) {tuple(np.argwhere((e_or > TOL) & ~small)[0])}")

    # the reference binary (it leaves a zero image, not the background, when there are no Gaussians at all)
    worst_ref = float("nan")
    if mod is not None and n > 0:
        img_r, radii_r = ref_render(mod, pos, cov, op, cam, bg, shs=shs, deg=deg, colors=colors)
        assert torch.equal(radii, radii_r), f"{label}: {int((radii != radii_r).sum())} radii differ from the reference binary"
        e_ref = (img - img_r).abs().amax(0).cpu().numpy()
        worst_ref = float(e_ref[~small].max()) if (~small).any() else 0.0
        assert worst_ref <= TOL, (f"{label}: {int((e_ref[~small] > TOL).sum())} pixels with margin > {TOL} differ from the "
                                  f"reference binary by up to {worst_ref:.3e}")
    print(f"[gs_edges] {label}: max|dev - oracle| {worst_or:.2e}, max|dev - binary| {worst_ref:.2e}, small-margin pixels "
          f"{int(small.sum())} / {small.size}, radius steps {len(step)}")
    return {"oracle": worst_or, "binary": worst_ref, "small": int(small.sum()), "img": img, "radii": radii}


# ------------------------------------------------------------------------------------------------ oracle margin (CPU)
def _hand_scenes():
    """The oracle's hand cases of test_gs_render.py plus a seeded ragged scene with ties and a saturating stack."""
    out = []
    cam = _cam_dict(_simple_cam(32, 32, f=32.0))
    out.append(([[0.0, 0.0, 2.0]], _iso_cov(0.01), [0.7], [[1.0, 0.5, 0.25]], cam, [0.0, 0.0, 0.0]))
    cam = _cam_dict(_simple_cam(16, 16))
    out.append(([[0.0, 0.0, 1.0]], _iso_cov(1.0), [1.0], [[1.0, 1.0, 1.0]], cam, [0.0, 0.0, 1.0]))
    out.append(([[0.0, 0.0, 1.0]], _iso_cov(1.0), [1.0 / 300], [[1.0, 1.0, 1.0]], cam, [0.2, 0.3, 0.4]))
    out.append(([[0.0, 0.0, 1.0 + 0.1 * k] for k in range(5)], _iso_cov(1.0, 5), [1.0] * 5, np.eye(3)[np.arange(5) % 3], cam,
                [0.0, 0.0, 0.0]))
    out.append(([[0.0, 0.0, 0.15], [0.0, 0.0, -1.0], [50.0, 0.0, 1.0], [0.0, 0.0, 1.0]], _iso_cov(0.001, 4), [0.9] * 4,
                np.ones((4, 3)), cam, [0.0, 0.0, 0.0]))
    out.append(([[0.0, 0.0, 1.0]] * 2, _iso_cov(0.01, 2), [0.5, 0.5], [[1.0, 0.0, 0.0], [0.0, 1.0, 0.0]], cam, [0.0, 0.0, 0.0]))
    rng = np.random.default_rng(0)
    n = 40
    W, H = 37, 21
    means = np.c_[rng.uniform(-0.5, 0.5, (n, 2)), rng.uniform(1.0, 2.0, n)]
    means[10:20] = means[20:30]                                           # exact depth ties
    cov = _iso_cov(0.002, n)
    cov[:, 1] = 0.0012                                                    # anisotropic
    out.append((means, cov, rng.uniform(0.3, 1.0, n), rng.uniform(0, 1, (n, 3)), _cam_dict(_simple_cam(W, H)), [0.1, 0.2, 0.3]))
    return out


def test_oracle_tiles_match_loop_on_hand_cases():
    for k, (means, cov, op, col, cam, bg) in enumerate(_hand_scenes()):
        img, radii, contrib, marg = R.rasterize(means, cov, op, col, cam, bg, margin=True)
        img_t, radii_t, marg_t = R.rasterize_tiles(means, cov, op, col, cam, bg)
        assert np.array_equal(radii, radii_t), k
        np.testing.assert_allclose(img_t, img, rtol=0, atol=1e-12, err_msg=str(k))
        assert np.array_equal(np.isinf(marg), np.isinf(marg_t)), k
        fin = np.isfinite(marg)
        np.testing.assert_allclose(marg_t[fin], marg[fin], rtol=1e-9, atol=0, err_msg=str(k))
        # a pixel that composited something has considered something
        assert all(np.isfinite(marg[y, x]) for (y, x), used in contrib.items() if used), k


def _one_tile_cam(W=16, H=16):
    return _cam_dict(_simple_cam(W, H))


@pytest.mark.parametrize("rel", [1e-7, 1e-3])
def test_oracle_margin_alpha_at_one_over_255(rel):
    """Opacity chosen so that α at pixel (5, 9) is (1 ± rel)/255: the pixel's margin is rel, and only the pixel above the
    threshold composites the Gaussian."""
    cam = _one_tile_cam()
    means, cov = [[0.013, -0.021, 1.0]], _iso_cov(0.004)
    g = R.preprocess(means, cov, cam)[0]
    y, x = 5, 9
    a, b, c = g["conic"]
    dx, dy = g["xy"][0] - x, g["xy"][1] - y
    e = math.exp(-0.5 * (a * dx * dx + c * dy * dy) - b * dx * dy)
    for sign in (1, -1):
        o = (1 + sign * rel) / 255.0 / e
        img, _, contrib, marg = R.rasterize(means, cov, [o], [[1.0, 1.0, 1.0]], cam, [0.0, 0.0, 0.0], margin=True)
        assert marg[y, x] == pytest.approx(rel, rel=1e-6)
        assert contrib[(y, x)] == ((0,) if sign > 0 else ())
        assert img[0, y, x] == (pytest.approx((1 + rel) / 255.0, rel=1e-12) if sign > 0 else 0.0)
        _, _, marg_t = R.rasterize_tiles(means, cov, [o], [[1.0, 1.0, 1.0]], cam, [0.0, 0.0, 0.0])
        assert marg_t[y, x] == pytest.approx(rel, rel=1e-6)


@pytest.mark.parametrize("stop", [3, 255, 256, 257])
@pytest.mark.parametrize("rel", [1e-7, 1e-2])
def test_oracle_margin_transmittance_at_chosen_entry(stop, rel):
    """A stack of equal wide splats whose α at the tile's centre pixel makes T·(1 − α) cross 1e-4 at entry `stop`
    (0-based), a relative `rel` below it: `stop` entries composite there and the margin is rel."""
    cam = _one_tile_cam()
    K = stop + 4
    Z = 1.0 + 1e-3 * np.arange(K)
    means = _world(7.5, 7.5, Z, 16, 16, 16.0)
    cov = _iso_cov_for(9e4, Z, 16.0)
    pre = R.preprocess(means, cov, cam)
    y = x = 7
    es = []
    for g in pre:
        a, b, c = g["conic"]
        dx, dy = g["xy"][0] - x, g["xy"][1] - y
        es.append(math.exp(-0.5 * (a * dx * dx + c * dy * dy) - b * dx * dy))
    # one alpha for every entry at this pixel: (1 - alpha)^(stop + 1) = 1e-4 (1 - rel)
    alpha = 1.0 - (1e-4 * (1 - rel)) ** (1.0 / (stop + 1))
    op = alpha / np.array(es)
    img, _, contrib, marg = R.rasterize(means, cov, op, _colors(K, 1), cam, [0.0, 0.0, 0.0], margin=True)
    assert contrib[(y, x)] == tuple(range(stop))
    assert marg[y, x] == pytest.approx(rel, rel=1e-3)
    _, _, marg_t = R.rasterize_tiles(means, cov, op, _colors(K, 1), cam, [0.0, 0.0, 0.0])
    assert marg_t[y, x] == pytest.approx(rel, rel=1e-3)


def test_oracle_margin_zero_where_tile_cover_is_a_last_bit_decision():
    """A splat whose left reach px − r lands on a tile edge covers the tile to its left only by rounding; pixels there
    that it could reach with α >= 1/255 get margin 0, and pixels of tiles it surely covers keep their margins."""
    W, H, f = 64, 16, 64.0
    cam = _cam_dict(_simple_cam(W, H, f))
    r = 16
    means, cov = _world(32.0, 7.5, 1.0, W, H, f), _iso_cov_for(_v_for_radius(r) - 0.0, 1.0, f)
    g = R.preprocess(means, cov, cam)[0]
    assert g["radius"] == r and abs(g["xy"][0] - r - 16.0) < 1e-6
    assert g["outer"][0] == 0 and g["inner"][0] == 1
    img, radii, marg = R.rasterize_tiles(means, cov, [1.0], [[1.0, 1.0, 1.0]], cam, [0.0, 0.0, 0.0])
    assert np.all(marg[:, :16][img[0, :, :16] > 0] == 0.0) or np.all(img[0, :, :16] == 0.0)
    assert np.all(marg[:, 16:48] > 1e-3)


# ------------------------------------------------------------------------------------------------ batch boundaries (GPU)
def _stack(K, cfg, order, W, H, dev):
    """K splats on the image centre, one per depth, equal screen footprint; ties: indices 250..261 and 505..519 share a
    depth (straddling the 256 and 512 batch boundaries). cfg: 'never' (T stays above 1e-4), 'stop<s>' (T crosses 1e-4 at
    entry s everywhere, margin ~1.8 %), 'partial' (narrower splats: the centre saturates in batch 0, the corners later)."""
    f = float(W)
    k = np.arange(K)
    Z = 1.0 + 1e-3 * k if order == "front_to_back" else 1.0 + 1e-3 * (K - 1 - k)
    for lo, hi in ((250, 262), (505, 520)):
        if K > lo:
            Z[lo:min(hi, K)] = Z[lo]
    if cfg == "partial":
        v, alpha = 400.0, 0.040
    else:
        v = 9e4
        alpha = 0.0045 if cfg == "never" else 1.0 - 1e-4 ** (1.0 / (int(cfg[4:]) + 0.5))
    means = _world((W - 1) / 2.0, (H - 1) / 2.0, Z, W, H, f)
    cov = _iso_cov_for(v, Z, f)
    op = np.full(K, alpha)
    return _dev(means, cov, op, _colors(K, K), dev=dev), f


@pytest.mark.gpu
@pytest.mark.parametrize("K", [255, 256, 257, 511, 512, 513, 1500])
@pytest.mark.parametrize("wh", [(16, 16), (33, 20)])
def test_blend_batch_boundaries(built_lib, cuda_dev, ref_mod, K, wh):
    W, H = wh
    for cfg in ("never", "stop255", "stop256", "stop257", "partial"):
        for order in ("front_to_back", "back_to_front"):
            (pos, cov, op, col), f = _stack(K, cfg, order, W, H, cuda_dev)
            cam = _simple_cam(W, H, f)
            s = three_way(ref_mod, pos, cov, op, cam, [0.2, 0.1, 0.3], colors=col, label=f"stack K={K} {W}x{H} {cfg} {order}")
            assert int((s["radii"] > 0).sum()) == K
            if W == 16 and K <= 513 and cfg.startswith("stop") and order == "front_to_back":
                # the stack does what it is built for: every pixel composites exactly `stop` entries (or all K)
                _, _, contrib = R.rasterize(*(t.cpu().double().numpy() for t in (pos, cov, op, col)), _cam_dict(cam), [0, 0, 0])
                assert {len(u) for u in contrib.values()} == {min(K, int(cfg[4:]))}, cfg


# ------------------------------------------------------------------------------------------------ tile-rectangle edges (GPU)
def _edge_scene(W, H, dev, seed):
    """Means at 16k − 1, 16k − 0.5, 16k, 16k + 0.5, 16k + 1 on both axes with radii 8, 16 and 32 (so px ± r lands on
    multiples of 16 and on one past them), and means off each side of the image whose rectangles just reach, or just
    miss, tile 0 and the last tile."""
    f = float(W)
    gx, gy = (W + 15) // 16, (H + 15) // 16
    offs = np.array([-1.0, -0.5, 0.0, 0.5, 1.0])
    rng = np.random.default_rng(seed)
    P, V = [], []
    for r in (8, 16, 32):
        xs = np.concatenate([16 * k + offs for k in range(1, gx)])
        ys = np.concatenate([16 * k + offs for k in range(1, gy)])
        X, Y = np.meshgrid(xs, ys[::3])
        P += [np.c_[X.ravel(), Y.ravel()]]
        V += [np.full(X.size, _v_for_radius(r))]
        side = np.concatenate([-r + offs + 0.5, 16 * gx + r + offs - 0.5, W - 1 + r + offs])
        ys_in = rng.uniform(0, H - 1, side.size)
        P += [np.c_[side, ys_in], np.c_[rng.uniform(0, W - 1, side.size), np.concatenate([-r + offs + 0.5, 16 * gy + r + offs - 0.5,
                                                                                          H - 1 + r + offs])]]
        V += [np.full(side.size, _v_for_radius(r))] * 2
    P, V = np.concatenate(P), np.concatenate(V)
    n = len(P)
    Z = rng.uniform(1.0, 3.0, n)
    means = _world(P[:, 0], P[:, 1], Z, W, H, f)
    cov = _iso_cov_for(V, Z, f)
    op = rng.uniform(0.1, 0.9, n)
    shs = rng.normal(0.0, 0.4, (n, 4, 3))
    return _dev(means, cov, op, _colors(n, seed), shs, dev=dev), f


@pytest.mark.gpu
@pytest.mark.parametrize("wh", [(81, 65), (80, 64), (49, 97)])
def test_tile_rectangle_edges(built_lib, cuda_dev, ref_mod, wh):
    W, H = wh
    (pos, cov, op, col, shs), f = _edge_scene(W, H, cuda_dev, seed=W * H)
    cam = _simple_cam(W, H, f)
    s = three_way(ref_mod, pos, cov, op, cam, [0.0, 0.0, 0.0], colors=col, label=f"tile edges {W}x{H} colours")
    assert set(s["radii"][s["radii"] > 0].unique().tolist()) <= {8, 16, 32}
    three_way(ref_mod, pos, cov, op, cam, [1.0, 1.0, 1.0], shs=shs, deg=1, label=f"tile edges {W}x{H} SH 1")


# ------------------------------------------------------------------------------------------------ sort width, image shape (GPU)
SHAPES = [(1, 1), (15, 17), (16, 16), (17, 15), (1, 1000), (1000, 1), (8192, 16), (16, 8192), (1024, 1024), (1024, 1040),
          (4096, 4096)]


def _shape_scene(W, H, dev, seed, big=True):
    """Small splats (σ about 1 % of the image) spread over and just off the image, a deep stack of 600 on tile 0, and
    (big=True) one splat covering every tile; depths from a few values, so many are exact ties, the big one's among them."""
    f = float(max(W, H))
    rng = np.random.default_rng(seed)
    n_small, n_deep = 300, 600
    sig = max(1.0, 0.01 * max(W, H))
    px = np.concatenate([rng.uniform(-2 * sig, W - 1 + 2 * sig, n_small), rng.uniform(0, min(W, 16) - 1, n_deep)])
    py = np.concatenate([rng.uniform(-2 * sig, H - 1 + 2 * sig, n_small), rng.uniform(0, min(H, 16) - 1, n_deep)])
    v = np.full(n_small + n_deep, sig * sig)
    depths = np.array([1.0, 1.25, 1.5, 2.0])
    Z = depths[rng.integers(0, 4, n_small + n_deep)]
    op = rng.uniform(0.02, 0.6, n_small + n_deep)
    if big:
        px, py = np.r_[(W - 1) / 2.0, px], np.r_[(H - 1) / 2.0, py]
        v, Z, op = np.r_[(0.8 * max(W, H)) ** 2, v], np.r_[1.5, Z], np.r_[0.5, op]
    n = len(px)
    means = _world(px, py, Z, W, H, f)
    cov = _iso_cov_for(v, Z, f)
    return _dev(means, cov, op, _colors(n, seed), dev=dev), f


@pytest.mark.gpu
@pytest.mark.parametrize("wh", SHAPES, ids=[f"{w}x{h}" for w, h in SHAPES])
def test_sort_width_and_image_shape(built_lib, cuda_dev, ref_mod, wh):
    W, H = wh
    for big in (True, False):
        (pos, cov, op, col), f = _shape_scene(W, H, cuda_dev, seed=W + 7 * H, big=big)
        cam = _simple_cam(W, H, f)
        s = three_way(ref_mod, pos, cov, op, cam, [0.3, 0.6, 0.9], colors=col, label=f"shape {W}x{H} big={big}")
        if big:
            gx, gy = (W + 15) // 16, (H + 15) // 16
            assert int(s["radii"][0]) >= max(W, H) and gx * gy >= 1
        del s
        torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ projection (GPU)
@pytest.mark.gpu
def test_projection_limits(built_lib, cuda_dev, ref_mod):
    W = H = 64
    f = 64.0
    cam = _simple_cam(W, H, f)
    rng = np.random.default_rng(5)
    # depths one float32 step either side of the 0.2 near plane, and on it
    z0 = np.float32(0.2)
    Zs = np.array([np.nextafter(z0, np.float32(0)), z0, np.nextafter(z0, np.float32(1)), np.float32(0.25)], np.float64)
    means = _world([31.5, 33.0, 30.0, 31.5], [31.5, 30.0, 33.0, 31.5], Zs, W, H, f)
    cov = _iso_cov_for(3.0, Zs, f)
    pos, cv, op, col = _dev(means, cov, [0.8] * 4, _colors(4, 1), dev=cuda_dev)
    s = three_way(ref_mod, pos, cv, op, cam, [0.0, 0.0, 0.0], colors=col, label="near plane")
    assert s["radii"][:2].tolist() == [0, 0] and bool((s["radii"][2:] > 0).all())
    # means on, inside and past the 1.3 tan(fov) clamp of the EWA Jacobian, on every side; wide enough to reach the image
    lim = 1.3 * (W / (2 * f))
    m = []
    for k in (1 - 1e-3, 1.0, 1 + 1e-3, 1.2):
        for sx, sy in ((1, 0), (-1, 0), (0, 1), (0, -1), (1, 1)):
            Z = rng.uniform(1.0, 2.0)
            m.append([sx * lim * k * Z, sy * lim * k * Z, Z])
    m = np.array(m)
    cov = _iso_cov_for(15.0 ** 2, m[:, 2], f)
    cov[:, 1] = cov[:, 0] * 0.3                                           # anisotropic, so the clamp changes the shape
    pos, cv, op, col = _dev(m, cov, rng.uniform(0.3, 0.9, len(m)), _colors(len(m), 2), dev=cuda_dev)
    three_way(ref_mod, pos, cv, op, cam, [0.0, 0.0, 0.0], colors=col, label="1.3 tan(fov) clamp")
    # zero covariance: only the +0.3 dilation is left (radius ceil(3 sqrt(0.3 + sqrt(0.1))) = 3)
    px = 31.5 + np.array([-2.0, -0.25, 0.0, 0.5, 1.75])
    m = _world(px, px[::-1], 1.5, W, H, f)
    pos, cv, op, col = _dev(m, np.zeros((5, 6)), [0.9, 0.5, 0.99, 0.3, 0.7], _colors(5, 3), dev=cuda_dev)
    s = three_way(ref_mod, pos, cv, op, cam, [0.1, 0.1, 0.1], colors=col, label="zero covariance")
    assert s["radii"].tolist() == [3] * 5
    # needles along the view ray
    m = _world(31.5 + np.array([0.0, 3.0, -5.0]), 31.5 + np.array([0.0, -2.0, 4.0]), np.array([1.0, 1.5, 2.0]), W, H, f)
    cov = []
    for p in m:
        d = p / np.linalg.norm(p)
        c = 0.05 * np.outer(d, d) + 1e-8 * np.eye(3)
        cov.append([c[0, 0], c[0, 1], c[0, 2], c[1, 1], c[1, 2], c[2, 2]])
    pos, cv, op, col = _dev(m, np.array(cov), [0.9, 0.6, 0.8], _colors(3, 4), dev=cuda_dev)
    three_way(ref_mod, pos, cv, op, cam, [0.0, 0.0, 0.0], colors=col, label="needles along the ray")
    # opacity 0 and 1, among ordinary splats, with SH colours
    n = 12
    m = _world(rng.uniform(10, 54, n), rng.uniform(10, 54, n), rng.uniform(1.0, 2.0, n), W, H, f)
    op = np.r_[[0.0, 1.0, 0.0, 1.0], rng.uniform(0.2, 0.8, n - 4)]
    pos, cv, op, shs = _dev(m, _iso_cov_for(rng.uniform(4.0, 60.0, n), m[:, 2], f), op, rng.normal(0, 0.4, (n, 16, 3)), dev=cuda_dev)
    three_way(ref_mod, pos, cv, op, cam, [0.0, 0.0, 0.0], shs=shs, deg=3, label="opacity 0 and 1")


# ------------------------------------------------------------------------------------------------ degenerate frames (GPU)
@pytest.mark.gpu
def test_empty_and_culled_frames(built_lib, cuda_dev, ref_mod):
    W, H, f = 37, 21, 37.0
    cam = _simple_cam(W, H, f)
    bg = [0.25, 0.5, 0.75]
    bg_img = torch.tensor(bg, device=cuda_dev)[:, None, None].expand(3, H, W)
    culled = np.array([[0.0, 0.0, -1.0], [0.0, 0.0, 0.1], [0.0, 0.0, F32_NEAR], [60.0, 0.0, 1.0], [0.0, -40.0, 1.0]])
    for n, means in ((0, np.zeros((0, 3))), (1, culled[:1]), (len(culled), culled)):
        cov = _iso_cov(1e-4, n).reshape(n, 6)
        pos, cv, op, col, shs = _dev(means, cov, [0.9] * n, _colors(n, 0).reshape(n, 3), np.full((n, 16, 3), 0.3), dev=cuda_dev)
        for kw in (dict(colors=col), dict(shs=shs, sh_degree=3)):
            img, radii = GR.rasterize(pos, cv, op, cam, bg, **kw)
            assert torch.equal(img, bg_img) and radii.shape == (n,) and int(radii.abs().sum()) == 0, (n, list(kw))
        if n:
            three_way(ref_mod, pos, cv, op, cam, bg, colors=col, label=f"all {n} culled")
    # one visible Gaussian
    pos, cv, op, shs = _dev(_world([20.0], [9.0], 1.3, W, H, f), _iso_cov_for(9.0, 1.3, f), [0.7], np.full((1, 16, 3), 0.2),
                            dev=cuda_dev)
    s = three_way(ref_mod, pos, cv, op, cam, bg, shs=shs, deg=2, label="n=1")
    assert int(s["radii"][0]) > 0


# ------------------------------------------------------------------------------------------------ renderer state (GPU)
def _big_frame(dev, n=33000, W=4096):
    """n centred splats on a W x W camera, each reaching every one of its (W / 16)^2 tiles."""
    f = float(W)
    Z = np.full(n, 2.0)
    means = _world(np.full(n, (W - 1) / 2.0), np.full(n, (W - 1) / 2.0), Z, W, W, f)
    cov = _iso_cov_for((0.2 * W) ** 2, Z, f)
    return _dev(means, cov, np.full(n, 0.5), _colors(n, 9), dev=dev), _simple_cam(W, W, f)


@pytest.mark.gpu
def test_pair_count_guard(built_lib, cuda_dev, ref_mod, fresh_renderers):
    (pos, cov, op, col), cam = _big_frame(cuda_dev)
    pairs = 33000 * (4096 // 16) ** 2
    assert pairs > 2 ** 31 - 1
    with pytest.raises(_lib.PixieError, match=str(pairs)):
        GR.rasterize(pos, cov, op, cam, [0, 0, 0], colors=col)
    r = GR._RENDERERS[torch.device(cuda_dev).index]
    del pos, cov, op, col
    torch.cuda.empty_cache()
    # the same renderer then draws normal frames: one held to both references, one bit-identical to a fresh renderer's
    (pos, cov, op, col), f = _shape_scene(160, 120, cuda_dev, seed=21)
    three_way(ref_mod, pos, cov, op, _simple_cam(160, 120, f), [0.0, 0.0, 0.0], colors=col, label="after the pair-count guard")
    cam = look_at_camera(160, 120, radius=3.0)
    pos, cov, op, shs, _ = seeded_scene(3000, seed=21, dev=cuda_dev, near_cam=cam)
    img, radii = GR.rasterize(pos, cov, op, cam, [0.0, 0.0, 0.0], shs=shs, sh_degree=3)
    assert GR._RENDERERS[torch.device(cuda_dev).index] is r
    GR._RENDERERS.clear()
    img_f, radii_f = GR.rasterize(pos, cov, op, cam, [0.0, 0.0, 0.0], shs=shs, sh_degree=3)
    assert torch.equal(img, img_f) and torch.equal(radii, radii_f)


def _state_frames(dev):
    """(label, inputs, camera) frames that grow and shrink n, the pair count and the image size."""
    out = []
    for seed, (n, (W, H)) in enumerate(((2000, (800, 800)), (100000, (801, 577)), (50, (64, 48)), (3000, (1024, 1024)),
                                        (0, (32, 32)), (20000, (200, 150)), (100000, (801, 577)), (1, (17, 15)))):
        cam = look_at_camera(W, H)
        pos, cov, op, shs, _ = seeded_scene(max(n, 1), seed=100 + seed, dev=dev, near_cam=cam)
        out.append((f"n={n} {W}x{H}", (pos[:n], cov[:n], op[:n], shs[:n]), cam))
    return out


@pytest.mark.gpu
def test_renderer_reuse_matches_fresh_renderer(built_lib, cuda_dev, monkeypatch, fresh_renderers):
    """A sequence through one renderer, with a failed call in the middle; each frame bit-identical to a fresh renderer's."""
    frames = _state_frames(cuda_dev)
    shared = {}
    for k, (label, (pos, cov, op, shs), cam) in enumerate(frames):
        if k == 4:
            (bp, bc, bo, bcol), bcam = _big_frame(cuda_dev)
            monkeypatch.setattr(GR, "_RENDERERS", shared)
            with pytest.raises(_lib.PixieError, match="exceed"):
                GR.rasterize(bp, bc, bo, bcam, [0, 0, 0], colors=bcol)
            del bp, bc, bo, bcol
            torch.cuda.empty_cache()
        monkeypatch.setattr(GR, "_RENDERERS", shared)
        img, radii = GR.rasterize(pos, cov, op, cam, [0.1, 0.2, 0.3], shs=shs, sh_degree=3)
        monkeypatch.setattr(GR, "_RENDERERS", {})
        img_f, radii_f = GR.rasterize(pos, cov, op, cam, [0.1, 0.2, 0.3], shs=shs, sh_degree=3)
        assert torch.equal(img, img_f) and torch.equal(radii, radii_f), label
    assert len(shared) == 1


# ------------------------------------------------------------------------------------------------ streams and threads (GPU)
def _heavy_and_light(dev):
    cam_a = look_at_camera(800, 800)
    a = seeded_scene(250000, seed=31, dev=dev, near_cam=cam_a)
    cam_b = look_at_camera(200, 150)
    b = seeded_scene(3000, seed=32, dev=dev, near_cam=cam_b)
    return (a, cam_a), (b, cam_b)


def _render(scene, cam, bg):
    pos, cov, op, shs, _ = scene
    return GR.rasterize(pos, cov, op, cam, bg, shs=shs, sh_degree=3)


@pytest.mark.gpu
def test_frames_on_two_streams_keep_their_order(built_lib, cuda_dev, fresh_renderers):
    """A heavy frame A on stream s1 and, with no host sync between, a light frame B on s2: B's preprocess, scan, keys and
    blend would otherwise overwrite the buffers A's sort, ranges and blend still read."""
    (a, cam_a), (b, cam_b) = _heavy_and_light(cuda_dev)
    ref_b = _render(b, cam_b, [0, 0, 0])          # warm with B, then A grows every buffer; B then grows none
    ref_a = _render(a, cam_a, [0, 0, 0])
    torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    for _ in range(3):
        torch.cuda.synchronize()
        with torch.cuda.stream(s1):
            img_a, radii_a = _render(a, cam_a, [0, 0, 0])
        with torch.cuda.stream(s2):
            img_b, radii_b = _render(b, cam_b, [0, 0, 0])
        torch.cuda.synchronize()
        assert torch.equal(img_a, ref_a[0]) and torch.equal(radii_a, ref_a[1]), \
            f"frame A corrupted: {int((img_a != ref_a[0]).any(0).sum())} pixels differ"
        assert torch.equal(img_b, ref_b[0]) and torch.equal(radii_b, ref_b[1]), "frame B corrupted"


@pytest.mark.gpu
def test_frames_from_two_host_threads(built_lib, cuda_dev, fresh_renderers):
    (a, cam_a), (b, cam_b) = _heavy_and_light(cuda_dev)
    ref_a, ref_b = _render(a, cam_a, [1, 1, 1]), _render(b, cam_b, [1, 1, 1])
    torch.cuda.synchronize()
    results, errors = {}, []

    def work(name, scene, cam):
        try:
            s = torch.cuda.Stream(device=cuda_dev)
            out = []
            with torch.cuda.device(cuda_dev), torch.cuda.stream(s):
                for _ in range(4):
                    out.append(_render(scene, cam, [1, 1, 1]))
            s.synchronize()
            results[name] = out
        except Exception as e:  # noqa: BLE001 - reported below
            errors.append(repr(e))

    threads = [threading.Thread(target=work, args=("a", a, cam_a)), threading.Thread(target=work, args=("b", b, cam_b))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    torch.cuda.synchronize()
    assert not errors, errors
    for name, ref in (("a", ref_a), ("b", ref_b)):
        for k, (img, radii) in enumerate(results[name]):
            assert torch.equal(img, ref[0]) and torch.equal(radii, ref[1]), f"thread {name} frame {k}"
