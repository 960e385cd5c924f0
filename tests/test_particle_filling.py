"""Particle filling (PG/particle_filling/filling.py:291-380). CPU: the numpy oracle against the reference's own Taichi kernels
(tests/golden/filling_golden.npz, made by tests/golden/make_filling_golden.py) and against hand cases; argument handling,
config defaults, exported symbols and a spill-free build. GPU: the device kernels against the golden file and against the
oracle at config size, seeds, capacity, and the scene driver with a filling block."""
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import particle_filling_ref as R  # noqa: E402

GOLDEN = os.path.join(HERE, "golden", "filling_golden.npz")
CASES = ["shell", "cups", "nested", "flat", "clipped", "ppc2", "boundary"]
F32 = np.float32


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def case(g, name):
    b = g[f"{name}/boundary"]
    kw = dict(grid_n=int(g[f"{name}/grid_n"]), max_samples=int(g[f"{name}/max_samples"]), grid_dx=float(g[f"{name}/grid_dx"]),
              density_thres=float(g[f"{name}/density_thres"]), search_thres=float(g[f"{name}/search_thres"]),
              max_particles_per_cell=int(g[f"{name}/max_particles_per_cell"]), search_exclude_dir=int(g[f"{name}/search_exclude_dir"]),
              ray_cast_dir=int(g[f"{name}/ray_cast_dir"]), boundary=[float(v) for v in b] if len(b) else None)
    return g[f"{name}/pos"], g[f"{name}/opacity"], g[f"{name}/cov"], kw


def frame(kw):
    """(grid_dx, origin) of the splat grid, as fill_particles derives them."""
    b = kw["boundary"]
    if b is None:
        return kw["grid_dx"], np.zeros(3)
    return max(b[2 * i + 1] - b[2 * i] for i in range(3)) / kw["grid_n"], np.array([b[0], b[2], b[4]], F32).astype(np.float64)


def cells_of(new, grid_dx, origin, grid_n):
    """Cell of every new particle (float64 arithmetic) and the largest distance outside that cell, in units of grid_dx."""
    q = (np.asarray(new, np.float64) - origin) / grid_dx
    c = np.clip(np.floor(q), 0, grid_n - 1)
    return c.astype(np.int64), float(np.max(np.maximum(c - q, q - (c + 1)), initial=-1.0))


def per_cell(cells, grid_n):
    h = np.zeros(grid_n ** 3, np.int64)
    np.add.at(h, (cells[:, 0] * grid_n + cells[:, 1]) * grid_n + cells[:, 2], 1)
    return h.reshape((grid_n,) * 3)


def assert_density(got, want, rtol):
    # densities are compared at the scale of the thresholds (O(1)); tails far below it only need the absolute bound
    np.testing.assert_allclose(got, want, rtol=rtol, atol=1e-6)


# ------------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference_kernels(golden, name):
    pos, opacity, cov, kw = case(golden, name)
    r = R.fill_particles(pos, opacity, cov, seed=1, **kw)
    assert np.array_equal(r["count"], golden[f"{name}/count_densify"])
    assert_density(r["density"], golden[f"{name}/density"], 1e-6)
    assert np.array_equal(r["count_dense"], golden[f"{name}/count_dense"])
    assert np.array_equal(r["count_internal"], golden[f"{name}/count_internal"])
    n_dense, n_total = int(golden[f"{name}/n_dense"]), int(golden[f"{name}/n_total"])
    assert (r["n_dense"], r["n_total"]) == (n_dense, n_total)
    assert n_total > n_dense > 0
    # the reference's own output: every input Gaussian first, then n_total new particles, dense-cell ones first
    out = golden[f"{name}/out"]
    assert out.shape == (len(pos) + n_total, 3) and np.array_equal(out[:len(pos)], pos)
    dx, origin = frame(kw)
    n = kw["grid_n"]
    want_dense = golden[f"{name}/count_dense"] - golden[f"{name}/count_densify"]
    want_inner = golden[f"{name}/count_internal"] - golden[f"{name}/count_dense"]
    for new in (out[len(pos):], r["out"][len(pos):]):
        c, outside = cells_of(new, dx, origin, n)
        assert outside <= 1e-5, outside
        assert np.array_equal(per_cell(c[:n_dense], n), want_dense)
        assert np.array_equal(per_cell(c[n_dense:], n), want_inner)
    assert np.array_equal(r["add_dense"], want_dense) and np.array_equal(r["add_interior"], want_inner)


def test_golden_cases_cover_the_rules(golden):
    """What the cases are there for: filled / unfilled cavities, clipped windows, clamped eigenvalues, max_ppc = 2."""
    inner = {k: golden[f"{k}/count_internal"] - golden[f"{k}/count_dense"] for k in CASES}
    c = lambda v: int(round(v * 24 / 2.0))                                           # noqa: E731  (simulation frame -> cell)
    assert inner["cups"][c(0.6), c(1.0), c(1.0)] == 1 and inner["cups"][c(1.4), c(1.0), c(1.0)] == 0
    assert inner["nested"][c(1.0), c(1.0), c(1.0)] == 0 and inner["nested"][c(1.0), c(1.0), c(0.45)] == 1
    assert inner["shell"][c(1.0), c(1.0), c(1.0)] == 1 and inner["flat"][c(1.0), c(1.0), c(1.0)] == 1
    assert np.any(golden["flat/cov"][:, 5] <= 0) and np.any(golden["flat/cov"][:, 5] < 0)
    assert int(golden["ppc2/max_particles_per_cell"]) == 2
    topped = (golden["ppc2/count_densify"] == 1) & (golden["ppc2/count_dense"] == 2)
    assert topped.sum() > 0
    pos = golden["boundary/pos"]
    b = golden["boundary/boundary"]
    assert np.any((pos < b[::2].astype(F32)) | (pos > b[1::2].astype(F32)))
    # the clipped case's first Gaussians have windows of radius >= 3 reaching past the grid
    sig = np.linalg.eigvalsh(golden["clipped/cov"][:4][:, [0, 1, 2, 1, 3, 4, 2, 4, 5]].reshape(-1, 3, 3).astype(np.float64))
    assert np.all(np.ceil(np.sqrt(sig.max(1)) / (2.0 / 24)) >= 3)


def test_oracle_isotropic_gaussian_is_analytic():
    n, dx, s, op = 12, 0.1, 0.13, 0.7
    p = np.array([[0.537, 0.612, 0.488]], F32)
    count, density = R.densify_grids(p, [op], [[s * s, 0, 0, s * s, 0, s * s]], n, dx)
    r = int(np.ceil(np.float32(s) / np.float32(dx)))
    c0 = np.floor(p[0] / F32(dx)).astype(int)
    want = np.zeros((n, n, n))
    for i, j, k in np.ndindex(n, n, n):
        if np.all(np.abs(np.array([i, j, k]) - c0) <= r):
            nodes = (np.array([i, j, k]) + np.array([[a, b, c] for a in (0, 1) for b in (0, 1) for c in (0, 1)])) * dx
            want[i, j, k] = op * np.mean(np.exp(-0.5 * ((p[0].astype(np.float64) - nodes) ** 2).sum(1) / (s * s)))
    assert count.sum() == 1 and count[tuple(c0)] == 1
    np.testing.assert_allclose(density, want, rtol=2e-6, atol=1e-12)


def cube_shells(n, shells, value=10.0):
    """A density grid holding the cell faces of the cubes [lo, hi]^3 (cell indices) and an empty count grid."""
    d = np.zeros((n, n, n), F32)
    for lo, hi in shells:
        box = np.zeros((n, n, n), bool)
        box[lo:hi + 1, lo:hi + 1, lo:hi + 1] = True
        inner = np.zeros((n, n, n), bool)
        inner[lo + 1:hi, lo + 1:hi, lo + 1:hi] = True
        d[box & ~inner] = value
    return np.zeros((n, n, n), np.int32), d


def box_mask(n, lo, hi):
    m = np.zeros((n, n, n), bool)
    m[lo:hi + 1, lo:hi + 1, lo:hi + 1] = True
    return m


def test_oracle_cube_shell_fills_exactly_its_interior():
    count, d = cube_shells(16, [(3, 11)])
    c1, c2, add_d, add_i = R.fill_grids(count, d, 5.0, 3.0, 1, 5, 4)
    assert np.array_equal(add_d > 0, d > 5.0)
    assert np.array_equal(add_i > 0, box_mask(16, 4, 10))


def test_oracle_nested_shells_leave_the_inner_cavity_empty():
    count, d = cube_shells(20, [(2, 17), (7, 12)])
    _, _, _, add_i = R.fill_grids(count, d, 5.0, 3.0, 1, 5, 4)
    filled = add_i > 0
    annulus = box_mask(20, 3, 16) & ~box_mask(20, 7, 12)
    column = np.zeros_like(filled)
    column[7:13, 7:13, :] = True
    assert not filled[8:12, 8:12, 8:12].any()                     # +z from the cavity: inner lid + outer lid = even
    assert not np.any(filled & ~annulus)
    assert filled[annulus & ~column].all()                        # one lid above
    assert filled[8:12, 8:12, 3:7].all()                          # inner floor, inner lid, outer lid: odd
    # above a side wall of the inner cube the +z ray meets the wall as ONE run, then the outer lid: even, not filled
    assert not filled[7, 9, 3:7].any()


def test_decode_filling_params_defaults():
    from pixie_b200.particle_filling import decode_filling_params
    p = decode_filling_params({}, {"n_grid": 50})
    assert p == {"n_grid": 200, "density_threshold": 5.0, "search_threshold": 3.0, "max_particles_num": 2000000,
                 "max_partciels_per_cell": 1, "search_exclude_direction": 5, "ray_cast_direction": 4, "boundary": None,
                 "smooth": False, "visualize": False}
    metal = {"n_grid": 50, "density_threshold": 40.0, "search_threshold": 0.5, "search_exclude_direction": 0, "ray_cast_direction": 1,
             "max_particles_num": 2000000, "max_partciels_per_cell": 1, "boundary": [0.86, 1.46, 0.7, 1.3, 0.7, 1.3]}
    q = decode_filling_params(metal, {"n_grid": 120})
    assert q == dict(metal, smooth=False, visualize=False) and "smooth" not in metal


def test_fill_particles_argument_checks():
    from pixie_b200 import _lib
    from pixie_b200.particle_filling import fill_particles
    p, o, c = torch.zeros(4, 3), torch.ones(4, 1), torch.zeros(4, 6)
    with pytest.raises(NotImplementedError, match="mcubes"):
        fill_particles(p, o, c, 10, 100, 0.1, smooth=True)                        # before any device check
    with pytest.raises(ValueError):
        fill_particles(p, o, c, 10, 100, 0.1, search_exclude_dir=6)
    with pytest.raises(ValueError):
        fill_particles(p, o, c, 10, 100, 0.1, ray_cast_dir=-1)
    with pytest.raises(ValueError):
        fill_particles(p, o, c, 0, 100, 0.1)
    with pytest.raises(ValueError):
        fill_particles(p, o[:3], c, 10, 100, 0.1)
    with pytest.raises(ValueError):
        fill_particles(p, o, c[:, :5], 10, 100, 0.1)
    with pytest.raises(_lib.PixieError):
        fill_particles(p, o, c, 10, 100, 0.1)


def test_library_exports_filling_symbols(built_lib):
    for s in ("pixie_fill_density", "pixie_fill_grids"):
        assert hasattr(built_lib, s)


def test_particle_fill_kernels_do_not_spill(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    src = os.path.join(ROOT, "pixie_b200", "csrc", "particle_fill.cu")
    res = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-c", src,
                          "-o", str(tmp_path / "particle_fill.o")], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", res.stderr)
    assert len(spills) >= 5
    assert all(s == ("0", "0") for s in spills), res.stderr


# ------------------------------------------------------------------------------------------------------------------ GPU
def _dev(x, dev):
    return torch.from_numpy(np.ascontiguousarray(x)).to(dev)


def crop(pos, opacity, cov, boundary, dev):
    """The Gaussians fill_particles splats, on the device: strictly inside the boundary, shifted to its corner."""
    p, o, c = _dev(pos, dev), _dev(opacity, dev), _dev(cov, dev)
    if boundary is None:
        return p, o, c
    b = boundary
    keep = torch.ones(len(pos), dtype=torch.bool, device=dev)
    for i in range(3):
        keep &= (p[:, i] > b[2 * i]) & (p[:, i] < b[2 * i + 1])
    return p[keep] - torch.tensor([b[0], b[2], b[4]], device=dev), o[keep], c[keep]


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_device_matches_reference_kernels(built_lib, cuda_dev, golden, name):
    from pixie_b200 import particle_filling as PF
    pos, opacity, cov, kw = case(golden, name)
    dx, origin = frame(kw)
    n = kw["grid_n"]
    # the grids, on the splat frame the reference uses (crop and shift as fill_particles does them)
    count, density = PF.densify_grids(*crop(pos, opacity, cov, kw["boundary"], cuda_dev), n, dx)
    assert np.array_equal(count.cpu().numpy(), golden[f"{name}/count_densify"])
    assert_density(density.cpu().numpy(), golden[f"{name}/density"], 1e-5)
    new, n_dense = PF.fill_grids(count, density, dx, kw["max_samples"], kw["density_thres"], kw["search_thres"], kw["max_particles_per_cell"],
                                 kw["search_exclude_dir"], kw["ray_cast_dir"], origin, seed=3)
    assert n_dense == int(golden[f"{name}/n_dense"]) and new.shape[0] == int(golden[f"{name}/n_total"])
    assert np.array_equal(count.cpu().numpy(), golden[f"{name}/count_internal"])
    cells, outside = cells_of(new.cpu().numpy(), dx, origin, n)
    assert outside <= 1e-5, outside
    assert np.array_equal(per_cell(cells[:n_dense], n), golden[f"{name}/count_dense"] - golden[f"{name}/count_densify"])
    assert np.array_equal(per_cell(cells[n_dense:], n), golden[f"{name}/count_internal"] - golden[f"{name}/count_dense"])
    # the public entry point: every input Gaussian first, bit for bit (those outside the boundary too), then the new ones
    out = PF.fill_particles(_dev(pos, cuda_dev), _dev(opacity, cuda_dev), _dev(cov, cuda_dev), seed=3, **kw)
    assert out.dtype == torch.float32 and out.device == torch.device(cuda_dev)
    assert torch.equal(out[:len(pos)].cpu(), torch.from_numpy(pos))
    assert torch.equal(out[len(pos):], new)


@pytest.mark.gpu
def test_device_cube_shells(built_lib, cuda_dev):
    from pixie_b200 import particle_filling as PF
    count, d = cube_shells(20, [(2, 17), (7, 12)])
    cd = _dev(count, cuda_dev)
    new, n_dense = PF.fill_grids(cd, _dev(d, cuda_dev), 0.05, 10 ** 5, 5.0, 3.0, 1, 5, 4)
    want = R.fill_grids(count, d, 5.0, 3.0, 1, 5, 4)
    assert n_dense == int(want[2].sum()) and new.shape[0] == int(want[2].sum() + want[3].sum())
    assert np.array_equal(cd.cpu().numpy(), want[1])


def shell_scene(n, center, radius, std, seed):
    rng = np.random.default_rng(seed)
    v = rng.standard_normal((n, 3))
    pos = (center + radius * (1 + 0.02 * rng.standard_normal((n, 1))) * v / np.linalg.norm(v, axis=1, keepdims=True)).astype(F32)
    s = rng.uniform(0.5, 1.5, size=(n, 3)) * std
    q = rng.standard_normal((n, 3, 3))
    Q, _ = np.linalg.qr(q)
    m = Q @ (s[:, :, None] ** 2 * np.eye(3)) @ Q.transpose(0, 2, 1)
    cov = np.stack([m[:, 0, 0], m[:, 0, 1], m[:, 0, 2], m[:, 1, 1], m[:, 1, 2], m[:, 2, 2]], axis=1).astype(F32)
    return pos, rng.uniform(0.3, 1.0, size=(n, 1)).astype(F32), cov


def clear_of(density, thr):
    """A threshold no cell density lies within 1e-5 (relative) of, near `thr`: the float32 summation order of the splat
    (about 1e-6 relative) cannot flip a cell."""
    for k in range(1000):
        t = thr * (1 + 3e-5 * k)
        if not np.any(np.abs(density.astype(np.float64) - t) <= 1e-5 * t):
            return t
    raise AssertionError("no clear threshold")


CONFIGS = {
    # metal / fruit / soda cans: n_grid 50 over the metal boundary, exclude +x, ray -x
    "metal": dict(center=(1.16, 1.0, 1.0), radius=0.22, std=0.004, grid_n=50, boundary=[0.86, 1.46, 0.7, 1.3, 0.7, 1.3],
                  density_thres=40.0, search_thres=0.5, search_exclude_dir=0, ray_cast_dir=1),
    # the n_grid 100 configs over a 1.2 box, exclude +y, ray +z
    "box100": dict(center=(1.0, 1.0, 1.0), radius=0.45, std=0.008, grid_n=100, boundary=[0.4, 1.6, 0.4, 1.6, 0.4, 1.6],
                   density_thres=100.0, search_thres=1.0, search_exclude_dir=2, ray_cast_dir=4),
}


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", sorted(CONFIGS))
def test_device_matches_oracle_at_config_size(built_lib, cuda_dev, cfg):
    from pixie_b200 import particle_filling as PF
    k = dict(CONFIGS[cfg])
    pos, opacity, cov = shell_scene(200_000, np.array(k.pop("center")), k.pop("radius"), k.pop("std"), seed=11)
    b = k["boundary"]
    lo, hi = np.array(b[::2], F32), np.array(b[1::2], F32)
    keep = np.all((pos > lo) & (pos < hi), axis=1)
    _, dens = R.densify_grids(pos[keep] - lo, opacity[keep], cov[keep], k["grid_n"], max(hi - lo) / k["grid_n"])
    # thresholds scaled to what this synthetic shell reaches, then moved clear of every cell density
    scale = float(np.percentile(dens[dens > 0], 90)) / k["density_thres"]
    k["density_thres"] = clear_of(dens, k["density_thres"] * scale)
    k["search_thres"] = clear_of(dens, k["search_thres"] * scale)
    want = R.fill_particles(pos, opacity, cov, max_samples=2_000_000, grid_dx=1.0, **k)
    # a shell this dense puts Gaussians in every cell above the density threshold: nearly all new particles are interior ones
    assert want["n_total"] - want["n_dense"] > 1000
    # same cells: the device's count grid after both fills is the oracle's, cell for cell
    n, dx = k["grid_n"], want["grid_dx"]
    count, density = PF.densify_grids(*crop(pos, opacity, cov, b, cuda_dev), n, dx)
    new, n_dense = PF.fill_grids(count, density, dx, 2_000_000, k["density_thres"], k["search_thres"], 1, k["search_exclude_dir"],
                                 k["ray_cast_dir"], want["origin"])
    assert (n_dense, new.shape[0]) == (want["n_dense"], want["n_total"])
    assert np.array_equal(count.cpu().numpy(), want["count_internal"])
    _, outside = cells_of(new.cpu().numpy(), dx, want["origin"].astype(np.float64), n)
    assert outside <= 1e-5
    out = PF.fill_particles(_dev(pos, cuda_dev), _dev(opacity, cuda_dev), _dev(cov, cuda_dev), max_samples=2_000_000, grid_dx=1.0, **k)
    assert out.shape[0] == len(pos) + want["n_total"] and torch.equal(out[:len(pos)].cpu(), torch.from_numpy(pos))
    assert torch.equal(out[len(pos):], new)


@pytest.mark.gpu
def test_seeds_and_capacity(built_lib, cuda_dev, golden):
    from pixie_b200 import _lib
    from pixie_b200 import particle_filling as PF
    pos, opacity, cov, kw = case(golden, "boundary")
    args = (_dev(pos, cuda_dev), _dev(opacity, cuda_dev), _dev(cov, cuda_dev))
    a = PF.fill_particles(*args, seed=5, **kw)
    b = PF.fill_particles(*args, seed=5, **kw)
    c = PF.fill_particles(*args, seed=6, **kw)
    assert torch.equal(a, b)
    assert a.shape == c.shape and torch.equal(a[:len(pos)], c[:len(pos)])
    dx, origin = frame(kw)
    ca, _ = cells_of(a[len(pos):].cpu().numpy(), dx, origin, kw["grid_n"])
    cc, _ = cells_of(c[len(pos):].cpu().numpy(), dx, origin, kw["grid_n"])
    assert np.array_equal(ca, cc)                                                     # same cells, in the same order
    assert (a[len(pos):] != c[len(pos):]).all(dim=1).float().mean() > 0.99            # different offsets
    total = int(golden["boundary/n_total"])
    with pytest.raises(_lib.PixieError, match=f"{total}.*{total - 1}"):
        PF.fill_particles(*args, **dict(kw, max_samples=total - 1))
    assert PF.fill_particles(*args, **dict(kw, max_samples=total)).shape[0] == len(pos) + total


@pytest.mark.gpu
def test_scene_driver_simulates_filled_scene(built_lib, cuda_dev):
    from oracle import unet_ref as O
    from pixie_b200 import frame_export as FE
    from pixie_b200 import material_transfer as MT
    from pixie_b200 import particle_filling as PF
    from pixie_b200 import scene_driver as SD
    from pixie_b200.mpm_solver_warp import MPM_Simulator_WARP
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
    mask = torch.ones((G, G, G))
    ranges = dict(density_min=2.95, density_max=3.05, E_min=4.4, E_max=4.6, nu_min=0.29, nu_max=0.31)
    cloud = MT.extract_material_points(torch.from_numpy(pred).to(dev), mask.to(dev), [-0.5] * 3, [0.5] * 3, ranges)
    # a hollow sphere in the Gaussians' frame: after transform2origin / shift2center111 it spans [0.5, 1.5]^3
    pos, opacity, cov = shell_scene(6000, np.zeros(3), 0.5, 0.02, seed=5)
    mp = {"n_grid": 32, "grid_lim": 2.0, "material": "jelly", "g": [0.0, 0.0, -9.8], "density": 1000.0, "E": 1e5, "nu": 0.3,
          "grid_v_damping_scale": 0.9999}
    t, scale, mean = SD.transform2origin(torch.from_numpy(pos).to(dev))
    pos0 = t + torch.tensor([1.0, 1.0, 1.0], device=dev)
    cov0 = torch.from_numpy(cov).to(dev) * scale ** 2
    bnd = [0.45, 1.55, 0.45, 1.55, 0.45, 1.55]
    # thresholds clear of every cell density, so that the float atomics' order cannot flip a cell between the two runs
    keep = ((pos0 > 0.45) & (pos0 < 1.55)).all(dim=1)
    _, dens = PF.densify_grids(pos0[keep] - torch.tensor([0.45] * 3, device=dev), torch.from_numpy(opacity).to(dev)[keep], cov0[keep], 50, (1.55 - 0.45) / 50)
    dens = dens.cpu().numpy()
    filling = {"n_grid": 50, "density_threshold": clear_of(dens, 2.0), "search_threshold": clear_of(dens, 0.5), "search_exclude_direction": 0,
               "ray_cast_direction": 1, "max_particles_num": 2000000, "max_partciels_per_cell": 1, "boundary": bnd}
    tp = {"substep_dt": 1e-4, "frame_dt": 2e-3, "frame_num": 3}
    sc = SD.Scene(name="can", grid=None, mask=None, min_bounds=[-0.5] * 3, max_bounds=[0.5] * 3, particles=torch.from_numpy(pos),
                  cov=torch.from_numpy(cov), opacity=torch.from_numpy(opacity), material_params=mp, bc_params=[{"type": "bounding_box"}],
                  time_params=tp, nn_distance_threshold=0.2, particle_filling=filling)
    rec = drv.run_physics_simulation(sc, cloud)
    n_gs = len(pos)
    assert rec["n_gaussians"] == n_gs and rec["n_particles"] > n_gs + 1000
    assert all(f.shape == (n_gs, 3) for f in rec["frames_pos"]) and all(f.shape == (n_gs, 6) for f in rec["frames_cov"])
    # by hand: fill_particles -> get_particle_volume -> solver -> kNN -> p2g2p_n
    full = PF.fill_particles(pos0, torch.from_numpy(opacity).to(dev), cov0, 50, 2000000, 2.0 / 50, filling["density_threshold"],
                             filling["search_threshold"], 1, 0, 1, bnd)
    assert full.shape[0] == rec["n_particles"]
    cov_full = torch.zeros((full.shape[0], 6), device=dev)
    cov_full[:n_gs] = cov0
    s = MPM_Simulator_WARP(10, device=dev)
    s.load_initial_data_from_torch(full, FE.get_particle_volume(full, 32, 2.0 / 32), cov_full, n_grid=32, grid_lim=2.0, device=dev)
    s.set_parameters_dict(dict(mp), device=dev)
    s.add_bounding_box()
    q, _ = FE.render_frame_transform(s.export_particle_x_to_torch(), None, 0.0, scale, mean, [])
    props = MT.perform_knn_smoothing(q, cloud, 10, 0.2)
    MT.apply_material_properties_to_solver(s, props[1], props[2], props[3], props[4], device=dev, exact_box_semantics=False)
    assert torch.equal(props[4].cpu(), rec["material_ids"].cpu())
    for f in range(3):
        x = s.export_particle_x_to_torch()
        pr, cr = FE.render_frame_transform(x[:n_gs], s.export_particle_cov_to_torch().view(-1, 6)[:n_gs], 0.0, scale, mean, [])
        assert (pr - rec["frames_pos"][f]).abs().max() < 2e-5, f
        assert (cr - rec["frames_cov"][f]).abs().max() < 1e-6
        s.p2g2p_n(20, 1e-4)
    assert (rec["frames_pos"][2] - rec["frames_pos"][0]).abs().max() > 1e-5           # the filled solid falls
    # without a filling block: the Gaussians only, as before
    plain = drv.run_physics_simulation(SD.Scene(**dict(sc.__dict__, particle_filling=None)), cloud)
    assert plain["n_particles"] == plain["n_gaussians"] == n_gs
    with pytest.raises(ValueError):
        drv.run_physics_simulation(SD.Scene(**dict(sc.__dict__, opacity=None)), cloud)
    with pytest.raises(NotImplementedError):
        drv.run_physics_simulation(SD.Scene(**dict(sc.__dict__, particle_filling=dict(filling, smooth=True, visualize=True))), cloud)
