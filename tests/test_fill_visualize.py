"""`particle_filling.visualize` and `sim_area` (gs_simulation.py:419-481, 602-606; filling.py:383-446).

CPU: the numpy oracle of the nearest-Gaussian search against the reference's own `get_attr_from_closest` /
`init_filled_particles` (tests/golden/fill_visualize_golden.npz, made by tests/golden/make_fill_visualize_golden.py) and
against a literal float32 brute force; argument checks, the exported symbol, a spill-free build, Scene defaults.
GPU: the device search against the fixture and the oracle (config-size shell, deep traversal, index ties, degenerate
boxes, non-finite Gaussians, no neighbour), determinism, and the scene driver with `visualize` and `sim_area` against the
same chain run by hand."""
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

from oracle import fill_visualize_ref as R  # noqa: E402

GOLDEN = os.path.join(HERE, "golden", "fill_visualize_golden.npz")
CASES = ["shell", "cups", "dup", "mirror", "sqrt", "exact", "far", "one"]
F32 = np.float32


@pytest.fixture(scope="module")
def golden():
    """The fixture's arrays; the shell / cups cases take their Gaussians and queries from filling_golden.npz (the
    Gaussians and filled particles of those scenes, every other one for the shell), as the generator does."""
    g = dict(np.load(GOLDEN))
    filling = np.load(os.path.join(HERE, "golden", "filling_golden.npz"))
    for name in ("shell", "cups"):
        pos = filling[f"{name}/pos"]
        new = filling[f"{name}/out"][len(pos):]
        g[f"{name}/pos"], g[f"{name}/new_pos"] = pos, (new[::2] if name == "shell" else new)
    return g


def check_outputs(out, g):
    """init_filled_particles' three outputs: the inputs first, then the reference's appended rows, bit for bit."""
    n = len(g["pos"])
    for got, x, want in zip(out, (g["shs"], g["opacity"], g["cov"]), (g["out_shs"], g["out_opacity"], g["out_cov"])):
        got = np.asarray(got)
        assert got.shape == (n + len(want),) + want.shape[1:]
        assert np.array_equal(bits(got[:n]), bits(x)) and np.array_equal(bits(got[n:]), bits(want))


def bits(a):
    return np.ascontiguousarray(a, F32).view(np.uint32)


def brute(pos, query, chunk=256):
    """get_attr_from_closest's loop, literally: float32 d of every pair, the first index of the smallest d < 1e10, else -1."""
    pos, query = np.asarray(pos, F32), np.asarray(query, F32)
    out = np.full(len(query), -1, np.int32)
    if len(pos) == 0:
        return out
    for s in range(0, len(query), chunk):
        d = R.nearest_dist_f32(query[s:s + chunk, None, :], pos[None, :, :])
        d = np.where(d < F32(1e10), d, np.inf)                    # NaN and d >= 1e10 never win
        j = np.argmin(d, axis=1)                                  # first occurrence: the lowest index
        ok = np.isfinite(d[np.arange(len(j)), j])
        out[s:s + chunk] = np.where(ok, j, -1)
    return out


def tie_counts(pos, query, index):
    """(queries whose winner has an equal-d rival at the same position, ... at another position)."""
    same = other = 0
    for q, i in zip(query, index):
        if i < 0:
            continue
        d = R.nearest_dist_f32(q, pos)
        rivals = np.nonzero(d == d[i])[0]
        rivals = rivals[rivals != i]
        assert np.all(rivals > i)
        if len(rivals):
            at = np.all(pos[rivals] == pos[i], axis=1)
            same += int(at.any())
            other += int((~at).any())
    return same, other


# ------------------------------------------------------------------------------------------------------------------ clouds
def cloud(kind, n, m, seed):
    rng = np.random.default_rng(seed)
    if kind == "random":
        pos = rng.uniform(0, 2, (n, 3))
        q = rng.uniform(-0.2, 2.2, (m, 3))
    elif kind == "clustered":
        c = rng.uniform(0, 2, (12, 3))
        pos = c[rng.integers(0, 12, n)] + rng.standard_normal((n, 3)) * 10.0 ** rng.uniform(-4, -1, (n, 1))
        q = rng.uniform(0, 2, (m, 3))
    elif kind == "duplicates":
        sites = rng.uniform(0, 2, (50, 3))
        pos = sites[rng.integers(0, 50, n)]
        q = np.concatenate([rng.uniform(0, 2, (m - 50, 3)), sites])
    elif kind == "collinear":
        t = rng.uniform(0, 2, n)
        pos = np.stack([t, 0.5 + 0 * t, 1.25 + 0 * t], axis=1)
        q = np.stack([rng.uniform(-0.5, 2.5, m), rng.uniform(0, 1, m), rng.uniform(1, 1.5, m)], axis=1)
    elif kind == "mirror":
        c = rng.integers(32, 96, (n // 2, 3)) / 64.0
        e = np.eye(3)[rng.integers(0, 3, n // 2)] * (rng.integers(1, 24, n // 2) / 64.0)[:, None]
        pos = np.stack([c - e, c + e], axis=1).reshape(-1, 3)
        pos = pos[rng.permutation(len(pos))]
        off = rng.integers(-40, 40, (n // 2, 3)) / 256.0 * (e == 0)
        q = (c + off)[:m]
    else:
        raise KeyError(kind)
    return pos.astype(F32), q.astype(F32)


# ------------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference_kernel(golden, name):
    g = {k: golden[f"{name}/{k}"] for k in ("pos", "shs", "opacity", "cov", "new_pos", "index", "out_shs", "out_opacity", "out_cov")}
    assert np.array_equal(R.nearest_index(g["pos"], g["new_pos"]), g["index"])
    check_outputs(R.init_filled_particles(g["pos"], g["shs"], g["cov"], g["opacity"], g["new_pos"]), g)
    assert np.array_equal(brute(g["pos"], g["new_pos"]), g["index"])


def test_fixture_covers_ties_and_sh_widths(golden):
    assert sorted({golden[f"{k}/shs"].shape[1] for k in CASES}) == [1, 4, 9, 16]
    same = other = 0
    for k in ("dup", "mirror", "sqrt"):
        a, b = tie_counts(golden[f"{k}/pos"], golden[f"{k}/new_pos"], golden[f"{k}/index"])
        same, other = same + a, other + b
    assert same >= 20 and other >= 20, (same, other)
    # the sqrt case ties on d with distinct float32 squares
    p, q, idx = golden["sqrt/pos"], golden["sqrt/new_pos"], golden["sqrt/index"]
    hits = 0
    for qq, i in zip(q, idx):
        dd = (q.dtype.type(0) + (qq - p)) ** 2
        s = (dd[:, 0] + dd[:, 1]) + dd[:, 2]
        d = np.sqrt(s)
        hits += int(np.any((d == d[i]) & (s != s[i])))
    assert hits >= 5, hits
    e = golden["exact/pos"]
    assert np.sum(R.nearest_dist_f32(golden["exact/new_pos"], e[golden["exact/index"]]) == 0) >= 300
    assert golden["one/pos"].shape[0] == 1 and np.all(golden["one/index"] == 0)
    far = golden["far/new_pos"]
    assert np.all(np.abs(far - 1.0).max(axis=1) > 50)


@pytest.mark.parametrize("kind", ["random", "clustered", "duplicates", "collinear", "mirror"])
@pytest.mark.parametrize("n,m", [(1, 50), (37, 300), (3000, 1500), (20000, 4000)])
def test_oracle_matches_brute_force(kind, n, m):
    if kind == "mirror" and n < 2:
        n = 2
    pos, q = cloud(kind, n, m, seed=n + m)
    assert np.array_equal(R.nearest_index(pos, q), brute(pos, q))


def test_oracle_non_finite_and_far():
    pos, q = cloud("random", 500, 200, seed=3)
    pos[::7, 1] = np.nan
    pos[3::11, 2] = np.inf
    pos[5::13, 0] = -np.inf
    q[::10] = np.nan
    q[1::10] = 3e10
    q[2::10, 2] = np.inf
    want = brute(pos, q)
    assert np.array_equal(R.nearest_index(pos, q), want)
    assert np.all(want[::10] == -1) and np.all(want[1::10] == -1) and np.all(want[2::10] == -1)
    assert np.all(R.nearest_index(np.zeros((0, 3), F32), q) == -1)
    with pytest.raises(ValueError, match="60"):
        R.init_filled_particles(pos, np.zeros((500, 1, 3)), np.zeros((500, 6)), np.zeros((500, 1)), q)


def test_init_filled_particles_argument_checks():
    from pixie_b200 import _lib
    from pixie_b200.particle_filling import init_filled_particles, nearest_gaussian
    p, s, c, o, q = torch.zeros(4, 3), torch.zeros(4, 16, 3), torch.zeros(4, 6), torch.ones(4, 1), torch.zeros(5, 3)
    with pytest.raises(ValueError):
        init_filled_particles(p[:, :2], s, c, o, q)
    with pytest.raises(ValueError):
        init_filled_particles(p, torch.zeros(4, 5, 3), c, o, q)                   # K not a square of 1..4
    with pytest.raises(ValueError):
        init_filled_particles(p, torch.zeros(4, 48), c, o, q)
    with pytest.raises(ValueError):
        init_filled_particles(p, s[:3], c, o, q)
    with pytest.raises(ValueError):
        init_filled_particles(p, s, c[:, :5], o, q)
    with pytest.raises(ValueError):
        init_filled_particles(p, s, c, o[:3], q)
    with pytest.raises(ValueError):
        init_filled_particles(p, s, c, o, q[:, :2])
    with pytest.raises(_lib.PixieError):
        init_filled_particles(p, s, c, o, q)                                       # CPU tensors: no fallback
    with pytest.raises(_lib.PixieError):
        nearest_gaussian(p, q)


def test_library_exports_nearest_symbol(built_lib):
    assert hasattr(built_lib, "pixie_nearest_gaussian")


def test_nearest_kernels_do_not_spill(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    src = os.path.join(ROOT, "pixie_b200", "csrc", "nearest.cu")
    res = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-c", src,
                          "-o", str(tmp_path / "nearest.o")], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    assert "query_kernel" in res.stderr
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", res.stderr)
    assert len(spills) >= 6
    assert all(s == ("0", "0") for s in spills), res.stderr


def test_scene_defaults_leave_visualize_and_sim_area_off():
    from pixie_b200 import scene_driver as SD
    from pixie_b200.particle_filling import decode_filling_params
    sc = SD.Scene(name="x", grid=None, mask=None, min_bounds=[0] * 3, max_bounds=[1] * 3, particles=torch.zeros(1, 3))
    assert sc.sim_area is None and sc.particle_filling is None
    assert decode_filling_params({}, {"n_grid": 32})["visualize"] is False


# ------------------------------------------------------------------------------------------------------------------ GPU
def _dev(x, dev):
    return torch.from_numpy(np.ascontiguousarray(x)).to(dev)


def device_index(pos, q, dev):
    from pixie_b200.particle_filling import nearest_gaussian
    return nearest_gaussian(_dev(pos, dev), _dev(q, dev)).cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_device_matches_reference_kernel(built_lib, cuda_dev, golden, name):
    from pixie_b200.particle_filling import init_filled_particles
    g = {k: golden[f"{name}/{k}"] for k in ("pos", "shs", "opacity", "cov", "new_pos", "index", "out_shs", "out_opacity", "out_cov")}
    assert np.array_equal(device_index(g["pos"], g["new_pos"], cuda_dev), g["index"])
    out = init_filled_particles(*[_dev(g[k], cuda_dev) for k in ("pos", "shs", "cov", "opacity", "new_pos")])
    assert all(t.dtype == torch.float32 and t.device == torch.device(cuda_dev) for t in out)
    check_outputs([t.cpu().numpy() for t in out], g)


def shell_fill(n, seed, dev):
    """A config-size scene: an n-Gaussian shell (radius 0.45 around (1, 1, 1)) filled at n_grid 100 over [0.4, 1.6]^3."""
    from pixie_b200 import particle_filling as PF
    rng = np.random.default_rng(seed)
    v = rng.standard_normal((n, 3))
    pos = (1.0 + 0.45 * (1 + 0.02 * rng.standard_normal((n, 1))) * v / np.linalg.norm(v, axis=1, keepdims=True)).astype(F32)
    s = rng.uniform(0.004, 0.012, (n, 3))
    cov = np.zeros((n, 6), F32)
    cov[:, 0], cov[:, 3], cov[:, 5] = s[:, 0] ** 2, s[:, 1] ** 2, s[:, 2] ** 2
    opacity = rng.uniform(0.3, 1.0, (n, 1)).astype(F32)
    p, o, c = _dev(pos, dev), _dev(opacity, dev), _dev(cov, dev)
    full = PF.fill_particles(p, o, c, 100, 2_000_000, 0.012, density_thres=2.0, search_thres=1.0, search_exclude_dir=2, ray_cast_dir=4,
                             boundary=[0.4, 1.6, 0.4, 1.6, 0.4, 1.6])
    return pos, opacity, cov, full[n:].cpu().numpy()


@pytest.mark.gpu
def test_device_matches_oracle_on_config_size_shell(built_lib, cuda_dev):
    pos, _, _, new = shell_fill(300_000, 7, cuda_dev)
    assert len(new) > 100_000
    got = device_index(pos, new, cuda_dev)
    want = R.nearest_index(pos, new)
    assert np.all(want >= 0)
    assert np.array_equal(got, want)


def _deep_cluster(rng):
    pos = (np.array([1.0, 1.0, 1.0]) + rng.standard_normal((100_000, 3)) * 1e-3).astype(F32)
    v = rng.standard_normal((20_000, 3))
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    return pos, (1.0 + v * 10.0 ** rng.uniform(-1, 3, (20_000, 1))).astype(F32)


def _three_sites(rng):
    sites = np.array([[0.5, 0.5, 0.5], [1.5, 0.5, 1.0], [1.0, 1.5, 1.5]], F32)
    return sites[rng.integers(0, 3, 10_000)], np.concatenate([rng.uniform(0, 2, (5000, 3)), sites]).astype(F32)


def _line(rng):
    t = rng.uniform(0, 2, 50_000)
    pos = np.stack([t, np.full_like(t, 0.75), np.full_like(t, 1.25)], axis=1).astype(F32)
    pos[:500] = pos[500:1000]                                                 # duplicates on the line too
    return pos, np.stack([rng.uniform(-0.5, 2.5, 20_000), rng.uniform(0, 1.5, 20_000), np.full(20_000, 1.25)], axis=1).astype(F32)


def _non_finite(rng):
    pos = rng.uniform(0, 2, (40_000, 3)).astype(F32)
    pos[::9, 0] = np.nan
    pos[4::17, 1] = np.inf
    pos[7::23, 2] = -np.inf
    pos[8::31] = np.array([3e38, -3e38, 3e38], F32)                          # finite, but every d overflows to Inf
    return pos, rng.uniform(-0.5, 2.5, (20_000, 3)).astype(F32)


def _mirror(rng):
    return cloud("mirror", 40_000, 20_000, 5)


@pytest.mark.gpu
@pytest.mark.parametrize("make", [_deep_cluster, _three_sites, _line, _non_finite, _mirror], ids=lambda f: f.__name__[1:])
def test_device_matches_oracle(built_lib, cuda_dev, make):
    pos, q = make(np.random.default_rng(11))
    got = device_index(pos, q, cuda_dev)
    assert np.array_equal(got, R.nearest_index(pos, q))
    assert np.all(got >= 0)
    sub = np.random.default_rng(1).choice(len(q), 300, replace=False)        # and the literal loop on a sample
    assert np.array_equal(got[sub], brute(pos, q[sub]))


@pytest.mark.gpu
def test_device_no_neighbour(built_lib, cuda_dev):
    from pixie_b200 import _lib
    from pixie_b200.particle_filling import init_filled_particles
    rng = np.random.default_rng(2)
    pos = rng.uniform(0, 2, (1000, 3)).astype(F32)
    q = rng.uniform(0, 2, (400, 3)).astype(F32)
    q[::10] = np.nan
    q[1::10] = F32(2e10)
    q[2::10, 1] = -np.inf
    q[3::10] = pos[3::10][:40] + np.array([0, 0, 1e10], F32)                # d >= 1e10 exactly: not < 1e10
    got = device_index(pos, q, cuda_dev)
    want = brute(pos, q)
    assert np.array_equal(got, want) and np.array_equal(got, R.nearest_index(pos, q))
    assert np.sum(got == -1) == 160
    assert np.all(device_index(np.zeros((0, 3), F32), q, cuda_dev) == -1)
    assert device_index(pos, np.zeros((0, 3), F32), cuda_dev).shape == (0,)
    args = [_dev(pos, cuda_dev), torch.zeros(1000, 4, 3, device=cuda_dev), torch.zeros(1000, 6, device=cuda_dev),
            torch.ones(1000, 1, device=cuda_dev)]
    with pytest.raises(_lib.PixieError, match="160 of 400"):
        init_filled_particles(*args, _dev(q, cuda_dev))
    s, o, c = init_filled_particles(*args, torch.zeros(0, 3, device=cuda_dev))
    assert s.shape == (1000, 4, 3) and o.shape == (1000, 1) and c.shape == (1000, 6)


@pytest.mark.gpu
def test_device_is_deterministic_and_permutation_equivariant(built_lib, cuda_dev):
    from pixie_b200.particle_filling import nearest_gaussian
    pos, q = cloud("duplicates", 60_000, 30_000, 9)
    p, qd = _dev(pos, cuda_dev), _dev(q, cuda_dev)
    a = nearest_gaussian(p, qd)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        b = nearest_gaussian(p, qd)
    torch.cuda.current_stream().wait_stream(side)
    assert torch.equal(a, b) and torch.equal(a, nearest_gaussian(p, qd))
    perm = torch.randperm(len(q), generator=torch.Generator().manual_seed(0)).to(cuda_dev)
    assert torch.equal(nearest_gaussian(p, qd[perm]), a[perm])


# ------------------------------------------------------------------------------------------------------------------ scene driver
def _driver(dev):
    from oracle import unet_ref as O
    from pixie_b200 import material_transfer as MT
    from pixie_b200 import scene_driver as SD
    C, G = 64, 16
    seg, reg = O.build_pair(C, G, seed=3)
    drv = SD.SceneBatchDriver(feature_channels=C, grid_size=G, device=dev, seg_state_dict=seg.state_dict(), cont_state_dict=reg.state_dict(),
                              **O.DEFAULT_CFG)
    rng = np.random.default_rng(4)
    K = 8
    pred = np.zeros((3 + K, G, G, G), F32)
    pred[:3] = rng.uniform(-0.2, 0.2, size=(3, G, G, G))
    pred[3 + rng.integers(0, K, size=(G, G, G)), np.arange(G)[:, None, None], np.arange(G)[None, :, None], np.arange(G)[None, None, :]] = 1.0
    ranges = dict(density_min=2.95, density_max=3.05, E_min=4.4, E_max=4.6, nu_min=0.29, nu_max=0.31)
    cloud_ = MT.extract_material_points(torch.from_numpy(pred).to(dev), torch.ones((G, G, G)).to(dev), [-0.5] * 3, [0.5] * 3, ranges)
    return drv, cloud_


ROT_Z = torch.tensor([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])        # exact in float32: rotated x = -y
CAMERA = {"default_camera_index": -1, "init_azimuthm": 30.0, "init_elevation": 10.0, "init_radius": 2.0, "move_camera": True,
          "delta_a": 5.0, "delta_e": 1.0, "delta_r": 0.02, "mpm_space_vertical_upward_axis": [0, 0, 1]}
CAMERAS = [{"width": 320, "height": 240, "position": [0.0, 0.0, 0.0], "rotation": np.eye(3).tolist(), "fx": 280.0, "fy": 280.0}]
MP = {"n_grid": 32, "grid_lim": 2.0, "material": "jelly", "g": [0.0, 0.0, -9.8], "density": 1000.0, "E": 1e5, "nu": 0.3}
TP = {"substep_dt": 1e-4, "frame_dt": 2e-3, "frame_num": 3}


def two_shells(rng, n):
    """A shell (radius 0.3 around (0, -0.1, 0), the simulated object) and a flat slab of n // 3 Gaussians at y in
    [0.3, 0.45] beside it, in the Gaussians' frame (inside the material cloud's [-0.5, 0.5]^3); SH degree 3."""
    v = rng.standard_normal((n, 3))
    shell = np.array([0.0, -0.1, 0.0]) + 0.3 * v / np.linalg.norm(v, axis=1, keepdims=True)
    slab = np.stack([rng.uniform(-0.45, 0.45, n // 3), rng.uniform(0.3, 0.45, n // 3), rng.uniform(-0.45, 0.45, n // 3)], axis=1)
    pos = np.concatenate([shell, slab]).astype(F32)
    pos[0] = [0.1, 0.25, 0.0]                                                 # rotated x = -0.25: exactly on the crop plane
    k = len(pos)
    s = rng.uniform(0.01, 0.02, (k, 3))
    cov = np.zeros((k, 6), F32)
    cov[:, 0], cov[:, 1], cov[:, 3], cov[:, 5] = s[:, 0] ** 2, 1e-5, s[:, 1] ** 2, s[:, 2] ** 2
    return pos, rng.uniform(0.3, 1.0, (k, 1)).astype(F32), cov, (rng.standard_normal((k, 16, 3)) * 0.4).astype(F32)


FILLING = {"n_grid": 40, "density_threshold": 0.5, "search_threshold": 0.2, "max_particles_num": 2000000}
AREA = [-0.25, 0.5, -0.5, 0.5, -0.5, 0.5]                                     # the shell, not the slab (rotated x = -y)


def by_hand(dev, cloud_, pos, opacity, cov, shs, rots, filling, sim_area, visualize):
    """gs_simulation.py's chain written out: crop, centre, fill, init_filled_particles, solver, kNN, then per frame the
    export and the render inputs (simulated particles, then the unselected Gaussians)."""
    from pixie_b200 import frame_export as FE
    from pixie_b200 import gs_render as GR
    from pixie_b200 import material_transfer as MT
    from pixie_b200 import particle_filling as PF
    from pixie_b200 import scene_driver as SD
    from pixie_b200.mpm_solver_warp import MPM_Simulator_WARP
    rots = [r.to(dev) for r in rots]
    p, o, c, s = _dev(pos, dev), _dev(opacity, dev), _dev(cov, dev), _dev(shs, dev)
    rotated = SD.apply_rotations(p, rots)
    unsel = None
    if sim_area is not None:
        mask = torch.ones(len(pos), dtype=torch.bool, device=dev)
        for i in range(3):
            mask &= (rotated[:, i] > sim_area[2 * i]) & (rotated[:, i] < sim_area[2 * i + 1])
        unsel = (p[~mask], c[~mask], o[~mask], s[~mask])
        rotated, c, o, s = rotated[mask], c[mask], o[mask], s[mask]
    t, scale, mean = SD.transform2origin(rotated)
    pos0 = t + torch.tensor([1.0, 1.0, 1.0], device=dev)
    cov0 = rotate_cov(c, rots, dev) * (scale ** 2)
    n = len(pos0)
    fp = PF.decode_filling_params(filling, {"n_grid": 32})
    full = PF.fill_particles(pos0, o, cov0, fp["n_grid"], fp["max_particles_num"], 2.0 / fp["n_grid"], fp["density_threshold"],
                             fp["search_threshold"], 1, 5, 4, None)
    if visualize:
        s_r, o_r, cov_full = PF.init_filled_particles(full[:n], s, cov0, o, full[n:])
        n_r = len(full)
    else:
        cov_full = torch.zeros((len(full), 6), device=dev)
        cov_full[:n] = cov0
        s_r, o_r, n_r = s, o, n
    sol = MPM_Simulator_WARP(10, device=dev)
    sol.load_initial_data_from_torch(full, FE.get_particle_volume(full, 32, 2.0 / 32), cov_full, n_grid=32, grid_lim=2.0, device=dev)
    sol.set_parameters_dict(dict(MP), device=dev)
    sol.add_bounding_box()
    q, _ = FE.render_frame_transform(sol.export_particle_x_to_torch(), None, 0.0, scale, mean, rots)
    props = MT.perform_knn_smoothing(q, cloud_, 10, 0.2)
    MT.apply_material_properties_to_solver(sol, props[1], props[2], props[3], props[4], device=dev, exact_box_semantics=False)
    cp = GR.decode_camera_params(CAMERA)
    vc, oc = GR.get_center_view_worldspace_and_observant_coordinate(cp["mpm_space_viewpoint_center"], cp["mpm_space_vertical_upward_axis"],
                                                                   rots, scale, mean)
    frames = []
    for f in range(3):
        x, cx = sol.export_particle_x_to_torch(), sol.export_particle_cov_to_torch().view(-1, 6)
        pr, cr = FE.render_frame_transform(x[:n_r], cx[:n_r], 0.0, scale, mean, rots)
        cam = GR.get_camera_view(CAMERAS, -1, vc, oc, False, 30.0, 10.0, 2.0, None, True, f, 5.0, 1.0, 0.02)
        frames.append((pr, cr, cam))
        sol.p2g2p_n(20, 1e-4)
    return dict(frames=frames, shs=s_r, opacity=o_r.reshape(-1), n=n, n_r=n_r, n_full=len(full), unsel=unsel, cov_full=cov_full)


def render_inputs(h, f, pos, cov):
    """The rasterize arguments of frame f for the simulated frame (pos, cov): the unselected Gaussians appended."""
    op, shs = h["opacity"], h["shs"]
    if h["unsel"] is not None:
        up, uc, uo, us = h["unsel"]
        pos, cov, op, shs = torch.cat([pos, up]), torch.cat([cov, uc]), torch.cat([op, uo.reshape(-1)]), torch.cat([shs, us])
    return pos, cov, op, shs


def rotate_cov(c, rots, dev):
    """apply_cov_rotations (gs_simulation.py:438): R C R^T per rotation, in the driver's operation order."""
    m = torch.stack([c[:, 0], c[:, 1], c[:, 2], c[:, 1], c[:, 3], c[:, 4], c[:, 2], c[:, 4], c[:, 5]], dim=1).view(-1, 3, 3)
    for Rm in rots:
        Rm = Rm.to(dev)
        m = Rm @ m @ Rm.T
    return torch.stack([m[:, 0, 0], m[:, 0, 1], m[:, 0, 2], m[:, 1, 1], m[:, 1, 2], m[:, 2, 2]], dim=1)


def clear_of(density, thr):
    """A threshold near `thr` that no cell density lies within 1e-5 (relative) of, so that the float atomics' order of the
    splat cannot flip a cell between two runs."""
    for k in range(1000):
        t = thr * (1 + 3e-5 * k)
        if not np.any(np.abs(density.astype(np.float64) - t) <= 1e-5 * t):
            return t
    raise AssertionError("no clear threshold")


def clear_filling(dev, pos, opacity, cov, rots, sim_area, visualize):
    """FILLING with thresholds moved clear of every cell density of this scene's fill grid."""
    from pixie_b200 import particle_filling as PF
    from pixie_b200 import scene_driver as SD
    p, o, c = _dev(pos, dev), _dev(opacity, dev), _dev(cov, dev)
    rotated = SD.apply_rotations(p, [r.to(dev) for r in rots])
    if sim_area is not None:
        mask = torch.ones(len(pos), dtype=torch.bool, device=dev)
        for i in range(3):
            mask &= (rotated[:, i] > sim_area[2 * i]) & (rotated[:, i] < sim_area[2 * i + 1])
        rotated, o, c = rotated[mask], o[mask], c[mask]
    t, scale, _ = SD.transform2origin(rotated)
    _, dens = PF.densify_grids(t + 1.0, o, rotate_cov(c, rots, dev) * scale ** 2, FILLING["n_grid"], 2.0 / FILLING["n_grid"])
    dens = dens.cpu().numpy()
    return dict(FILLING, density_threshold=clear_of(dens, FILLING["density_threshold"]),
                search_threshold=clear_of(dens, FILLING["search_threshold"]), visualize=visualize)


def check_driver(monkeypatch, dev, visualize, sim_area, rots):
    from pixie_b200 import gs_render as GR
    from pixie_b200 import scene_driver as SD
    drv, cloud_ = _driver(dev)
    pos, opacity, cov, shs = two_shells(np.random.default_rng(6), 6000)
    filling = clear_filling(dev, pos, opacity, cov, rots, sim_area, visualize)
    seen = []
    real = GR.rasterize
    monkeypatch.setattr(GR, "rasterize", lambda *a, **kw: (seen.append((a, kw)), real(*a, **kw))[1])
    sc = SD.Scene(name="obj", grid=None, mask=None, min_bounds=[-0.5] * 3, max_bounds=[0.5] * 3, particles=torch.from_numpy(pos),
                  cov=torch.from_numpy(cov), opacity=torch.from_numpy(opacity), material_params=dict(MP), bc_params=[{"type": "bounding_box"}],
                  time_params=TP, nn_distance_threshold=0.2, particle_filling=filling, sim_area=sim_area, rotation_matrices=rots,
                  shs=torch.from_numpy(shs), sh_degree=3, camera_params=CAMERA, cameras=CAMERAS)
    rec = drv.run_physics_simulation(sc, cloud_)
    h = by_hand(dev, cloud_, pos, opacity, cov, shs, rots, filling, sim_area, visualize)
    assert rec["n_particles"] == h["n_full"] and rec["n_gaussians"] == h["n"] and rec["n_filled"] == h["n_full"] - h["n"] > 500
    assert rec["n_unselected"] == (0 if h["unsel"] is None else len(h["unsel"][0]))
    assert len(rec["frames_rgb"]) == 3 and len(seen) == 3
    for f, (pr, cr, cam) in enumerate(h["frames"]):
        assert rec["frames_pos"][f].shape == (h["n_r"], 3) and rec["frames_cov"][f].shape == (h["n_r"], 6)
        assert (pr - rec["frames_pos"][f]).abs().max() < 2e-5, f
        assert (cr - rec["frames_cov"][f]).abs().max() < 1e-6, f
        # the driver's render inputs: its own frame, then the unselected Gaussians bit for bit; the by-hand attributes
        a, kw = seen[f]
        p_in, c_in, o_in, s_in = render_inputs(h, f, rec["frames_pos"][f], rec["frames_cov"][f])
        assert torch.equal(a[0], p_in) and torch.equal(a[1], c_in) and torch.equal(a[2], o_in) and torch.equal(kw["shs"], s_in)
        img, _ = real(p_in, c_in, o_in, cam, [0, 0, 0], shs=s_in, sh_degree=3)
        assert torch.equal(img, rec["frames_rgb"][f]), f
    return rec, h


@pytest.mark.gpu
def test_scene_driver_visualize(built_lib, cuda_dev, monkeypatch):
    rec, h = check_driver(monkeypatch, cuda_dev, True, None, [])
    n = h["n"]
    assert h["n_r"] == rec["n_particles"]
    # the filled particles carry their nearest Gaussian's (scaled) covariance: exported non-zero
    assert bool((rec["frames_cov"][0][n:].abs().sum(dim=1) > 0).all())


@pytest.mark.gpu
def test_scene_driver_sim_area(built_lib, cuda_dev, monkeypatch):
    pos, _, _, _ = two_shells(np.random.default_rng(6), 6000)
    rotated = pos @ ROT_Z.numpy().T
    keep = np.ones(len(pos), bool)
    for i in range(3):
        keep &= (rotated[:, i] > F32(AREA[2 * i])) & (rotated[:, i] < F32(AREA[2 * i + 1]))
    assert rotated[0, 0] == F32(-0.25) and not keep[0]                       # on the plane: unselected
    rec, h = check_driver(monkeypatch, cuda_dev, False, AREA, [ROT_Z])
    assert rec["n_unselected"] == int((~keep).sum()) >= 2000 and rec["n_gaussians"] == int(keep.sum())
    assert torch.equal(h["unsel"][0].cpu(), torch.from_numpy(pos[~keep]))


@pytest.mark.gpu
def test_scene_driver_sim_area_with_visualize(built_lib, cuda_dev, monkeypatch):
    rec, h = check_driver(monkeypatch, cuda_dev, True, AREA, [ROT_Z])
    assert rec["n_unselected"] > 0 and h["n_r"] == rec["n_particles"]
    assert bool((rec["frames_cov"][0][h["n"]:].abs().sum(dim=1) > 0).all())


@pytest.mark.gpu
def test_scene_driver_sim_area_rejects_empty_selection(built_lib, cuda_dev):
    from pixie_b200 import scene_driver as SD
    drv, cloud_ = _driver(cuda_dev)
    pos, opacity, cov, shs = two_shells(np.random.default_rng(6), 600)
    sc = SD.Scene(name="obj", grid=None, mask=None, min_bounds=[-0.5] * 3, max_bounds=[0.5] * 3, particles=torch.from_numpy(pos),
                  cov=torch.from_numpy(cov), opacity=torch.from_numpy(opacity), material_params=dict(MP), time_params=TP,
                  sim_area=[5, 6, 5, 6, 5, 6])
    with pytest.raises(ValueError):
        drv.run_physics_simulation(sc, cloud_)
    # visualize without SH
    with pytest.raises(ValueError):
        drv.run_physics_simulation(SD.Scene(**dict(sc.__dict__, sim_area=None, particle_filling=dict(FILLING, visualize=True))), cloud_)
    # without rendering, sim_area still crops the simulation
    rec = drv.run_physics_simulation(SD.Scene(**dict(sc.__dict__, sim_area=AREA, shs=torch.from_numpy(shs))), cloud_)
    assert rec["n_unselected"] > 0 and rec["n_gaussians"] == len(pos) - rec["n_unselected"] and "frames_rgb" not in rec
    assert rec["frames_pos"][0].shape == (rec["n_gaussians"], 3)
