"""Ground and stationary-cluster boundary conditions of the material-field hand-off (PG/material_field.py:296-550).

tests/golden/stationary_golden.npz was written by executing the reference's own `handle_stationary_clusters`, `fix_to_ground`
and `apply_material_field_to_simulation` (tests/golden/make_stationary_golden.py). CPU: the numpy / scikit-learn oracle
(tests/stationary_ref.py) and the product's `fix_to_ground` reproduce it bit-exactly. GPU (`-m gpu`): the device DBSCAN
(csrc/cluster.cu) through pixie_b200.material_transfer reproduces the labels, BC dicts and solver colliders bit-exactly, and
the whole hand-off matches the reference's upload."""
import json
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import stationary_ref as R  # noqa: E402

G = np.load(os.path.join(HERE, "golden", "stationary_golden.npz"))
STATIONARY = ["mixed_largest", "mixed_all", "mixed_defaults", "all_noise", "none"]
GROUND = ["ground_driver", "ground_defaults", "ground_p5"]


def _bcs(name):
    return json.loads(str(G[f"{name}/bcs"]))


def _kwargs(name):
    return json.loads(str(G[f"{name}/kwargs"]))


def _plain(bcs):
    """BC dicts with numpy scalars as Python numbers (values unchanged: float32 -> float64 is exact)."""
    conv = lambda v: [conv(x) for x in v] if isinstance(v, (list, tuple)) else (float(v) if isinstance(v, (float, np.floating)) else v)
    return [{k: conv(v) for k, v in bc.items()} for bc in bcs]


def _solver_colliders(solver):
    rows = [R.collider_row(list(c.point), list(c.size), list(c.velocity), c.start_time, c.end_time, c.reset) for c in solver.collider_params]
    return np.stack(rows) if rows else np.zeros((0, 12), np.float32)


# ------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("name", STATIONARY)
def test_oracle_stationary_clusters_bit_exact(name):
    s = R.RecordingSolver()
    x, ids = G[f"{name}/x"], G[f"{name}/ids"]
    got = R.handle_stationary_clusters(s, x, ids, **_kwargs(name))
    assert _plain(got) == _bcs(name)
    want = G[f"{name}/colliders"]
    assert np.array_equal(np.stack(s.colliders) if s.colliders else np.zeros((0, 12), np.float32), want)
    if f"{name}/labels" in G:
        assert np.array_equal(R.dbscan_labels(x[ids == R.STATIONARY_ID], 0.03, _kwargs(name).get("min_samples", 10)), G[f"{name}/labels"])


def test_golden_covers_the_corner_cases():
    lab = G["mixed_all/labels"]
    sizes = [bc["cluster_size"] for bc in _bcs("mixed_all")]
    assert sorted(sizes)[-1] == sorted(sizes)[-2]                                  # a tie for the largest cluster ...
    assert _bcs("mixed_largest")[0]["cluster_id"] == min(i for i, s in enumerate(sizes) if s == max(sizes))   # ... goes to the smaller label
    assert 8 in sizes and (lab == -1).any()                                        # exactly min_samples; noise
    assert (G["mixed_all/ids"] != R.STATIONARY_ID).sum() > 50                      # interleaved non-stationary particles
    assert _bcs("all_noise") == [] and "all_noise/labels" in G and (G["all_noise/labels"] == -1).all()
    assert _bcs("none") == [] and "none/labels" not in G


@pytest.mark.parametrize("name", GROUND)
def test_fix_to_ground_on_cpu_tensors_matches_reference(name):
    from pixie_b200 import material_transfer as MT
    x = G[f"{name}/x"]
    for impl, pos in ((R.fix_to_ground, x), (MT.fix_to_ground, torch.from_numpy(x))):
        s = R.RecordingSolver()
        got = impl(s, pos, **_kwargs(name))
        assert _plain(got) == _bcs(name), impl
        assert np.array_equal(np.stack(s.colliders), G[f"{name}/colliders"]), impl
        assert [type(v) for v in got[0]["point"]] == [np.float32] * 3                # numpy float32 scalars, as the reference returns


def test_dbscan_without_device_raises():
    from pixie_b200 import _lib
    from pixie_b200 import material_transfer as MT
    with pytest.raises(_lib.PixieError):
        MT.dbscan(torch.zeros(10, 3), 0.03, 8)               # no device, or a CPU tensor: there is no CPU fallback
    with pytest.raises(ValueError):
        MT.dbscan(torch.zeros(10, 3), 0.0, 8)
    with pytest.raises(ValueError):
        MT.dbscan(torch.zeros(10, 3), 0.03, 0)


# ------------------------------------------------------------------------------------------------------- GPU
def _solver(dev, x=None, n_grid=16):
    from pixie_b200.mpm_solver_warp import MPM_Simulator_WARP
    s = MPM_Simulator_WARP(10, device=dev)
    if x is None:
        x = np.full((8, 3), 1.0, np.float32)
    s.load_initial_data_from_torch(torch.from_numpy(x).to(dev), torch.full((len(x),), 1e-5, device=dev), None, n_grid=n_grid, grid_lim=2.0,
                                   device=dev)
    return s


@pytest.mark.gpu
@pytest.mark.parametrize("name", STATIONARY)
def test_cuda_stationary_clusters_match_reference(built_lib, cuda_dev, name):
    from pixie_b200 import material_transfer as MT
    x, ids = G[f"{name}/x"], G[f"{name}/ids"]
    kw = _kwargs(name)
    xd, idd = torch.from_numpy(x).to(cuda_dev), torch.from_numpy(ids).to(cuda_dev)
    labels = MT.dbscan(xd, 0.03, kw.get("min_samples", 10), idd)
    if f"{name}/labels" in G:
        assert np.array_equal(labels.cpu().numpy(), G[f"{name}/labels"])
    else:
        assert labels.numel() == 0
    s = _solver(cuda_dev, x)
    got = MT.handle_stationary_clusters(s, xd, idd, **kw)
    assert _plain(got) == _bcs(name)
    assert np.array_equal(_solver_colliders(s), G[f"{name}/colliders"])
    assert s.n_bcs == len(got)


@pytest.mark.gpu
def test_cuda_apply_material_field_matches_reference(built_lib, cuda_dev):
    from pixie_b200 import material_transfer as MT
    dev = cuda_dev
    x = G["apply/x"]
    from pixie_b200.mpm_solver_warp import MPM_Simulator_WARP
    s = MPM_Simulator_WARP(10, device=dev)
    s.load_initial_data_from_torch(torch.from_numpy(x).to(dev), torch.from_numpy(G["apply/vol"]).to(dev), None, n_grid=16, grid_lim=2.0, device=dev)
    s.set_parameters_dict({"material": "jelly", "E": 1e5, "nu": 0.3, "density": 1000.0}, device=dev)
    params = {k: torch.from_numpy(np.ascontiguousarray(G[f"apply/field/{k}"])).to(dev)
              for k in ("pos", "part_labels", "material_id", "density", "E", "nu", "conf")}
    conf, bcs = MT.apply_material_field_to_simulation(s, params, dev, torch.from_numpy(G["apply/scale"]), torch.from_numpy(G["apply/mean"]),
                                                      [torch.from_numpy(r) for r in G["apply/rots"]])
    assert _plain(bcs) == _bcs("apply")
    assert np.array_equal(_solver_colliders(s), G["apply/colliders"])
    assert np.abs(conf.cpu().numpy() / G["apply/conf"] - 1).max() < 2e-6
    assert np.array_equal(s.mpm_state.particle_material.numpy(), G["apply/material"])
    for got, k in ((s.mpm_model.E.numpy(), "E"), (s.mpm_model.nu.numpy(), "nu"), (s.mpm_state.particle_density.numpy(), "density"),
                   (s.mpm_state.particle_mass.numpy(), "mass")):
        assert np.abs(got / G[f"apply/{k}"] - 1).max() < 2e-6, k


def _random_cloud(seed):
    """>= 200k float32 points: a surface shell, dense clumps (two of 5000 points inside one eps cell), sparse noise, far
    outliers (some forming a cluster), negative coordinates; interleaved with particles of other materials."""
    rng = np.random.default_rng(seed)
    d = rng.standard_normal((185_000, 3))
    shell = d / np.linalg.norm(d, axis=1, keepdims=True) * 0.6 + rng.normal(0, 0.004, size=(185_000, 3)) - 0.2
    clumps = [c + rng.uniform(-0.012, 0.012, size=(5000, 3)) for c in ([-0.5, 0.1, -0.3], [0.9, -0.7, 0.2])]
    small = [c + rng.normal(0, 0.01, size=(rng.integers(5, 60), 3)) for c in rng.uniform(-1.5, 1.5, size=(300, 3))]
    noise = rng.uniform(-2.0, 2.0, size=(3000, 3))
    far = np.concatenate([rng.uniform(-900, 900, size=(40, 3)), np.array([-613.0, 402.5, -77.25]) + rng.uniform(-0.01, 0.01, size=(15, 3))])
    stat = np.concatenate([shell, *clumps, *small, noise, far]).astype(np.float32)
    other = rng.uniform(-1, 1, size=(40_000, 3)).astype(np.float32)
    x = np.concatenate([stat, other])
    ids = np.concatenate([np.full(len(stat), 6, np.int32), rng.integers(0, 6, size=len(other)).astype(np.int32)])
    perm = rng.permutation(len(x))
    return x[perm].copy(), ids[perm].copy()


@pytest.mark.gpu
def test_cuda_dbscan_matches_sklearn_on_a_large_cloud(built_lib, cuda_dev):
    from pixie_b200 import material_transfer as MT
    x, ids = _random_cloud(3)
    sel = x[ids == 6]
    assert len(sel) >= 200_000
    want = R.dbscan_labels(sel, 0.03, 8)
    xd, idd = torch.from_numpy(x).to(cuda_dev), torch.from_numpy(ids).to(cuda_dev)
    a = MT.dbscan(xd, 0.03, 8, idd).cpu().numpy()
    b = MT.dbscan(xd, 0.03, 8, idd).cpu().numpy()
    assert np.array_equal(a, b)
    assert want.max() > 100 and (want == -1).sum() > 1000
    assert np.array_equal(a, want), f"{(a != want).sum()} labels differ"


@pytest.mark.gpu
def test_stationary_block_stays_in_place_under_gravity(built_lib, cuda_dev):
    from pixie_b200 import material_transfer as MT
    dev = cuda_dev
    n_grid, dx = 32, 2.0 / 32
    g = np.arange(0.0, 0.4, dx / 4) + 0.7 + dx / 8              # spacing dx / 4 < eps: every particle is core
    x = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3).astype(np.float32)
    deep = np.all((x > x.min(0) + 2 * dx) & (x < x.max(0) - 2 * dx), axis=1)
    assert deep.sum() > 100

    def run(bcs_on):
        s = _solver(dev, x, n_grid)
        s.set_parameters_dict({"material": "jelly", "E": 2e4, "nu": 0.3, "density": 1000.0, "g": [0.0, 0.0, -9.8]}, device=dev)
        s.add_bounding_box()
        ids = torch.full((len(x),), 6, dtype=torch.int32, device=dev)
        bcs = []
        if bcs_on:
            bcs = MT.handle_stationary_clusters(s, s.export_particle_x_to_torch(), ids, eps=0.03, min_samples=8, start_time=0.0, end_time=1e9,
                                                buffer=0.1)
        n = len(x)
        MT.apply_material_properties_to_solver(s, torch.full((n,), 1000.0, device=dev), torch.full((n,), 2e4, device=dev),
                                               torch.full((n,), 0.3, device=dev), ids, device=dev, exact_box_semantics=False)
        x0 = s.export_particle_x_to_torch().clone()
        s.p2g2p_n(200, 1e-4)
        return bcs, (s.export_particle_x_to_torch() - x0).cpu().numpy()

    bcs, moved = run(True)
    assert len(bcs) == 1 and bcs[0]["cluster_size"] == len(x)
    assert np.abs(moved[deep]).max() == 0.0
    _, fell = run(False)
    assert fell[:, 2].mean() < -1e-4


@pytest.mark.gpu
def test_too_many_clusters_raise_before_registering(built_lib, cuda_dev):
    from pixie_b200 import _lib
    from pixie_b200 import material_transfer as MT
    from pixie_b200.mpm_solver_warp import MAX_BCS
    rng = np.random.default_rng(5)
    centres = np.stack(np.meshgrid(*[np.arange(7) * 0.2 + 0.3] * 3, indexing="ij"), -1).reshape(-1, 3)     # 343 clumps
    x = np.concatenate([c + rng.uniform(-0.005, 0.005, size=(8, 3)) for c in centres]).astype(np.float32)
    s = _solver(cuda_dev, x)
    s.add_bounding_box()
    ids = torch.full((len(x),), 6, dtype=torch.int32, device=cuda_dev)
    assert len(centres) > MAX_BCS
    with pytest.raises(_lib.PixieError):
        MT.handle_stationary_clusters(s, torch.from_numpy(x).to(cuda_dev), ids, eps=0.03, min_samples=8, only_handle_largest_cluster=False)
    assert s.n_bcs == 1 and len(s.collider_params) == 1
    assert len(MT.handle_stationary_clusters(s, torch.from_numpy(x).to(cuda_dev), ids, eps=0.03, min_samples=8)) == 1


@pytest.mark.gpu
def test_scene_driver_material_field_bcs(built_lib, cuda_dev, tmp_path):
    from oracle import unet_ref as O
    from pixie_b200 import frame_export as FE
    from pixie_b200 import material_transfer as MT
    from pixie_b200 import scene_driver as SD
    from pixie_b200 import voxel_io as V
    from pixie_b200.mpm_solver_warp import MPM_Simulator_WARP
    from test_scene_driver import _scenes
    C, Gs, NP = 64, 16, 100_000                 # dense enough (about 10 particles within eps) for stationary clusters
    seg, reg = O.build_pair(C, Gs, seed=3)
    sc_off = _scenes(str(tmp_path), 1, C, Gs, NP)[0]
    sc_on = SD.Scene(**{**sc_off.__dict__, "name": "on", "material_field_bcs": True})
    ranges = dict(density_min=2.95, density_max=3.05, E_min=4.4, E_max=4.6, nu_min=0.29, nu_max=0.31)
    drv = SD.SceneBatchDriver(feature_channels=C, grid_size=Gs, device=cuda_dev, seg_state_dict=seg.state_dict(),
                              cont_state_dict=reg.state_dict(), ranges=ranges, **O.DEFAULT_CFG)
    cloud = drv.generate_neural_segmentation([sc_off])[0]
    # make a third of the field stationary so that clusters exist whatever the random networks predict
    cloud["material_id"] = torch.where(cloud["pos"][:, 2] < -0.2, 6, cloud["material_id"]).to(torch.int32)
    rec_off = drv.run_physics_simulation(sc_off, cloud)
    rec_on = drv.run_physics_simulation(sc_on, cloud)
    assert rec_off["bc_conditions"] == []
    types = [b["type"] for b in rec_on["bc_conditions"]]
    assert types == ["ground", "stationary_cluster"]
    # the same scene composed by hand through the new entry points
    dev = cuda_dev
    R_ = sc_on.rotation_matrices[0].to(dev)
    t, scale, mean = SD.transform2origin(sc_on.particles.to(dev) @ R_.T)
    pos0 = t + torch.tensor([1.0, 1.0, 1.05], device=dev)
    s = MPM_Simulator_WARP(10, device=dev)
    cm = sc_on.cov.to(dev)
    m = torch.stack([cm[:, 0], cm[:, 1], cm[:, 2], cm[:, 1], cm[:, 3], cm[:, 4], cm[:, 2], cm[:, 4], cm[:, 5]], dim=1).view(-1, 3, 3)
    m = R_ @ m @ R_.T
    cov0 = torch.stack([m[:, 0, 0], m[:, 0, 1], m[:, 0, 2], m[:, 1, 1], m[:, 1, 2], m[:, 2, 2]], dim=1) * scale ** 2
    s.load_initial_data_from_torch(pos0, FE.get_particle_volume(pos0, 32, 2.0 / 32), cov0, n_grid=32, grid_lim=2.0, device=dev)
    s.set_parameters_dict(dict(sc_on.material_params), device=dev)
    s.add_bounding_box()
    conf, bcs = MT.apply_material_field_to_simulation(s, cloud, dev, scale, mean, [R_], nn_distance_threshold=0.2, exact_box_semantics=False)
    assert _plain(bcs) == _plain(rec_on["bc_conditions"])
    assert torch.equal(s.mpm_state.particle_material.tensor.cpu(), rec_on["material_ids"].cpu())
    for f in range(3):
        pr, _ = FE.render_frame_transform(s.export_particle_x_to_torch(), None, 0.05, scale, mean, [R_])
        assert (pr - rec_on["frames_pos"][f]).abs().max() < 2e-5, f
        s.p2g2p_n(20, 1e-4)
    assert (rec_on["frames_pos"][2] - rec_off["frames_pos"][2]).abs().max() > 1e-5        # the cuboids change the rollout
