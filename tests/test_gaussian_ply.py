"""Per-frame 3DGS PLY export (gs_simulation.py:253-322, gaussian_model.py:177-208). CPU: the fp64 oracle against the
reference's own functions (tests/golden/gaussian_ply_golden.npz) and a hand case; GPU: the record kernel against the
oracle and the fixture, export_gaussians_to_ply's file, and the scene driver's save_ply.

eigh's eigenvector signs are LAPACK's choice, so rotations are compared, not raw quaternions:
  (a) eigenvalues: |exp(2 ls) - max(lambda_ref, 1e-12)| <= 1e-6 lambda_max; log scales to 1e-5 where lambda_ref >= 1e-3
      lambda_max (1e-2 lambda_max against the reference's own float32 eigh, whose eigenvalues are only good to ~1e-7
      lambda_max: 4e-5 in the log at 1.2e-3 lambda_max in the fixture), and the clamp log 1e-6 where lambda_ref <= 1e-12
  (b) R(q) diag(exp(2 ls)) R(q)^T reproduces the covariance to 1e-5 lambda_max (clamped directions count as 0)
  (c) where both eigen-gaps are >= 1e-2 lambda_max, R(q)^T R_ref is diagonal +-1 with determinant +1, to 1e-4
  (d) |q| = 1 to 1e-6 and scipy's from_matrix(R(q)), as (w, x, y, z), is q to 1e-6 (either sign where two of Markley's
      decision values of R(q) are within 1e-5: there the choice, and so the sign, is rounding's)
  (e) xyz, f_dc, f_rest and opacity are bit-exact copies; the normals are exactly 0
"""
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import frame_export_ref as FR  # noqa: E402
from oracle import gaussian_ply_ref as R  # noqa: E402

F32 = np.float32
CLAMP = np.log(np.sqrt(1e-12))
GOLDEN_EXPORTS = ["k16_orig", "k16_raw", "k4_orig", "k4_raw"]
_UP = [0, 1, 2, 1, 3, 4, 2, 4, 5]


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(os.path.join(ROOT, "tests", "golden", "gaussian_ply_golden.npz")))


def eig_ref(cov):
    """fp64 eigenvalues (descending) of the float32 covariances as given."""
    m = np.asarray(cov, np.float64).reshape(-1, 6)[:, _UP].reshape(-1, 3, 3)
    return np.linalg.eigvalsh(m)[:, ::-1]


def check_rotation(cov, ls, q, lam_ref, R_ref, log_floor=1e-3):
    """(a)-(d) for log scales `ls` (N, 3) and quaternions `q` (N, 4, w x y z) of covariances `cov` (N, 6), against the
    reference eigenvalues lam_ref (N, 3, descending) and right-handed eigenvector matrices R_ref (N, 3, 3)."""
    ls, q = np.asarray(ls, np.float64), np.asarray(q, np.float64)
    lam_max = np.abs(lam_ref).max(axis=1, keepdims=True)
    # (a)
    lam = np.exp(2 * ls)
    assert np.all(np.abs(lam - np.maximum(lam_ref, 1e-12)) <= 1e-6 * lam_max + 1e-16)
    big = lam_ref >= log_floor * lam_max
    assert np.all(np.abs(ls - np.log(np.sqrt(np.maximum(lam_ref, 1e-12))))[big] <= 1e-5)
    clamped = lam_ref <= 1e-12 * (1 + 1e-6)
    assert np.all(np.abs(ls[clamped] - CLAMP) <= 1e-5)
    # (b)
    Rq = R.matrix_from_quat_wxyz(q)
    lam_b = np.where(clamped, 0.0, lam)
    rebuilt = np.einsum("nij,nj,nkj->nik", Rq, lam_b, Rq)
    m = np.asarray(cov, np.float64).reshape(-1, 6)[:, _UP].reshape(-1, 3, 3)
    assert np.all(np.abs(rebuilt - m).max(axis=(1, 2)) <= 1e-5 * lam_max[:, 0] + 1e-11)
    # (c)
    gaps = np.minimum(lam_ref[:, 0] - lam_ref[:, 1], lam_ref[:, 1] - lam_ref[:, 2])
    sep = gaps >= 1e-2 * lam_max[:, 0]
    M = np.einsum("nji,njk->nik", Rq[sep], R_ref[sep])
    d = np.sign(np.einsum("nii->ni", M))
    assert np.all(np.abs(M - d[:, :, None] * np.eye(3)).max(axis=(1, 2)) <= 1e-4)
    assert np.all(d.prod(axis=1) == 1)
    # (d)
    assert np.all(np.abs(np.linalg.norm(q, axis=1) - 1) <= 1e-6)
    back = Rotation.from_matrix(Rq).as_quat()[:, [3, 0, 1, 2]]
    dec = np.sort(np.stack([Rq[:, 0, 0], Rq[:, 1, 1], Rq[:, 2, 2], np.trace(Rq, axis1=1, axis2=2)], axis=1), axis=1)
    tie = dec[:, 3] - dec[:, 2] < 1e-5
    err = np.abs(back - q).max(axis=1)
    err[tie] = np.minimum(err[tie], np.abs(back + q).max(axis=1)[tie])
    assert np.all(err <= 1e-6)
    return int(sep.sum())


def check_against_oracle(cov, ls, q):
    """(a)-(d) against the fp64 oracle of the same float32 covariances."""
    _, q_ref = R.cov3D_to_log_scales_and_quats(cov)
    return check_rotation(cov, ls, q, eig_ref(cov), R.matrix_from_quat_wxyz(q_ref))


def check_against_golden(cov, ls, q, g_ls, g_q):
    """(a)-(d) against the reference's own outputs: lambda_ref = exp(2 ls_ref) (its float32 eigh), R_ref = R(q_ref)."""
    return check_rotation(cov, ls, q, np.exp(2 * g_ls.astype(np.float64)), R.matrix_from_quat_wxyz(g_q), log_floor=1e-2)


def check_copies(rec, pos, shs, opacity):
    """(e) on records (N, 14 + 3K)."""
    n, K = shs.shape[0], shs.shape[1]
    assert rec.shape == (n, 14 + 3 * K) and rec.dtype == F32
    assert np.array_equal(rec[:, :3], pos)
    assert np.all(rec[:, 3:6] == 0) and not np.signbit(rec[:, 3:6]).any()
    assert np.array_equal(rec[:, 6:9], shs[:, 0, :])
    assert np.array_equal(rec[:, 9:9 + 3 * (K - 1)], shs[:, 1:, :].transpose(0, 2, 1).reshape(n, -1))
    assert np.array_equal(rec[:, 6 + 3 * K], np.asarray(opacity, F32).reshape(-1))


def golden_export(g, name):
    gs = int(g[f"{name}/gs_num"])
    return dict(gs=gs, rec=g[f"{name}/records"], cov=g[f"{name}/cov_world"], shs=g[f"{name}/shs"][:gs],
                opacity=g[f"{name}/opacity"][:gs], x=g[f"{name}/x"], names=[str(s) for s in g[f"{name}/names"]])


def degenerate_covs():
    """Zero, isotropic, two equal eigenvalues, diagonal, rotated diagonal, 1e6-anisotropic, a -1e-9 eigenvalue."""
    Q = Rotation.from_euler("xyz", [0.3, -1.1, 2.0]).as_matrix()

    def up(m):
        return np.array([m[0, 0], m[0, 1], m[0, 2], m[1, 1], m[1, 2], m[2, 2]])
    rows = [np.zeros(6), up(np.eye(3) * 3e-4), up(Q @ np.diag([5e-4, 5e-4, 2e-6]) @ Q.T), up(Q @ np.diag([5e-4, 2e-6, 2e-6]) @ Q.T),
            up(np.diag([2e-6, 4e-3, 3e-4])), up(Q @ np.diag([4e-3, 3e-4, 2e-6]) @ Q.T), up(Q @ np.diag([1e-2, 1e-5, 1e-8]) @ Q.T),
            up(np.diag([1e-3, 5e-4, -1e-9])), up(Q @ np.diag([1e-3, 5e-4, -1e-9]) @ Q.T), up(np.diag([7e-4, 7e-4, 7e-4]))]
    return np.stack(rows).astype(F32)


def random_inputs(n, K, seed):
    rng = np.random.default_rng(seed)
    ev = 10.0 ** rng.uniform(-6, -2, size=(n, 3))
    Q = Rotation.random(n, random_state=seed).as_matrix()
    m = Q @ (ev[:, :, None] * np.eye(3)) @ Q.transpose(0, 2, 1)
    cov = np.stack([m[:, 0, 0], m[:, 0, 1], m[:, 0, 2], m[:, 1, 1], m[:, 1, 2], m[:, 2, 2]], axis=1).astype(F32)
    deg = degenerate_covs()
    at = rng.choice(n, size=min(n, 4 * len(deg)), replace=False)             # the degenerate ones scattered over the blocks
    cov[at] = deg[np.arange(len(at)) % len(deg)]
    pos = rng.uniform(-2, 2, size=(n, 3)).astype(F32)
    shs = rng.normal(scale=0.5, size=(n, K, 3)).astype(F32)
    opacity = rng.uniform(0, 1, size=n).astype(F32)
    return pos, cov, shs, opacity


def read_ply(path):
    """(header bytes, attribute names, rows (N, n_attr) float32) of a binary little-endian PLY of float properties."""
    data = open(path, "rb").read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    lines = data[:end].decode("ascii").split("\n")
    n = int(next(ln for ln in lines if ln.startswith("element vertex")).split()[-1])
    names = [ln.split()[-1] for ln in lines if ln.startswith("property float")]
    dt = np.dtype([(nm, "<f4") for nm in names])
    assert len(data) == end + n * dt.itemsize
    arr = np.frombuffer(data, dtype=dt, count=n, offset=end)
    return data[:end], names, np.stack([arr[nm] for nm in names], axis=1) if n else np.zeros((0, len(names)), F32)


# ------------------------------------------------------------------------------------------------------------------ CPU
def test_oracle_matches_reference_eigen_step(golden):
    cov = golden["eig/cov"]
    ls, q = R.cov3D_to_log_scales_and_quats(cov)
    assert check_against_golden(cov, ls, q, golden["eig/log_scales"], golden["eig/quats"]) > 150
    assert np.sum(golden["eig/quats"][:, 0] < 0) > 0                      # the reference's w is not forced >= 0
    assert np.sum(np.abs(golden["eig/log_scales"] - CLAMP) < 1e-5) >= 5    # zero and -1e-9 eigenvalues clamp


@pytest.mark.parametrize("name", GOLDEN_EXPORTS)
def test_oracle_matches_reference_export(golden, name):
    e = golden_export(golden, name)
    rec = e["rec"]
    want = R.ply_records(rec[:, :3], e["cov"], e["shs"], e["opacity"])
    check_copies(rec, rec[:, :3], e["shs"], e["opacity"])
    check_copies(want, rec[:, :3], e["shs"], e["opacity"])
    check_against_golden(e["cov"], want[:, -7:-4], want[:, -4:], rec[:, -7:-4], rec[:, -4:])
    g = golden
    if name.endswith("raw"):                                                 # the solver's own positions
        assert np.array_equal(rec[:, :3], e["x"][:e["gs"]])
    else:
        p, c = FR.render_frame_transform(e["x"][:e["gs"]], g[f"{name}/sim_cov"][:e["gs"]], float(g[f"{name}/z_shift"]),
                                         float(g[f"{name}/scale"]), g[f"{name}/mean"], list(g[f"{name}/rots"]))
        assert np.abs(p - rec[:, :3]).max() < 1e-5
        assert np.abs(c - e["cov"]).max() <= 1e-6 * np.abs(e["cov"]).max()


@pytest.mark.parametrize("name", GOLDEN_EXPORTS)
def test_header_matches_reference_attributes(golden, name):
    from pixie_b200.frame_export import gaussian_ply_attributes, gaussian_ply_header
    e = golden_export(golden, name)
    K = e["shs"].shape[1]
    assert R.attribute_names(K) == e["names"] == gaussian_ply_attributes(K)
    h = R.ply_header(e["gs"], K)
    assert gaussian_ply_header(e["gs"], K) == h
    lines = h.decode("ascii").split("\n")
    assert lines[:3] == ["ply", "format binary_little_endian 1.0", f"element vertex {e['gs']}"]
    assert lines[3:-2] == [f"property float {nm}" for nm in e["names"]] and lines[-2:] == ["end_header", ""]


def test_header_without_rest_coefficients():
    from pixie_b200.frame_export import gaussian_ply_header
    h = gaussian_ply_header(3, 1).decode("ascii")
    assert "f_rest" not in h and "property float f_dc_2\nproperty float opacity\n" in h and h.endswith("rot_3\nend_header\n")
    with pytest.raises(ValueError):
        gaussian_ply_header(3, 5)


def test_oracle_hand_case():
    cov = np.array([[4e-4, 0, 0, 1e-4, 0, 2.5e-5]], F32)
    ls, q = R.cov3D_to_log_scales_and_quats(cov)
    assert np.allclose(ls, np.log([2e-2, 1e-2, 5e-3]), atol=1e-7)
    assert np.allclose(q, [[1, 0, 0, 0]], atol=1e-12)
    rec = R.ply_records(np.array([[1, 2, 3]], F32), cov, np.arange(12, dtype=F32).reshape(1, 4, 3), np.array([0.5], F32))
    assert rec.shape == (1, 26)
    assert rec[0, :6].tolist() == [1, 2, 3, 0, 0, 0]
    assert rec[0, 6:9].tolist() == [0, 1, 2] and rec[0, 9:18].tolist() == [3, 6, 9, 4, 7, 10, 5, 8, 11]
    assert rec[0, 18] == F32(0.5) and rec[0, 22:].tolist() == [1, 0, 0, 0]


def test_scene_defaults_leave_save_ply_off():
    from pixie_b200 import scene_driver as SD
    sc = SD.Scene(name="x", grid=None, mask=None, min_bounds=[0] * 3, max_bounds=[1] * 3, particles=torch.zeros(1, 3))
    assert sc.save_ply is False and sc.to_original_coord is True


def test_ply_kernel_does_not_spill(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    src = os.path.join(ROOT, "pixie_b200", "csrc", "gs_ply.cu")
    res = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-c", src,
                          "-o", str(tmp_path / "gs_ply.o")], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    assert res.stderr.count("ply_records_kernel") >= 4                      # K = 1, 4, 9, 16
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", res.stderr)
    assert len(spills) == 4 and all(s == ("0", "0") for s in spills), res.stderr


def test_library_exports_ply_symbol(built_lib):
    assert hasattr(built_lib, "pixie_gaussian_ply_records")


# ------------------------------------------------------------------------------------------------------------------ GPU
def _dev(x, dev):
    return torch.from_numpy(np.ascontiguousarray(x)).to(dev)


@pytest.mark.gpu
@pytest.mark.parametrize("K", [1, 4, 9, 16])
@pytest.mark.parametrize("n", [1, 255, 256, 257, 100_000])
def test_device_records_match_oracle(built_lib, cuda_dev, n, K):
    from pixie_b200.frame_export import gaussian_ply_records
    pos, cov, shs, opacity = random_inputs(n, K, seed=n * 17 + K)
    if n == 1:
        cov = degenerate_covs()[7:8]                                          # the -1e-9 eigenvalue alone
    rec = gaussian_ply_records(*[_dev(a, cuda_dev) for a in (pos, cov, shs, opacity)]).cpu().numpy()
    check_copies(rec, pos, shs, opacity)
    check_against_oracle(cov, rec[:, -7:-4], rec[:, -4:])


@pytest.mark.gpu
def test_device_records_all_degenerate_and_unaligned(built_lib, cuda_dev):
    """Every degenerate covariance in every lane of a block, and inputs / output that are not 16 B aligned."""
    from pixie_b200.frame_export import gaussian_ply_records
    deg = degenerate_covs()
    n = 3 * 128 + 5
    pos, _, shs, opacity = random_inputs(n, 16, seed=5)
    cov = deg[np.arange(n) % len(deg)]

    def shifted(a):                                                           # a view one float into a larger buffer
        flat = torch.zeros(a.size + 1, device=cuda_dev)
        flat[1:] = _dev(a, cuda_dev).reshape(-1)
        return flat[1:].view(a.shape)
    rec = gaussian_ply_records(shifted(pos), shifted(cov), shifted(shs), shifted(opacity)).cpu().numpy()
    check_copies(rec, pos, shs, opacity)
    check_against_oracle(cov, rec[:, -7:-4], rec[:, -4:])
    assert np.all(np.abs(rec[np.arange(n) % len(deg) == 0, -7:-4] - CLAMP) < 1e-5)          # zero covariance
    assert np.all(rec[np.arange(n) % len(deg) == 0, -4:] == [1, 0, 0, 0])
    assert np.all(np.abs(rec[np.arange(n) % len(deg) == 7, -5] - CLAMP) < 1e-5)             # -1e-9: clamped
    from pixie_b200 import _lib
    from pixie_b200.frame_export import cov3D_to_log_scales_and_quats
    ls, q = cov3D_to_log_scales_and_quats(_dev(cov, cuda_dev))
    assert ls.dtype == torch.float32 and q.dtype == torch.float32 and ls.shape == (n, 3) and q.shape == (n, 4)
    assert np.array_equal(ls.cpu().numpy(), rec[:, -7:-4]) and np.array_equal(q.cpu().numpy(), rec[:, -4:])
    with pytest.raises(ValueError):
        gaussian_ply_records(_dev(pos, cuda_dev), _dev(cov, cuda_dev), torch.zeros(n, 5, 3, device=cuda_dev), _dev(opacity, cuda_dev))
    with pytest.raises(_lib.PixieError):
        cov3D_to_log_scales_and_quats(torch.from_numpy(cov))
    empty = gaussian_ply_records(*(torch.zeros(s, device=cuda_dev) for s in ((0, 3), (0, 6), (0, 4, 3), (0,))))
    assert empty.shape == (0, 26)


@pytest.mark.gpu
def test_device_matches_reference_fixture(built_lib, cuda_dev, golden):
    from pixie_b200.frame_export import cov3D_to_log_scales_and_quats, gaussian_ply_records
    cov = golden["eig/cov"]
    ls, q = cov3D_to_log_scales_and_quats(_dev(cov, cuda_dev))
    check_against_golden(cov, ls.cpu().numpy(), q.cpu().numpy(), golden["eig/log_scales"], golden["eig/quats"])
    for name in GOLDEN_EXPORTS:
        e = golden_export(golden, name)
        rec = e["rec"]
        got = gaussian_ply_records(*[_dev(a, cuda_dev) for a in (rec[:, :3], e["cov"], e["shs"], e["opacity"])]).cpu().numpy()
        check_copies(got, rec[:, :3], e["shs"], e["opacity"])
        check_against_golden(e["cov"], got[:, -7:-4], got[:, -4:], rec[:, -7:-4], rec[:, -4:])


def _solver(dev, n, seed):
    from pixie_b200.mpm_solver_warp import MPM_Simulator_WARP
    rng = np.random.default_rng(seed)
    x = rng.uniform(0.7, 1.3, size=(n, 3)).astype(F32)
    _, cov, _, _ = random_inputs(n, 1, seed)
    s = MPM_Simulator_WARP(10, device=dev)
    s.load_initial_data_from_torch(_dev(x, dev), torch.full((n,), 1e-6, device=dev), _dev(cov, dev), n_grid=32, grid_lim=2.0, device=dev)
    s.set_parameters_dict({"material": "jelly", "g": [0.0, 0.0, -9.8], "density": 1000.0, "E": 1e5, "nu": 0.3}, device=dev)
    s.add_bounding_box()
    s.finalize_mu_lam()
    return s


@pytest.mark.gpu
@pytest.mark.parametrize("to_orig", [True, False])
def test_export_gaussians_to_ply_file(built_lib, cuda_dev, tmp_path, to_orig):
    from pixie_b200 import frame_export as FE
    n, gs = 3000, 2900
    s = _solver(cuda_dev, n, 3)
    s.p2g2p_n(5, 1e-4)
    rng = np.random.default_rng(4)
    shs = _dev(rng.normal(size=(n, 16, 3)).astype(F32), cuda_dev)
    opacity = _dev(rng.uniform(size=(n, 1)).astype(F32), cuda_dev)
    rots = [torch.from_numpy(Rotation.from_euler("z", 30, degrees=True).as_matrix().astype(F32)),
            torch.from_numpy(Rotation.from_euler("x", -50, degrees=True).as_matrix().astype(F32))]
    scale, mean, pp = torch.tensor(0.6), torch.tensor([0.1, -0.2, 0.3]), {"z_shift_value": 0.07}
    path = FE.export_gaussians_to_ply(str(tmp_path / "ply"), s, 3, gs, scale, rots, opacity, shs, 12, pp, mean, to_original_coord=to_orig)
    assert path == str(tmp_path / "ply" / "frame_00012.ply")
    x = s.export_particle_x_to_torch()[:gs]
    pr, cw = FE.render_frame_transform(x, s.export_particle_cov_to_torch().view(-1, 6)[:gs], 0.07, scale, mean, rots)
    rec = FE.gaussian_ply_records(pr if to_orig else x, cw, shs[:gs], opacity[:gs]).cpu().numpy()
    header, names, rows = read_ply(path)
    assert header == FE.gaussian_ply_header(gs, 16) and names == R.attribute_names(16)
    assert open(path, "rb").read() == header + rec.astype("<f4").tobytes()
    check_copies(rows, (pr if to_orig else x).cpu().numpy(), shs[:gs].cpu().numpy(), opacity[:gs].cpu().numpy())
    check_against_oracle(cw.cpu().numpy(), rows[:, -7:-4], rows[:, -4:])


@pytest.mark.gpu
def test_frame_writer_overlaps_and_reports_errors(built_lib, cuda_dev, tmp_path):
    from pixie_b200 import frame_export as FE
    d = tmp_path / "frames"
    frames = [random_inputs(1000 + 300 * f, 9, seed=f) for f in range(5)]
    with FE.PlyFrameWriter(str(d), cuda_dev) as w:
        for f, a in enumerate(frames):
            w.submit(f, *[_dev(t, cuda_dev) for t in a])
    for f, (pos, cov, shs, opacity) in enumerate(frames):
        header, _, rows = read_ply(str(d / f"frame_{f:05d}.ply"))
        assert header == FE.gaussian_ply_header(len(pos), 9)
        check_copies(rows, pos, shs, opacity)
        check_against_oracle(cov, rows[:, -7:-4], rows[:, -4:])
    (d / "frame_00001.ply").unlink()
    (d / "frame_00001.ply").mkdir()                                          # this frame cannot be written
    w = FE.PlyFrameWriter(str(d), cuda_dev)
    w.submit(0, *[_dev(t, cuda_dev) for t in frames[0]])
    w.submit(1, *[_dev(t, cuda_dev) for t in frames[1]])
    with pytest.raises(IsADirectoryError):
        w.close()
    assert (d / "frame_00000.ply").stat().st_size == len(FE.gaussian_ply_header(1000, 9)) + 1000 * 4 * 41


# ------------------------------------------------------------------------------------------------------------------ scene driver
MP = {"n_grid": 32, "grid_lim": 2.0, "material": "jelly", "g": [0.0, 0.0, -9.8], "density": 1000.0, "E": 1e5, "nu": 0.3}
TP = {"substep_dt": 1e-4, "frame_dt": 2e-3, "frame_num": 3}
ROT_Z = torch.tensor([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])
AREA = [-0.25, 0.5, -0.5, 0.5, -0.5, 0.5]
CAMERA = {"default_camera_index": -1, "init_azimuthm": 30.0, "init_elevation": 10.0, "init_radius": 2.0, "move_camera": True,
          "delta_a": 5.0, "delta_e": 1.0, "delta_r": 0.02, "mpm_space_vertical_upward_axis": [0, 0, 1]}
CAMERAS = [{"width": 160, "height": 120, "position": [0.0, 0.0, 0.0], "rotation": np.eye(3).tolist(), "fx": 140.0, "fy": 140.0}]


def _driver(dev):
    from oracle import unet_ref as O
    from pixie_b200 import material_transfer as MT
    from pixie_b200 import scene_driver as SD
    C, G = 64, 16
    seg, reg = O.build_pair(C, G, seed=3)
    drv = SD.SceneBatchDriver(feature_channels=C, grid_size=G, device=dev, seg_state_dict=seg.state_dict(), cont_state_dict=reg.state_dict(),
                              **O.DEFAULT_CFG)
    rng = np.random.default_rng(4)
    pred = np.zeros((11, G, G, G), F32)
    pred[:3] = rng.uniform(-0.2, 0.2, size=(3, G, G, G))
    pred[3 + rng.integers(0, 8, size=(G, G, G)), np.arange(G)[:, None, None], np.arange(G)[None, :, None], np.arange(G)[None, None, :]] = 1.0
    ranges = dict(density_min=2.95, density_max=3.05, E_min=4.4, E_max=4.6, nu_min=0.29, nu_max=0.31)
    cloud = MT.extract_material_points(torch.from_numpy(pred).to(dev), torch.ones((G, G, G)).to(dev), [-0.5] * 3, [0.5] * 3, ranges)
    return drv, cloud


def _scene(n=3000, **kw):
    """A shell (radius 0.3 around (0, -0.1, 0)) and a slab of n // 3 Gaussians beside it, SH degree 3."""
    from pixie_b200 import scene_driver as SD
    rng = np.random.default_rng(6)
    v = rng.standard_normal((n, 3))
    shell = np.array([0.0, -0.1, 0.0]) + 0.3 * v / np.linalg.norm(v, axis=1, keepdims=True)
    slab = np.stack([rng.uniform(-0.45, 0.45, n // 3), rng.uniform(0.3, 0.45, n // 3), rng.uniform(-0.45, 0.45, n // 3)], axis=1)
    pos = np.concatenate([shell, slab]).astype(F32)
    k = len(pos)
    s = rng.uniform(0.01, 0.02, (k, 3))
    cov = np.zeros((k, 6), F32)
    cov[:, 0], cov[:, 1], cov[:, 3], cov[:, 5] = s[:, 0] ** 2, 1e-5, s[:, 1] ** 2, s[:, 2] ** 2
    args = dict(name="obj", grid=None, mask=None, min_bounds=[-0.5] * 3, max_bounds=[0.5] * 3, particles=torch.from_numpy(pos),
                cov=torch.from_numpy(cov), opacity=torch.from_numpy(rng.uniform(0.3, 1.0, (k, 1)).astype(F32)),
                shs=torch.from_numpy((rng.standard_normal((k, 16, 3)) * 0.4).astype(F32)), material_params=dict(MP),
                bc_params=[{"type": "bounding_box"}], time_params=TP, nn_distance_threshold=0.2, rotation_matrices=[ROT_Z],
                z_shift_value=0.1)
    args.update(kw)
    return SD.Scene(**args)


def _capture_solver_positions(monkeypatch):
    """The positions the driver hands to render_frame_transform each frame (the solver's own, first n_render)."""
    from pixie_b200 import frame_export as FE
    seen, real = [], FE.render_frame_transform

    def spy(pos, cov, *a, **k):
        if cov is not None:
            seen.append(pos.clone())
        return real(pos, cov, *a, **k)
    monkeypatch.setattr(FE, "render_frame_transform", spy)
    return seen


def check_driver_files(rec, ply_dir, n_rows, positions, shs, opacity):
    from pixie_b200 import frame_export as FE
    files = sorted(os.listdir(ply_dir))
    assert files == [f"frame_{f:05d}.ply" for f in range(TP["frame_num"])]
    for f in range(TP["frame_num"]):
        path = os.path.join(ply_dir, files[f])
        assert os.path.getsize(path) == len(FE.gaussian_ply_header(n_rows, 16)) + n_rows * 4 * (14 + 3 * 16)
        _, _, rows = read_ply(path)
        check_copies(rows, positions[f], shs, opacity)
        cov = rec["frames_cov"][f].cpu().numpy()
        check_against_oracle(cov, rows[:, -7:-4], rows[:, -4:])


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["original", "solver_frame", "visualize", "sim_area"])
def test_scene_driver_save_ply(built_lib, cuda_dev, tmp_path, monkeypatch, variant):
    drv, cloud = _driver(cuda_dev)
    kw = {"save_ply": True}
    if variant == "solver_frame":
        kw["to_original_coord"] = False
    if variant == "visualize":
        kw["particle_filling"] = {"n_grid": 40, "density_threshold": 0.5, "search_threshold": 0.2, "max_particles_num": 2000000,
                                  "visualize": True}
    if variant == "sim_area":
        kw["sim_area"] = AREA
    sc = _scene(**kw)
    seen = _capture_solver_positions(monkeypatch)
    if variant == "visualize":                                                 # the filled particles' render attributes
        from pixie_b200 import particle_filling as PF
        attrs, real = [], PF.init_filled_particles
        monkeypatch.setattr(PF, "init_filled_particles", lambda *a: (attrs.append(real(*a)), attrs[-1])[1])
    ply_dir = str(tmp_path / "ply_files")
    os.makedirs(ply_dir)
    open(os.path.join(ply_dir, "frame_00000.ply"), "wb").write(b"stale")     # overwritten, not deleted
    rec = drv.run_physics_simulation(sc, cloud, ply_dir=ply_dir)
    n_rows = rec["frames_pos"][0].shape[0]
    shs, opacity = sc.shs.numpy(), sc.opacity.numpy().reshape(-1)
    if variant == "visualize":
        assert n_rows == rec["n_particles"] > rec["n_gaussians"]
        shs, opacity = attrs[0][0].cpu().numpy(), attrs[0][1].cpu().numpy().reshape(-1)
    elif variant == "sim_area":
        assert rec["n_unselected"] > 0 and n_rows == rec["n_gaussians"] == len(shs) - rec["n_unselected"]
        keep = np.ones(len(shs), bool)
        rotated = sc.particles.numpy() @ ROT_Z.numpy().T
        for i in range(3):
            keep &= (rotated[:, i] > F32(AREA[2 * i])) & (rotated[:, i] < F32(AREA[2 * i + 1]))
        shs, opacity = shs[keep], opacity[keep]
    else:
        assert n_rows == rec["n_gaussians"] == len(shs)
    if variant == "solver_frame":
        positions = [p.cpu().numpy() for p in seen]
        assert not np.array_equal(positions[1], rec["frames_pos"][1].cpu().numpy())
    else:
        positions = [p.cpu().numpy() for p in rec["frames_pos"]]
    check_driver_files(rec, ply_dir, n_rows, positions, shs, opacity)


@pytest.mark.gpu
def test_scene_driver_record_unchanged_by_save_ply(built_lib, cuda_dev, tmp_path, monkeypatch):
    """Two real rollouts differ in the last bits (float atomics in the particle-to-grid scatter), so this compares runs
    whose substeps are replaced by a fixed deterministic move of every particle: everything else in the frame loop, the
    export, the render and the PLY path, runs as it does."""
    from pixie_b200.mpm_solver_warp import MPM_Simulator_WARP
    monkeypatch.setattr(MPM_Simulator_WARP, "p2g2p_n", lambda self, n, dt, *a, **k: self.export_particle_x_to_torch().add_(1e-3))
    drv, cloud = _driver(cuda_dev)
    runs = []
    for save in (False, True):
        runs.append(drv.run_physics_simulation(_scene(save_ply=save, camera_params=CAMERA, cameras=CAMERAS), cloud,
                                               ply_dir=str(tmp_path / "ply") if save else None))
    off, on = runs
    assert set(off) == set(on)
    for k in ("frames_pos", "frames_cov", "frames_rgb"):
        assert len(off[k]) == len(on[k]) == TP["frame_num"]
        assert all(torch.equal(a, b) for a, b in zip(off[k], on[k])), k
    for k in ("material_ids", "E"):
        assert torch.equal(off[k], on[k])
    assert all(off[k] == on[k] for k in ("n_particles", "n_gaussians", "substeps", "time", "n_filled", "n_unselected"))
    assert len(os.listdir(tmp_path / "ply")) == TP["frame_num"]


@pytest.mark.gpu
def test_scene_driver_save_ply_checks_inputs_first(built_lib, cuda_dev, tmp_path, monkeypatch):
    from pixie_b200.mpm_solver_warp import MPM_Simulator_WARP

    def no_substeps(self, *a, **k):
        raise AssertionError("a substep ran")
    monkeypatch.setattr(MPM_Simulator_WARP, "p2g2p_n", no_substeps)
    drv, cloud = _driver(cuda_dev)
    for missing in ("shs", "opacity", "cov"):
        with pytest.raises(ValueError, match="save_ply"):
            drv.run_physics_simulation(_scene(save_ply=True, **{missing: None}), cloud, ply_dir=str(tmp_path))
    with pytest.raises(ValueError, match="ply_dir"):
        drv.run_physics_simulation(_scene(save_ply=True), cloud)
    assert os.listdir(tmp_path) == []


@pytest.mark.gpu
def test_run_writes_ply_files_under_out_dir(built_lib, cuda_dev, tmp_path, monkeypatch):
    drv, cloud = _driver(cuda_dev)
    monkeypatch.setattr(drv, "generate_neural_segmentation", lambda scenes, out_dir=None: [cloud] * len(scenes))
    recs = drv.run([_scene(n=900, save_ply=True, name="a"), _scene(n=900, name="b")], str(tmp_path))
    assert [r["name"] for r in recs] == ["a", "b"]
    assert sorted(os.listdir(tmp_path / "a" / "ply_files")) == [f"frame_{f:05d}.ply" for f in range(TP["frame_num"])]
    assert not (tmp_path / "b").exists()
