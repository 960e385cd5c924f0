"""ORACLE (test infrastructure, not product code): numpy fp64 restatement of the per-frame 3DGS PLY export.

  cov3D_to_log_scales_and_quats   third_party/PhysGaussian/gs_simulation.py:253-288 (torch.linalg.eigh, descending sort,
                                  sqrt(clamp(lambda, 1e-12)), log, third eigenvector negated when det R < 0, scipy
                                  Rotation.from_matrix -> (w, x, y, z))
  ply_records / ply_header        export_gaussians_to_ply (:290-322) with gaussian-splatting/scene/gaussian_model.py:177-208
                                  (construct_list_of_attributes, save_ply) and the header plyfile writes for that array

from_matrix is restated as scipy computes it for an orthogonal matrix (Markley's decision: the largest of R00, R11, R22
and the trace, first on ties, builds its component first; then normalise; no sign canonicalisation). eigh's eigenvectors
are orthogonal to fp64 rounding, so scipy's orthogonalisation of a non-orthogonal input does not arise here.
PINNED BY THE REFERENCE'S OWN FUNCTIONS: tests/golden/make_gaussian_ply_golden.py runs them on CPU torch;
tests/test_gaussian_ply.py compares against that fixture. Only tests/ may import this file.
"""
import numpy as np

_FULL_FROM_UPPER = [0, 1, 2, 1, 3, 4, 2, 4, 5]


def cov3D_to_log_scales_and_quats(cov3D):
    """(log_scales (N, 3), quats_wxyz (N, 4)) in float64 from (N, 6) upper-triangular covariances. A row with a NaN or
    +-Inf entry gives NaN log scales and quaternion (the product's convention; the reference raises or returns NaN)."""
    u = np.asarray(cov3D, np.float64).reshape(-1, 6)
    bad = ~np.isfinite(u).all(axis=1)
    evals, R = eigen_frame(np.where(bad[:, None], 0.0, u))
    ls, q = np.log(np.sqrt(np.maximum(evals, 1e-12))), quat_wxyz_from_matrix(R)
    ls[bad], q[bad] = np.nan, np.nan
    return ls, q


def eigen_frame(cov3D):
    """(eigenvalues (N, 3) descending, R (N, 3, 3)) of finite (N, 6) covariances in fp64: the eigenvectors as columns,
    the third negated where det R < 0, as cov3D_to_log_scales_and_quats hands R to from_matrix."""
    m = np.asarray(cov3D, np.float64).reshape(-1, 6)[:, _FULL_FROM_UPPER].reshape(-1, 3, 3)
    evals, evecs = np.linalg.eigh(m)                                       # ascending
    idx = np.argsort(-evals, axis=1, kind="stable")
    evals = np.take_along_axis(evals, idx, axis=1)
    R = np.take_along_axis(evecs, idx[:, None, :], axis=2).copy()
    neg = np.linalg.det(R) < 0
    R[neg, :, 2] *= -1
    return evals, R


def quat_wxyz_from_matrix(R):
    """scipy Rotation.from_matrix(R).as_quat() reordered to (w, x, y, z), for orthogonal R (N, 3, 3)."""
    R = np.asarray(R, np.float64).reshape(-1, 3, 3)
    tr = R[:, 0, 0] + R[:, 1, 1] + R[:, 2, 2]
    decision = np.stack([R[:, 0, 0], R[:, 1, 1], R[:, 2, 2], tr], axis=1)
    choice = np.argmax(decision, axis=1)
    q = np.empty((len(R), 4))                                              # x y z w
    for n in range(len(R)):
        c = choice[n]
        if c == 3:
            q[n] = [R[n, 2, 1] - R[n, 1, 2], R[n, 0, 2] - R[n, 2, 0], R[n, 1, 0] - R[n, 0, 1], 1 + tr[n]]
        else:
            i, j, k = c, (c + 1) % 3, (c + 2) % 3
            q[n, i] = 1 - tr[n] + 2 * R[n, i, i]
            q[n, j] = R[n, j, i] + R[n, i, j]
            q[n, k] = R[n, k, i] + R[n, i, k]
            q[n, 3] = R[n, k, j] - R[n, j, k]
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    return q[:, [3, 0, 1, 2]]


def matrix_from_quat_wxyz(q):
    """The rotation matrix of unit quaternions (w, x, y, z) (N, 4), in fp64."""
    w, x, y, z = np.asarray(q, np.float64).reshape(-1, 4).T
    return np.stack([
        np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], axis=1),
        np.stack([2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)], axis=1),
        np.stack([2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], axis=1)], axis=1)


def attribute_names(K):
    """construct_list_of_attributes for features_dc (N, 1, 3) and features_rest (N, K - 1, 3)."""
    names = ["x", "y", "z", "nx", "ny", "nz"] + [f"f_dc_{i}" for i in range(3)] + [f"f_rest_{i}" for i in range(3 * (K - 1))]
    return names + ["opacity"] + [f"scale_{i}" for i in range(3)] + [f"rot_{i}" for i in range(4)]


def ply_header(n, K):
    """What plyfile writes before the binary vertex table of save_ply's structured array."""
    lines = ["ply", "format binary_little_endian 1.0", f"element vertex {n}"]
    lines += [f"property float {a}" for a in attribute_names(K)]
    return ("\n".join(lines + ["end_header"]) + "\n").encode("ascii")


def ply_records(pos, cov, shs, opacity):
    """save_ply's attribute rows (N, 14 + 3K) float32: xyz, zero normals, f_dc, f_rest (transpose(1, 2).flatten),
    opacity, log scales, quaternion (w, x, y, z)."""
    pos = np.asarray(pos, np.float32).reshape(-1, 3)
    shs = np.asarray(shs, np.float32)
    n, K = shs.shape[0], shs.shape[1]
    ls, q = cov3D_to_log_scales_and_quats(cov)
    f_dc = shs[:, :1, :].transpose(0, 2, 1).reshape(n, 3)
    f_rest = shs[:, 1:, :].transpose(0, 2, 1).reshape(n, 3 * (K - 1))
    return np.concatenate([pos, np.zeros_like(pos), f_dc, f_rest, np.asarray(opacity, np.float32).reshape(n, 1),
                           ls.astype(np.float32), q.astype(np.float32)], axis=1)
