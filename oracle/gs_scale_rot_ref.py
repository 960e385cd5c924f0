"""fp64 restatement of what the reference rasterizer's preprocess builds from scales and rotations (forward.cu's
computeCov3D at scale_modifier 1), for the device rasterizer's scale/rotation entry point.

    cov3d_from_scale_rot(scales, rotations)     (N, 6) upper triangle xx xy xz yy yz zz of Sigma

computeCov3D writes R with glm's column-major constructor, so its R is the transpose of the usual rotation matrix Q of
the quaternion (w, x, y, z); M = S R and Sigma = M^T M = Q S^2 Q^T. The colours computeColorFromSH gives are
gs_render_ref.eval_sh_colors: it evaluates the same terms in the same order.
"""
from __future__ import annotations

import numpy as np


def quat_to_rotmat(q: np.ndarray) -> np.ndarray:
    """(N, 3, 3) usual rotation matrices of quaternions (w, x, y, z), used as given (not normalised)."""
    q = np.asarray(q, np.float64)
    r, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    return np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y)], -1),
                     np.stack([2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x)], -1),
                     np.stack([2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], -1)], 1)


def cov3d_from_scale_rot(scales: np.ndarray, rotations: np.ndarray) -> np.ndarray:
    Q = quat_to_rotmat(rotations)
    s2 = np.asarray(scales, np.float64) ** 2
    sig = np.einsum("nij,nj,nkj->nik", Q, s2, Q)
    return np.stack([sig[:, 0, 0], sig[:, 0, 1], sig[:, 0, 2], sig[:, 1, 1], sig[:, 1, 2], sig[:, 2, 2]], 1)
