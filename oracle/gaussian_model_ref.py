"""Oracle of the trained-checkpoint decode (pixie_gaussian_checkpoint_decode): GaussianModel.load_ply
(gaussian-splatting/scene/gaussian_model.py:215-260), get_xyz / get_features / get_opacity / get_covariance (:27-31,
:117-118 with utils/general_utils.py:64-110) and the opacity filter of gs_simulation.py:405.

Two forms of the same computation, both from a checkpoint's raw columns `raw` = {"xyz" (N, 3), "f_dc" (N, 3), "f_rest"
(N, 3 (K-1)) in f_rest_* numeric order, "opacity" (N,), "scale" (N, 3), "rot" (N, 4)}, float32:
- `decode_f64`: numpy in float64, the exact values the float32 pipeline approximates;
- `torch_reference`: the reference's float32 torch expressions, op by op, to run on the same device as the kernel.
"""
from __future__ import annotations

import numpy as np


def shs_from_columns(f_dc: np.ndarray, f_rest: np.ndarray) -> np.ndarray:
    """(N, K, 3): shs[p, 0, c] = f_dc_c, shs[p, k, c] = f_rest_{c (K-1) + k - 1} (load_ply's reshape (P, 3, K-1), transpose)."""
    n = f_dc.shape[0]
    k1 = f_rest.shape[1] // 3
    return np.concatenate([f_dc.reshape(n, 1, 3), f_rest.reshape(n, 3, k1).transpose(0, 2, 1)], axis=1)


def rotation_f64(rot: np.ndarray) -> np.ndarray:
    """build_rotation in float64: the quaternion (w, x, y, z) normalised, then the rotation matrix."""
    q = rot.astype(np.float64)
    with np.errstate(invalid="ignore", divide="ignore"):
        q = q / np.sqrt((q * q).sum(axis=1, keepdims=True))
    w, x, y, z = q.T
    return np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
                     2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
                     2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], axis=1).reshape(-1, 3, 3)


def decode_f64(raw) -> dict:
    """pos (N, 3), shs (N, K, 3), opacity (N, 1), cov (N, 6) and s_max (N,) = the largest scale, in float64."""
    with np.errstate(over="ignore", invalid="ignore"):
        opacity = 1.0 / (1.0 + np.exp(-raw["opacity"].astype(np.float64)))
        s = np.exp(raw["scale"].astype(np.float64))
        L = rotation_f64(raw["rot"]) * s[:, None, :]
        S = L @ L.transpose(0, 2, 1)
    return {"pos": raw["xyz"].astype(np.float64), "shs": shs_from_columns(raw["f_dc"], raw["f_rest"]).astype(np.float64),
            "opacity": opacity[:, None], "cov": S[:, [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]], "s_max": s.max(axis=1)}


def keep_mask(opacity_f32: np.ndarray, threshold: float) -> np.ndarray:
    """gs_simulation.py:405: opacity > threshold, the threshold rounded to float32 as torch compares a float32 tensor with
    a Python float (strict; NaN is dropped)."""
    return np.asarray(opacity_f32, dtype=np.float32).reshape(-1) > np.float32(threshold)


def torch_reference(raw, device) -> dict:
    """The reference's float32 torch ops on `device`: pos, shs (get_features), opacity (sigmoid), cov (strip_symmetric of
    L L^T with L = build_rotation(rot) @ diag(exp(scale))) and L itself."""
    import torch
    t = lambda a: torch.tensor(np.asarray(a, dtype=np.float32), dtype=torch.float, device=device)   # noqa: E731
    n = raw["xyz"].shape[0]
    k1 = raw["f_rest"].shape[1] // 3
    xyz = t(raw["xyz"])
    dc = t(raw["f_dc"].reshape(n, 3, 1)).transpose(1, 2).contiguous()
    rest = t(raw["f_rest"].reshape(n, 3, k1)).transpose(1, 2).contiguous()
    opacity = torch.sigmoid(t(raw["opacity"].reshape(n, 1)))
    s = torch.exp(t(raw["scale"]))
    r = t(raw["rot"])
    norm = torch.sqrt(r[:, 0] * r[:, 0] + r[:, 1] * r[:, 1] + r[:, 2] * r[:, 2] + r[:, 3] * r[:, 3])
    q = r / norm[:, None]
    w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R = torch.zeros((n, 3, 3), device=device)
    R[:, 0, 0] = 1 - 2 * (y * y + z * z)
    R[:, 0, 1] = 2 * (x * y - w * z)
    R[:, 0, 2] = 2 * (x * z + w * y)
    R[:, 1, 0] = 2 * (x * y + w * z)
    R[:, 1, 1] = 1 - 2 * (x * x + z * z)
    R[:, 1, 2] = 2 * (y * z - w * x)
    R[:, 2, 0] = 2 * (x * z - w * y)
    R[:, 2, 1] = 2 * (y * z + w * x)
    R[:, 2, 2] = 1 - 2 * (x * x + y * y)
    D = torch.zeros((n, 3, 3), dtype=torch.float, device=device)
    D[:, 0, 0], D[:, 1, 1], D[:, 2, 2] = s[:, 0], s[:, 1], s[:, 2]
    L = R @ D
    S = L @ L.transpose(1, 2)
    cov = torch.stack([S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2]], dim=1)
    return {"pos": xyz, "shs": torch.cat((dc, rest), dim=1), "opacity": opacity, "cov": cov, "L": L}
