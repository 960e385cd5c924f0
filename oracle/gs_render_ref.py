"""fp64 numpy restatement of the frame renderer gs_simulation.py:573-631 uses: spherical-harmonic colours as
utils/render_utils.py:113-130 (convert_SH) evaluates them, and the forward pass of Inria's diff-gaussian-rasterization
(scale_modifier 1, prefiltered false, precomputed covariances) as a brute-force compositor for small CPU tests.

    eval_sh_colors(deg, shs, means, campos)            (N, 3): SH toward the camera centre, +0.5, clamped at 0
    preprocess(means, cov, cam)                        per Gaussian: visible, depth, mean2D, conic, radius, tile rectangle
    rasterize(means, cov, opacity, colors, cam, bg)    (image (3, H, W), radii, contributors): per pixel, every Gaussian
                                                       whose tile rectangle covers the pixel's tile, in (depth, index)
                                                       order, composited with the reference's thresholds

`cam` is a dict: view (4, 4) and proj (4, 4) as stored (row-vector convention), campos (3,), tan_fovx, tan_fovy, W, H.
"""
from __future__ import annotations

import math

import numpy as np

TILE = 16
SH_C0 = 0.28209479177387814
SH_C1 = 0.4886025119029199
SH_C2 = (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396)
SH_C3 = (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
         1.445305721320277, -0.5900435899266435)


def eval_sh(deg: int, sh: np.ndarray, dirs: np.ndarray) -> np.ndarray:
    """Real SH up to degree 3: sh (N, K, 3) coefficients, dirs (N, 3) unit directions -> (N, 3)."""
    sh = np.asarray(sh, np.float64)
    x, y, z = (dirs[:, i:i + 1] for i in range(3))
    r = SH_C0 * sh[:, 0]
    if deg > 0:
        r = r - SH_C1 * y * sh[:, 1] + SH_C1 * z * sh[:, 2] - SH_C1 * x * sh[:, 3]
    if deg > 1:
        xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
        r = (r + SH_C2[0] * xy * sh[:, 4] + SH_C2[1] * yz * sh[:, 5] + SH_C2[2] * (2.0 * zz - xx - yy) * sh[:, 6]
             + SH_C2[3] * xz * sh[:, 7] + SH_C2[4] * (xx - yy) * sh[:, 8])
    if deg > 2:
        r = (r + SH_C3[0] * y * (3 * xx - yy) * sh[:, 9] + SH_C3[1] * xy * z * sh[:, 10]
             + SH_C3[2] * y * (4 * zz - xx - yy) * sh[:, 11] + SH_C3[3] * z * (2 * zz - 3 * xx - 3 * yy) * sh[:, 12]
             + SH_C3[4] * x * (4 * zz - xx - yy) * sh[:, 13] + SH_C3[5] * z * (xx - yy) * sh[:, 14]
             + SH_C3[6] * x * (xx - 3 * yy) * sh[:, 15])
    return r


def eval_sh_colors(deg: int, shs: np.ndarray, means: np.ndarray, campos: np.ndarray) -> np.ndarray:
    d = np.asarray(means, np.float64) - np.asarray(campos, np.float64)[None]
    d = d / np.linalg.norm(d, axis=1, keepdims=True)
    return np.maximum(eval_sh(deg, shs, d) + 0.5, 0.0)


def _rect(px, py, r, gx, gy):
    x0 = min(gx, max(0, int((px - r) / TILE)))
    y0 = min(gy, max(0, int((py - r) / TILE)))
    x1 = min(gx, max(0, int((px + r + TILE - 1) / TILE)))
    y1 = min(gy, max(0, int((py + r + TILE - 1) / TILE)))
    return x0, y0, x1, y1


def preprocess(means, cov, cam):
    """Per Gaussian a dict (or None when culled): depth, xy, conic (a, b, c), radius, rect (x0, y0, x1, y1), and the
    unrounded ceil argument 3 sqrt(lambda_max) (`r_arg`)."""
    V = np.asarray(cam["view"], np.float64)
    P = np.asarray(cam["proj"], np.float64)
    W, H = int(cam["W"]), int(cam["H"])
    tfx, tfy = float(cam["tan_fovx"]), float(cam["tan_fovy"])
    fx, fy = W / (2.0 * tfx), H / (2.0 * tfy)
    gx, gy = (W + TILE - 1) // TILE, (H + TILE - 1) // TILE
    out = []
    for p, s in zip(np.asarray(means, np.float64), np.asarray(cov, np.float64)):
        ph = np.append(p, 1.0)
        t = ph @ V[:, :3]
        if t[2] <= 0.2:
            out.append(None)
            continue
        h = ph @ P
        pw = 1.0 / (h[3] + 1e-7)
        lx, ly = 1.3 * tfx, 1.3 * tfy
        tx = min(lx, max(-lx, t[0] / t[2])) * t[2]
        ty = min(ly, max(-ly, t[1] / t[2])) * t[2]
        J = np.array([[fx / t[2], 0.0, -fx * tx / t[2] ** 2], [0.0, fy / t[2], -fy * ty / t[2] ** 2]])
        Rv = V[:3, :3].T                               # world -> view rotation (column-vector form)
        Sig = np.array([[s[0], s[1], s[2]], [s[1], s[3], s[4]], [s[2], s[4], s[5]]])
        M = J @ Rv
        c2 = M @ Sig @ M.T
        a, b, c = c2[0, 0] + 0.3, c2[0, 1], c2[1, 1] + 0.3
        det = a * c - b * b
        if det == 0.0:
            out.append(None)
            continue
        mid = 0.5 * (a + c)
        l1 = mid + math.sqrt(max(0.1, mid * mid - det))
        l2 = mid - math.sqrt(max(0.1, mid * mid - det))
        r_arg = 3.0 * math.sqrt(max(l1, l2))
        radius = math.ceil(r_arg)
        xy = (((h[0] * pw + 1.0) * W - 1.0) * 0.5, ((h[1] * pw + 1.0) * H - 1.0) * 0.5)
        rect = _rect(xy[0], xy[1], radius, gx, gy)
        if (rect[2] - rect[0]) * (rect[3] - rect[1]) == 0:
            out.append(None)
            continue
        out.append({"depth": t[2], "xy": xy, "conic": (c / det, -b / det, a / det), "radius": radius, "rect": rect, "r_arg": r_arg})
    return out


def rasterize(means, cov, opacity, colors, cam, bg):
    """(image (3, H, W), radii (N,) int, contributors: {(y, x): tuple of the Gaussian indices composited there})."""
    W, H = int(cam["W"]), int(cam["H"])
    pre = preprocess(means, cov, cam)
    op = np.asarray(opacity, np.float64).reshape(-1)
    col = np.asarray(colors, np.float64)
    bg = np.asarray(bg, np.float64)
    radii = np.array([0 if g is None else g["radius"] for g in pre], np.int64)
    img = np.zeros((3, H, W))
    contrib = {}
    tiles = {}
    for i, g in enumerate(pre):
        if g is None:
            continue
        x0, y0, x1, y1 = g["rect"]
        for ty in range(y0, y1):
            for tx in range(x0, x1):
                tiles.setdefault((ty, tx), []).append(i)
    for ty in range((H + TILE - 1) // TILE):
        for tx in range((W + TILE - 1) // TILE):
            order = sorted(tiles.get((ty, tx), []), key=lambda i: (pre[i]["depth"], i))
            for y in range(ty * TILE, min(H, ty * TILE + TILE)):
                for x in range(tx * TILE, min(W, tx * TILE + TILE)):
                    T, C, used = 1.0, np.zeros(3), []
                    for i in order:
                        g = pre[i]
                        dx, dy = g["xy"][0] - x, g["xy"][1] - y
                        a, b, c = g["conic"]
                        power = -0.5 * (a * dx * dx + c * dy * dy) - b * dx * dy
                        if power > 0.0:
                            continue
                        alpha = min(0.99, op[i] * math.exp(power))
                        if alpha < 1.0 / 255.0:
                            continue
                        test_T = T * (1 - alpha)
                        if test_T < 1e-4:
                            break
                        C += col[i] * alpha * T
                        T = test_T
                        used.append(i)
                    img[:, y, x] = C + T * bg
                    contrib[(y, x)] = tuple(used)
    return img, radii, contrib
