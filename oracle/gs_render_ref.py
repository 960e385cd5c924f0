"""fp64 numpy restatement of the frame renderer gs_simulation.py:573-631 uses: spherical-harmonic colours as
utils/render_utils.py:113-130 (convert_SH) evaluates them, and the forward pass of Inria's diff-gaussian-rasterization
(scale_modifier 1, prefiltered false, precomputed covariances) as a brute-force compositor for small CPU tests.

    eval_sh_colors(deg, shs, means, campos)            (N, 3): SH toward the camera centre, +0.5, clamped at 0
    preprocess(means, cov, cam)                        per Gaussian: visible, depth, mean2D, conic, radius, tile rectangle
    rasterize(means, cov, opacity, colors, cam, bg)    (image (3, H, W), radii, contributors): per pixel, every Gaussian
                                                       whose tile rectangle covers the pixel's tile, in (depth, index)
                                                       order, composited with the reference's thresholds; with
                                                       margin=True also the per-pixel threshold margin (H, W)
    rasterize_tiles(...)                               (image, radii, margin): the same compositing vectorised over
                                                       pixels and tiles, for images and stacks the loop is too slow for

The threshold margin of a pixel is the smallest relative distance, over the Gaussians the pixel considered, of each
value the compositor compares from its threshold: power from 0 (relative to the magnitude of its terms), alpha from
1/255, o·e^power from the 0.99 clamp, and T·(1 − α) from 1e-4. It is 0 where a Gaussian that could contribute
(α ≥ 1/255) covers the pixel's tile only under a last-bit change of its screen position or radius. A float32
rasterizer may decide the other way where the margin is small; everywhere else it must composite the same set.

`cam` is a dict: view (4, 4) and proj (4, 4) as stored (row-vector convention), campos (3,), tan_fovx, tan_fovy, W, H.
"""
from __future__ import annotations

import math

import numpy as np

TILE = 16
NEAR = float(np.float32(0.2))   # the reference culls at view z <= 0.2f
# relative perturbations under which a float32 pipeline may land elsewhere: the screen position (relative to the
# image size plus its magnitude) and the radius's ceil argument (the existing ±1 radius rule)
POS_REL, R_ARG_TOL = 1e-6, 1e-5
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
    """Per Gaussian a dict (or None when culled): depth, xy, conic (a, b, c), radius, rect (x0, y0, x1, y1), the
    unrounded ceil argument 3 sqrt(lambda_max) (`r_arg`), and the rectangles `outer` / `inner` that hold every / only the
    tiles the rectangle covers under a last-bit change of the screen position (POS_REL) or of a ceil argument within
    R_ARG_TOL of an integer. A Gaussian whose own rectangle is empty but whose outer one is not is culled only by such
    a change: it gets radius 0 and `rect_culled` True, and stays in the dict list so that its pixels get margin 0."""
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
        if t[2] <= NEAR:
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
        dx, dy = POS_REL * (abs(xy[0]) + W), POS_REL * (abs(xy[1]) + H)
        rs = {math.ceil(r_arg - R_ARG_TOL), radius, math.ceil(r_arg + R_ARG_TOL)}
        rects = [_rect(xy[0] + sx * dx, xy[1] + sy * dy, rr, gx, gy) for sx in (-1, 1) for sy in (-1, 1) for rr in rs]
        outer = tuple(f(r[k] for r in rects) for k, f in enumerate((min, min, max, max)))
        inner = tuple(f(r[k] for r in rects) for k, f in enumerate((max, max, min, min)))
        culled = (rect[2] - rect[0]) * (rect[3] - rect[1]) == 0
        if culled and (outer[2] - outer[0]) * (outer[3] - outer[1]) == 0:
            out.append(None)
            continue
        out.append({"depth": t[2], "xy": xy, "conic": (c / det, -b / det, a / det), "radius": 0 if culled else radius, "rect": rect,
                    "r_arg": r_arg, "outer": outer, "inner": inner, "rect_culled": culled})
    return out


def _in_rect(r, tx, ty):
    return (tx >= r[0]) & (tx < r[2]) & (ty >= r[1]) & (ty < r[3])


def _power_margin(a, b, c, dx, dy, power):
    """|power| relative to the magnitude of its terms; at the mean itself, the least such ratio over directions."""
    absq = 0.5 * (abs(a) * dx * dx + abs(c) * dy * dy) + np.abs(b * dx * dy)
    rho = abs(b) / math.sqrt(a * c) if a * c > 0 else 1.0
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where(absq > 0, np.abs(power) / np.where(absq > 0, absq, 1.0), (1 - rho) / (1 + rho))


def rasterize(means, cov, opacity, colors, cam, bg, margin=False):
    """(image (3, H, W), radii (N,) int, contributors: {(y, x): tuple of the Gaussian indices composited there}), and
    with margin=True the threshold margin (H, W) as a fourth element (inf where a pixel considered nothing)."""
    W, H = int(cam["W"]), int(cam["H"])
    pre = preprocess(means, cov, cam)
    op = np.asarray(opacity, np.float64).reshape(-1)
    col = np.asarray(colors, np.float64)
    bg = np.asarray(bg, np.float64)
    radii = np.array([0 if g is None else g["radius"] for g in pre], np.int64)
    img = np.zeros((3, H, W))
    marg = np.full((H, W), np.inf)
    contrib = {}
    tiles = {}
    for i, g in enumerate(pre):
        if g is None:
            continue
        x0, y0, x1, y1 = g["outer"]
        for ty in range(y0, y1):
            for tx in range(x0, x1):
                tiles.setdefault((ty, tx), []).append(i)
    for ty in range((H + TILE - 1) // TILE):
        for tx in range((W + TILE - 1) // TILE):
            order = sorted(tiles.get((ty, tx), []), key=lambda i: (pre[i]["depth"], i))
            for y in range(ty * TILE, min(H, ty * TILE + TILE)):
                for x in range(tx * TILE, min(W, tx * TILE + TILE)):
                    T, C, used, m = 1.0, np.zeros(3), [], np.inf
                    for i in order:
                        g = pre[i]
                        inside = bool(_in_rect(g["rect"], tx, ty))
                        doubt = not _in_rect(g["inner"], tx, ty)
                        dx, dy = g["xy"][0] - x, g["xy"][1] - y
                        a, b, c = g["conic"]
                        power = -0.5 * (a * dx * dx + c * dy * dy) - b * dx * dy
                        m = min(m, float(_power_margin(a, b, c, dx, dy, power)))
                        if power > 0.0:
                            continue
                        raw = op[i] * math.exp(power)
                        alpha = min(0.99, raw)
                        m = min(m, abs(raw - 0.99) / 0.99, abs(alpha - 1.0 / 255.0) * 255.0)
                        if alpha < 1.0 / 255.0:
                            continue
                        if doubt:
                            m = 0.0
                        if not inside:
                            continue
                        test_T = T * (1 - alpha)
                        m = min(m, abs(test_T - 1e-4) / 1e-4)
                        if test_T < 1e-4:
                            break
                        C += col[i] * alpha * T
                        T = test_T
                        used.append(i)
                    img[:, y, x] = C + T * bg
                    contrib[(y, x)] = tuple(used)
                    marg[y, x] = m
    return (img, radii, contrib, marg) if margin else (img, radii, contrib)


def rasterize_tiles(means, cov, opacity, colors, cam, bg, chunk_tiles=2048):
    """rasterize() vectorised: every tile's (depth, index)-ordered list is walked one entry at a time for all pixels of a
    chunk of tiles at once (tiles of similar list length together). Returns (image (3, H, W), radii (N,), margin (H, W))."""
    W, H = int(cam["W"]), int(cam["H"])
    gx = (W + TILE - 1) // TILE
    pre = preprocess(means, cov, cam)
    n = len(pre)
    op = np.asarray(opacity, np.float64).reshape(-1)
    col = np.asarray(colors, np.float64).reshape(n, 3)
    bg = np.asarray(bg, np.float64)
    radii = np.array([0 if g is None else g["radius"] for g in pre], np.int64)
    img = np.broadcast_to(bg[:, None, None], (3, H, W)).copy()
    marg = np.full((H, W), np.inf)
    vis = [i for i, g in enumerate(pre) if g is not None]
    if not vis:
        return img, radii, marg
    gs, ts, ins, dbt = [], [], [], []
    for i in vis:
        g = pre[i]
        x0, y0, x1, y1 = g["outer"]
        X, Y = np.meshgrid(np.arange(x0, x1), np.arange(y0, y1))
        X, Y = X.ravel(), Y.ravel()
        gs.append(np.full(X.size, i))
        ts.append(Y * gx + X)
        ins.append(_in_rect(g["rect"], X, Y))
        dbt.append(~_in_rect(g["inner"], X, Y))
    gs, ts, ins, dbt = (np.concatenate(v) for v in (gs, ts, ins, dbt))
    depth = np.zeros(n)
    depth[vis] = [pre[i]["depth"] for i in vis]
    o = np.lexsort((gs, depth[gs], ts))
    gs, ts, ins, dbt = gs[o], ts[o], ins[o], dbt[o]
    tile_ids, starts, counts = np.unique(ts, return_index=True, return_counts=True)
    px_m = np.zeros(n); py_m = np.zeros(n); ca = np.ones(n); cb = np.zeros(n); cc = np.ones(n)
    for i in vis:
        px_m[i], py_m[i] = pre[i]["xy"]
        ca[i], cb[i], cc[i] = pre[i]["conic"]
    rho = np.abs(cb) / np.sqrt(ca * cc)
    lane = np.arange(TILE * TILE)
    by_len = np.argsort(counts, kind="stable")
    for c0 in range(0, len(by_len), chunk_tiles):
        sel = by_len[c0:c0 + chunk_tiles]
        tid, st, cnt = tile_ids[sel], starts[sel], counts[sel]
        X = (tid % gx)[:, None] * TILE + lane % TILE
        Y = (tid // gx)[:, None] * TILE + lane // TILE
        valid = (X < W) & (Y < H)
        T = np.ones(X.shape)
        C = np.zeros(X.shape + (3,))
        m = np.full(X.shape, np.inf)
        done = ~valid
        for k in range(int(cnt.max())):
            act = ~done & (k < cnt)[:, None]
            if not act.any():
                break
            e = st + np.minimum(k, cnt - 1)
            g = gs[e]
            a, b, c = ca[g][:, None], cb[g][:, None], cc[g][:, None]
            dx, dy = px_m[g][:, None] - X, py_m[g][:, None] - Y
            power = -0.5 * (a * dx * dx + c * dy * dy) - b * dx * dy
            absq = 0.5 * (np.abs(a) * dx * dx + np.abs(c) * dy * dy) + np.abs(b * dx * dy)
            with np.errstate(invalid="ignore", divide="ignore"):
                mp = np.where(absq > 0, np.abs(power) / np.where(absq > 0, absq, 1.0), ((1 - rho[g]) / (1 + rho[g]))[:, None])
            m = np.where(act, np.minimum(m, mp), m)
            ok = act & (power <= 0.0)
            with np.errstate(over="ignore"):
                raw = op[g][:, None] * np.exp(np.minimum(power, 0.0))
            alpha = np.minimum(0.99, raw)
            m = np.where(ok, np.minimum(m, np.minimum(np.abs(raw - 0.99) / 0.99, np.abs(alpha - 1.0 / 255.0) * 255.0)), m)
            seen = ok & (alpha >= 1.0 / 255.0)
            m = np.where(seen & dbt[e][:, None], 0.0, m)
            blend = seen & ins[e][:, None]
            test_T = T * (1 - alpha)
            m = np.where(blend, np.minimum(m, np.abs(test_T - 1e-4) / 1e-4), m)
            stop = blend & (test_T < 1e-4)
            done = done | stop
            go = blend & ~stop
            C = C + np.where(go[..., None], col[g][:, None, :] * (alpha * T)[..., None], 0.0)
            T = np.where(go, test_T, T)
        yy, xx = Y[valid], X[valid]
        img[:, yy, xx] = (C[valid] + T[valid][:, None] * bg).T
        marg[yy, xx] = m[valid]
    return img, radii, marg
