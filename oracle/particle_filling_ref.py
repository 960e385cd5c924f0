"""Vectorised numpy restatement of the reference's particle filling (PG/particle_filling/filling.py:26-380, Taichi f32 / i32),
fast enough for inputs of config size. Pinned to the reference's own kernels through tests/golden/filling_golden.npz
(tests/golden/make_filling_golden.py executes them).

Float32 throughout like Taichi's default precision, with the reference's operation order inside one Gaussian's
contribution; contributions are accumulated in a different order (np.add.at over groups of equal window radius), so
densities agree with the reference to float32 rounding, not bit for bit. Like the device code, a Gaussian outside the grid
counts in the nearest border cell.
"""
from __future__ import annotations

import numpy as np

F32 = np.float32


def _sym_precision(cov):
    """sig, P = Q diag(1 / max(sig, 1e-8)) Q^T in float32 from the signed eigen-decomposition (float64 eigh, rounded)."""
    m = cov[:, [0, 1, 2, 1, 3, 4, 2, 4, 5]].reshape(-1, 3, 3).astype(np.float64)
    w, V = np.linalg.eigh(m)
    sig = np.maximum(w.astype(F32), F32(1e-8))
    Q = V.astype(F32)
    M = Q * (F32(1.0) / sig)[:, None, :]
    P = np.empty_like(Q)
    for r in range(3):
        for q in range(3):
            P[:, r, q] = (M[:, r, 0] * Q[:, q, 0] + M[:, r, 1] * Q[:, q, 1]) + M[:, r, 2] * Q[:, q, 2]
    return sig, P


def densify_grids(pos, opacity, cov, grid_n, grid_dx, chunk=1 << 16):
    """(count int32, density float32) grids of shape (grid_n,)*3, filling.py:26-87."""
    pos = np.asarray(pos, F32).reshape(-1, 3)
    opacity = np.asarray(opacity, F32).reshape(-1)
    cov = np.asarray(cov, F32).reshape(-1, 6)
    n, dx = int(grid_n), F32(grid_dx)
    count = np.zeros((n, n, n), np.int32)
    density = np.zeros(n ** 3, F32)
    c0 = np.floor(pos / dx).astype(np.int64)
    cc = np.clip(c0, 0, n - 1)
    np.add.at(count, (cc[:, 0], cc[:, 1], cc[:, 2]), 1)
    sig, P = _sym_precision(cov)
    r = np.minimum(np.ceil(np.sqrt(sig).max(axis=1) / dx), n).astype(np.int64)
    corners = [(a, b, c) for a in range(2) for b in range(2) for c in range(2)]
    for rv in np.unique(r):
        ax = np.arange(-rv, rv + 1)
        off = np.stack(np.meshgrid(ax, ax, ax, indexing="ij"), axis=-1).reshape(-1, 3)
        sel = np.nonzero(r == rv)[0]
        for s in range(0, len(sel), max(1, chunk // len(off))):
            g = sel[s:s + max(1, chunk // len(off))]
            cell = c0[g][:, None, :] + off[None]                                   # (G, W, 3)
            ok = np.all((cell >= 0) & (cell < n), axis=-1)
            p, Pg = pos[g][:, None, :], P[g][:, None]
            gw = np.zeros(ok.shape, F32)
            for corner in corners:
                d = p - (cell + np.array(corner)).astype(F32) * dx
                y = [(Pg[..., q, 0] * d[..., 0] + Pg[..., q, 1] * d[..., 1]) + Pg[..., q, 2] * d[..., 2] for q in range(3)]
                e = (d[..., 0] * y[0] + d[..., 1] * y[1]) + d[..., 2] * y[2]
                gw = gw + np.exp(F32(-0.5) * e)
            val = opacity[g][:, None] * gw / F32(8.0)
            flat = (cell[..., 0] * n + cell[..., 1]) * n + cell[..., 2]
            np.add.at(density, flat[ok], val[ok])
    return count, density.reshape(n, n, n)


def _beyond(b):
    """Along axis 0 in the +direction: (any dense cell strictly beyond t, number of runs of dense cells strictly beyond t)."""
    n = b.shape[0]
    hit = np.zeros_like(b)
    hit[:-1] = np.flip(np.logical_or.accumulate(np.flip(b[1:], 0), axis=0), 0)
    rise = b.copy()
    rise[1:] &= ~b[:-1]
    suffix = np.zeros((n + 1,) + b.shape[1:], np.int64)
    suffix[:-1] = np.flip(np.cumsum(np.flip(rise, 0), axis=0), 0)                  # suffix[s] = sum(rise[s:])
    runs = np.zeros(b.shape, np.int64)
    runs[:-1] = b[1:].astype(np.int64) + suffix[2:]                                # the cell after t always starts a run
    return hit, runs


def classify(density, search_thres, exclude_dir, ray_cast_dir):
    """Per cell: enclosed (collision_search hits in every direction but exclude_dir) and the collision_times parity."""
    b = density > F32(search_thres)
    enclosed = np.ones(b.shape, bool)
    runs_ray = None
    for d in range(6):
        axis, minus = d // 2, d % 2
        v = np.moveaxis(b, axis, 0)
        if minus:
            v = np.flip(v, 0)
        hit, runs = _beyond(v)
        if minus:
            hit, runs = np.flip(hit, 0), np.flip(runs, 0)
        hit, runs = np.moveaxis(hit, 0, axis), np.moveaxis(runs, 0, axis)
        if d != exclude_dir:
            enclosed &= hit
        if d == ray_cast_dir:
            runs_ray = runs
    return enclosed, runs_ray % 2 == 1


def fill_grids(count, density, density_thres, search_thres, max_particles_per_cell, exclude_dir, ray_cast_dir):
    """fill_dense_grids + internal_filling: (count after dense fill, count after internal fill, new per cell dense, interior)."""
    ppc = int(max_particles_per_cell)
    c1 = count.copy()
    dense = (density > F32(density_thres)) & (c1 < ppc)
    add_d = np.where(dense, ppc - c1, 0).astype(np.int32)
    c1[dense] = ppc
    enclosed, odd = classify(density, search_thres, exclude_dir, ray_cast_dir)
    inner = (c1 == 0) & enclosed & odd
    add_i = np.where(inner, ppc, 0).astype(np.int32)
    c2 = c1.copy()
    c2[inner] = ppc
    return c1, c2, add_d, add_i


def emit(add, grid_dx, origin, rng):
    """(cell + U[0,1)^3) * dx + origin for add[c] particles per cell, C order of cells."""
    n = add.shape[0]
    flat = np.repeat(np.arange(add.size), add.ravel())
    cell = np.stack(np.unravel_index(flat, (n, n, n)), axis=1).astype(F32)
    u = rng.random((len(flat), 3), dtype=F32)
    return (cell + u) * F32(grid_dx) + np.asarray(origin, F32)


def fill_particles(pos, opacity, cov, grid_n, max_samples, grid_dx, density_thres=2.0, search_thres=1.0, max_particles_per_cell=1,
                   search_exclude_dir=5, ray_cast_dir=4, boundary=None, seed=0):
    """filling.py:291-380 with every intermediate: dict(out, count, density, count_dense, count_internal, add_dense,
    add_interior, n_dense, n_total, grid_dx, origin)."""
    pos = np.asarray(pos, F32).reshape(-1, 3)
    p, o, c = pos, np.asarray(opacity, F32).reshape(-1), np.asarray(cov, F32).reshape(-1, 6)
    origin = np.zeros(3, F32)
    if boundary is not None:
        keep = np.ones(len(p), bool)
        for i in range(3):
            keep &= (p[:, i] > F32(boundary[2 * i])) & (p[:, i] < F32(boundary[2 * i + 1]))
        grid_dx = max(boundary[2 * i + 1] - boundary[2 * i] for i in range(3)) / grid_n
        origin = np.array([boundary[0], boundary[2], boundary[4]], F32)
        p, o, c = p[keep] - origin, o[keep], c[keep]
    count, density = densify_grids(p, o, c, grid_n, grid_dx)
    c1, c2, add_d, add_i = fill_grids(count, density, density_thres, search_thres, max_particles_per_cell, search_exclude_dir, ray_cast_dir)
    n_dense, n_total = int(add_d.sum()), int(add_d.sum() + add_i.sum())
    if n_total > max_samples:
        raise ValueError(f"filling adds {n_total} particles but max_samples is {max_samples}")
    rng = np.random.default_rng(seed)
    new = np.concatenate([emit(add_d, grid_dx, origin, rng), emit(add_i, grid_dx, origin, rng)])
    return dict(out=np.concatenate([pos, new]), count=count, density=density, count_dense=c1, count_internal=c2, add_dense=add_d,
                add_interior=add_i, n_dense=n_dense, n_total=n_total, grid_dx=grid_dx, origin=origin)
