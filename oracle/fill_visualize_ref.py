"""Numpy restatement of the reference's nearest-Gaussian step of particle filling (PG/particle_filling/filling.py:383-446:
get_attr_from_closest / init_filled_particles, reached with the config's `particle_filling.visualize`), exact at any
size: indices and copied rows bit for bit. Pinned to the reference's own functions through
tests/golden/fill_visualize_golden.npz (tests/golden/make_fill_visualize_golden.py executes them).
"""
from __future__ import annotations

import numpy as np

F32 = np.float32
NEAREST_SLACK = 1.0 + 2.0 ** -19       # the float32 distance is within a few units of 2^-24 of the exact one (csrc/nearest.cu)
NEAREST_FLOOR = 2.0 ** -50             # covers the absolute error of squares that underflow
NEAREST_NONE = F32(1e10)               # get_attr_from_closest's initial min_dist


def nearest_dist_f32(query, pos):
    """|q - p| as get_attr_from_closest evaluates it: float32, one rounding per operation, ((dx^2 + dy^2) + dz^2), sqrt."""
    with np.errstate(over="ignore", invalid="ignore", under="ignore"):
        d = np.asarray(query, F32) - np.asarray(pos, F32)
        return np.sqrt((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2])


def nearest_index(pos, query):
    """get_attr_from_closest's min_idx for every query (int32, -1 when no Gaussian has d < 1e10): the argmin of the float32
    distance, ties to the lowest index. A k-d tree gives the fp64 minimum distance d_min; every finite Gaussian within
    d_min (1 + 2^-19) + 2^-50 is a candidate (the float32 minimum lies among them), and the float32 formula decides."""
    from scipy.spatial import cKDTree
    pos = np.asarray(pos, F32).reshape(-1, 3)
    query = np.asarray(query, F32).reshape(-1, 3)
    out = np.full(len(query), -1, np.int32)
    fin = np.nonzero(np.all(np.isfinite(pos), axis=1))[0]
    live = np.nonzero(np.all(np.isfinite(query), axis=1))[0]
    if len(fin) == 0 or len(live) == 0:
        return out
    tree = cKDTree(pos[fin].astype(np.float64))
    q64 = query[live].astype(np.float64)
    dmin, first = tree.query(q64, workers=-1)
    near = dmin <= float(NEAREST_NONE) * NEAREST_SLACK             # farther: every float32 d is >= 1e10
    cand = tree.query_ball_point(q64[near], dmin[near] * NEAREST_SLACK + NEAREST_FLOOR, workers=-1)
    lone = np.fromiter(map(len, cand), np.int64, len(cand)) == 1
    qn, jn = live[near][lone], fin[first[near][lone]]               # a single candidate: the k-d tree's own nearest
    d = nearest_dist_f32(query[qn], pos[jn])
    out[qn] = np.where(d < NEAREST_NONE, jn, -1)
    for qi, c in zip(live[near][~lone], (c for c, one in zip(cand, lone) if not one)):
        j = fin[np.asarray(c, np.int64)]
        d = nearest_dist_f32(query[qi], pos[j])
        ok = d < NEAREST_NONE
        if ok.any():
            dj, jj = d[ok], j[ok]
            out[qi] = jj[dj == dj.min()].min()
    return out


def init_filled_particles(pos, shs, cov, opacity, new_pos):
    """init_filled_particles (filling.py:408-446) in numpy: (shs (N+M, K, 3), opacity (N+M, 1), cov (N+M, 6)) float32, the
    inputs first, then the rows of each new particle's nearest Gaussian. Raises ValueError where the reference would read
    index -1."""
    pos = np.asarray(pos, F32).reshape(-1, 3)
    n = len(pos)
    shs = np.asarray(shs, F32).reshape(n, -1, 3)
    cov = np.asarray(cov, F32).reshape(n, 6)
    opacity = np.asarray(opacity, F32).reshape(n, 1)
    idx = nearest_index(pos, new_pos)
    if np.any(idx < 0):
        raise ValueError(f"{int(np.sum(idx < 0))} new particles have no Gaussian closer than 1e10")
    return (np.concatenate([shs, shs[idx]]), np.concatenate([opacity, opacity[idx]]), np.concatenate([cov, cov[idx]]))
