"""Particle filling of hollow Gaussian objects, on the device (PG/particle_filling/filling.py:291-380, Taichi in the reference).

A trained Gaussian Splatting scene puts its Gaussians on the object's surface; without filling, MPM simulates a hollow shell
that buckles like a sheet. `fill_particles` adds particles to the cells the Gaussians make dense and to the cells they
enclose, with the reference's names, arguments and defaults:

    fill_particles(pos, opacity, cov, grid_n, max_samples, grid_dx, density_thres=2.0, search_thres=1.0,
                   max_particles_per_cell=1, search_exclude_dir=5, ray_cast_dir=4, boundary=None, smooth=False, seed=0)
    decode_filling_params(filling, material_params)          utils/decode_param.py:177-208 (defaults of the config block)
    init_filled_particles(pos, shs, cov, opacity, new_pos)   filling.py:383-446 (`visualize`: each new particle takes the
                                                             SH, opacity and covariance of its nearest Gaussian)

Deviations from the reference: new particles come in a fixed order (dense cells first, then interior cells, each in C order
of cells) with offsets drawn from a counter-based generator keyed on `seed`; a total above `max_samples` raises instead of
writing out of bounds; a Gaussian outside the grid counts in the nearest border cell; `smooth` (PyMCubes constrained
smoothing) is not available. `init_filled_particles` finds the same nearest Gaussian as the reference's brute-force loop
(same float32 distance, ties to the lowest index) through a tree instead of O(M N) work; where the reference would read
index -1 (no Gaussian closer than 1e10: none at all, a NaN query, or all that far) it raises; with no new particles it
returns its inputs. No CPU fallback.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional, Sequence, Tuple

import torch

from . import _lib

_DIRS = "0: +x, 1: -x, 2: +y, 3: -y, 4: +z, 5: -z"


def decode_filling_params(filling: Dict, material_params: Dict) -> Dict:
    """The `particle_filling` block of a physics config with the defaults of decode_param.py:177-208 (a new dict; the
    reference fills them in place). `max_partciels_per_cell` is the reference's own spelling of the key."""
    p = dict(filling)
    p.setdefault("n_grid", material_params["n_grid"] * 4)
    p.setdefault("density_threshold", 5.0)
    p.setdefault("search_threshold", 3.0)
    p.setdefault("max_particles_num", 2000000)
    p.setdefault("max_partciels_per_cell", 1)
    p.setdefault("search_exclude_direction", 5)
    p.setdefault("ray_cast_direction", 4)
    p.setdefault("boundary", None)
    p.setdefault("smooth", False)
    p.setdefault("visualize", False)
    return p


def _check_grid_n(grid_n: int):
    if int(grid_n) < 1:
        raise ValueError(f"grid_n must be >= 1, got {grid_n}")


def densify_grids(pos: torch.Tensor, opacity: torch.Tensor, cov: torch.Tensor, grid_n: int, grid_dx: float) -> Tuple[torch.Tensor, torch.Tensor]:
    """densify_grids (filling.py:26-87): (count int32, density float32), both (grid_n, grid_n, grid_n), for Gaussians whose
    positions are already in the grid's frame."""
    _check_grid_n(grid_n)
    _lib.require_device()
    _lib.require_cuda("densify_grids", pos, opacity, cov)
    p = pos.detach().reshape(-1, 3).to(torch.float32).contiguous()
    o = opacity.detach().reshape(-1).to(p.device, torch.float32).contiguous()
    c = cov.detach().reshape(-1, 6).to(p.device, torch.float32).contiguous()
    n = p.shape[0]
    if o.shape[0] != n or c.shape[0] != n:
        raise ValueError(f"pos, opacity and cov disagree on the Gaussian count ({n}, {o.shape[0]}, {c.shape[0]})")
    g = int(grid_n)
    count = torch.empty((g, g, g), dtype=torch.int32, device=p.device)
    density = torch.empty((g, g, g), dtype=torch.float32, device=p.device)
    _lib.call("pixie_fill_density", p.device, p, o, c, n, g, float(grid_dx), count, density)
    return count, density


def fill_grids(count: torch.Tensor, density: torch.Tensor, grid_dx: float, max_samples: int, density_thres: float = 2.0,
               search_thres: float = 1.0, max_particles_per_cell: int = 1, search_exclude_dir: int = 5, ray_cast_dir: int = 4,
               origin: Sequence[float] = (0.0, 0.0, 0.0), seed: int = 0) -> Tuple[torch.Tensor, int]:
    """fill_dense_grids + internal_filling (filling.py:90-234) on the grids of `densify_grids`: returns the new particles
    (m, 3) float32, shifted by `origin`, and how many of them (the first ones) went to dense cells. `count` is updated in
    place like the reference's grid. Raises PixieError when more than `max_samples` particles would be added."""
    for name, d in (("search_exclude_dir", search_exclude_dir), ("ray_cast_dir", ray_cast_dir)):
        if not 0 <= int(d) <= 5:
            raise ValueError(f"{name} must be in 0..5 ({_DIRS}), got {d}")
    if int(max_particles_per_cell) < 1:
        raise ValueError(f"max_particles_per_cell must be >= 1, got {max_particles_per_cell}")
    _lib.require_device()
    _lib.require_cuda("fill_grids", count, density)
    g = count.shape[0]
    if count.dtype != torch.int32 or density.dtype != torch.float32 or tuple(count.shape) != (g, g, g) or density.shape != count.shape \
            or not count.is_contiguous() or not density.is_contiguous():
        raise ValueError("count / density must be contiguous (n, n, n) int32 / float32 grids")
    dev = count.device
    n_dense, n_total = C.c_int(0), C.c_int(0)
    out = torch.empty((max(int(max_samples), 0), 3), dtype=torch.float32, device=dev)
    _lib.call("pixie_fill_grids", dev, count, density, g, float(grid_dx), (C.c_float * 3)(*[float(v) for v in origin]),
              float(density_thres), float(search_thres), int(max_particles_per_cell), int(search_exclude_dir), int(ray_cast_dir),
              int(seed) & (2 ** 64 - 1), out, int(max_samples), C.byref(n_dense), C.byref(n_total))
    return out[:n_total.value], n_dense.value


def fill_particles(pos: torch.Tensor, opacity: torch.Tensor, cov: torch.Tensor, grid_n: int, max_samples: int, grid_dx: float,
                   density_thres=2.0, search_thres=1.0, max_particles_per_cell=1, search_exclude_dir=5, ray_cast_dir=4,
                   boundary: Optional[list] = None, smooth: bool = False, *, seed: int = 0) -> torch.Tensor:
    """fill_particles (filling.py:291-380): cat([pos, new particles]) float32 on pos's device. With `boundary`
    [x0, x1, y0, y1, z0, z1], only the Gaussians strictly inside it are splatted, on a grid of spacing
    max extent / grid_n (grid_dx is then ignored) anchored at (x0, y0, z0); every input Gaussian is still returned first."""
    if smooth:
        raise NotImplementedError(
            "particle filling with smooth=True runs mcubes.smooth(..., 'constrained') on the density field; PyMCubes is neither "
            "vendored nor installable here, so that step can be neither reproduced nor pinned")
    _check_grid_n(grid_n)
    for name, d in (("search_exclude_dir", search_exclude_dir), ("ray_cast_dir", ray_cast_dir)):
        if not 0 <= int(d) <= 5:
            raise ValueError(f"{name} must be in 0..5 ({_DIRS}), got {d}")
    if pos.dim() != 2 or pos.shape[1] != 3:
        raise ValueError(f"pos must be (N, 3), got {tuple(pos.shape)}")
    n = pos.shape[0]
    if opacity.numel() != n or cov.numel() != 6 * n:
        raise ValueError(f"opacity must hold N and cov N x 6 values for N = {n} Gaussians, got {tuple(opacity.shape)} and {tuple(cov.shape)}")
    if boundary is not None and len(boundary) != 6:
        raise ValueError("boundary must be [x0, x1, y0, y1, z0, z1]")
    _lib.require_cuda("fill_particles", pos, opacity, cov)
    pos_clone = pos.detach().to(torch.float32).clone()
    p, o, c = pos_clone, opacity.detach().reshape(-1), cov.detach().reshape(-1, 6)
    origin = (0.0, 0.0, 0.0)
    if boundary is not None:
        # torch compares the float32 tensor against float32(boundary); grid_dx from the extents in double (filling.py:306-322)
        mask = torch.ones(n, dtype=torch.bool, device=p.device)
        max_diff = 0.0
        for i in range(3):
            mask = torch.logical_and(mask, p[:, i] > boundary[2 * i])
            mask = torch.logical_and(mask, p[:, i] < boundary[2 * i + 1])
            max_diff = max(max_diff, boundary[2 * i + 1] - boundary[2 * i])
        new_origin = torch.tensor([boundary[0], boundary[2], boundary[4]], dtype=torch.float32, device=p.device)
        p, o, c = p[mask] - new_origin, o[mask], c[mask]
        grid_dx = max_diff / grid_n
        origin = [float(v) for v in new_origin.cpu()]
    count, density = densify_grids(p, o, c, grid_n, grid_dx)
    new, _ = fill_grids(count, density, grid_dx, max_samples, density_thres, search_thres, max_particles_per_cell, search_exclude_dir,
                        ray_cast_dir, origin, seed)
    return torch.cat([pos_clone, new], dim=0)


def nearest_gaussian(pos: torch.Tensor, query: torch.Tensor) -> torch.Tensor:
    """The search of get_attr_from_closest (filling.py:383-405): (M,) int32, for each query the index of the Gaussian at
    the smallest float32 distance (ties to the lowest index), or -1 when none is closer than 1e10. Exact, on the device."""
    _lib.require_device()
    _lib.require_cuda("nearest_gaussian", pos, query)
    if pos.dim() != 2 or pos.shape[1] != 3 or query.dim() != 2 or query.shape[1] != 3:
        raise ValueError(f"pos and query must be (N, 3) and (M, 3), got {tuple(pos.shape)} and {tuple(query.shape)}")
    dev = query.device
    p = pos.detach().to(dev, torch.float32).contiguous()
    q = query.detach().to(torch.float32).contiguous()
    index = torch.empty(q.shape[0], dtype=torch.int32, device=dev)
    _lib.call("pixie_nearest_gaussian", dev, p, p.shape[0], q, q.shape[0], index)
    return index


def init_filled_particles(pos: torch.Tensor, shs: torch.Tensor, cov: torch.Tensor, opacity: torch.Tensor,
                          new_pos: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """init_filled_particles (filling.py:408-446), the `particle_filling.visualize` step: every new particle takes the SH,
    opacity and covariance of its nearest Gaussian. pos (N, 3), shs (N, K, 3) with K in 1, 4, 9, 16, cov (N, 6), opacity
    (N, 1) or (N,), new_pos (M, 3); returns (shs (N+M, K, 3), opacity (N+M, 1), cov (N+M, 6)) float32 on pos's device, the
    Gaussians' rows first, then the copied rows bit for bit. Raises PixieError when a new particle has no Gaussian closer
    than 1e10 (the reference would read index -1). With M = 0 the inputs come back in those shapes."""
    if pos.dim() != 2 or pos.shape[1] != 3:
        raise ValueError(f"pos must be (N, 3), got {tuple(pos.shape)}")
    n = pos.shape[0]
    if shs.dim() != 3 or shs.shape[0] != n or shs.shape[1] not in (1, 4, 9, 16) or shs.shape[2] != 3:
        raise ValueError(f"shs must be (N, K, 3) with K in 1, 4, 9, 16 for N = {n} Gaussians, got {tuple(shs.shape)}")
    if opacity.numel() != n or cov.numel() != 6 * n:
        raise ValueError(f"opacity must hold N and cov N x 6 values for N = {n} Gaussians, got {tuple(opacity.shape)} and {tuple(cov.shape)}")
    if new_pos.dim() != 2 or new_pos.shape[1] != 3:
        raise ValueError(f"new_pos must be (M, 3), got {tuple(new_pos.shape)}")
    _lib.require_cuda("init_filled_particles", pos, shs, cov, opacity, new_pos)
    dev = pos.device
    s = shs.detach().to(dev, torch.float32)
    o = opacity.detach().to(dev, torch.float32).reshape(n, 1)
    c = cov.detach().to(dev, torch.float32).reshape(n, 6)
    if new_pos.shape[0] == 0:
        return s.clone(), o.clone(), c.clone()
    index = nearest_gaussian(pos, new_pos.to(dev))
    missing = int((index < 0).sum())
    if missing:
        raise _lib.PixieError(f"init_filled_particles: {missing} of {index.shape[0]} new particles have no Gaussian closer than 1e10")
    idx = index.long()
    return (torch.cat([s, torch.index_select(s, 0, idx)]), torch.cat([o, torch.index_select(o, 0, idx)]),
            torch.cat([c, torch.index_select(c, 0, idx)]))
