"""Particle filling (PG/particle_filling/filling.py) at its edges. tests/golden/filling_edges_golden.npz (made by
tests/golden/make_filling_edges_golden.py from the reference's own kernels) holds
  (a) fill_dense_grids + internal_filling on hand-built (count, density) grids of 1 to 16 cells a side, for all 36
      (search_exclude_dir, ray_cast_dir) pairs: box walls on the grid faces, a holed box, alternating lines, all-dense and
      all-empty grids, densities at float32(thr) and one step either side, cells already holding 0 .. ppc + 1 Gaussians;
  (b) densify_grids on hand-built Gaussians: cell faces and nodes, clipped windows, integer window radii, degenerate
      covariances, 5000 Gaussians in one cell, and Gaussians outside the grid whose windows reach into it.
CPU: the numpy oracle against both parts, against a float64 restatement of the splat, and against a literal ray march.
GPU: the device kernels against both parts and the float64 restatement, the boundary crop at its planes, a config-size
scene at n_grid 200, and empty inputs.

Deviation from the reference, added back before exact comparison: a Gaussian outside the grid counts in its nearest border
cell (the reference's count store for it is out of range, and the fixture's lenient count field drops it).
"""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import particle_filling_ref as R  # noqa: E402

GOLDEN = os.path.join(HERE, "golden", "filling_edges_golden.npz")
F32 = np.float32
with np.load(GOLDEN) as _g:
    A_CASES = [str(s) for s in _g["a_cases"]]
    B_CASES = [str(s) for s in _g["b_cases"]]
DIRS = [(1, 0, 0), (-1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, 1), (0, 0, -1)]
GRID_DX = 0.1                          # (a): the spacing only places the new particles


@pytest.fixture(scope="module")
def golden():
    with np.load(GOLDEN) as g:
        return {k: g[k] for k in g.files}


def grid_case(g, name):
    k = f"a/{name}/"
    dthr, sthr = (float(v) for v in g[k + "thres"])
    return dict(count=g[k + "count"].astype(np.int32), density=g[k + "density"], dthr=dthr, sthr=sthr, ppc=int(g[k + "ppc"]),
                pairs=[tuple(int(v) for v in p) for p in g[k + "pairs"]], c1=g[k + "count_dense"].astype(np.int32),
                c2=g[k + "count_internal"].astype(np.int32), n_dense=int(g[k + "n_dense"]), n_total=[int(v) for v in g[k + "n_total"]])


def cell_of(pos, grid_dx):
    """The reference's cell, ti.floor(x / grid_dx) in float32, in float64 so that positions far outside cannot overflow."""
    return np.floor(np.asarray(pos, F32) / F32(grid_dx)).astype(np.float64)


def splat_case(g, name):
    """(pos, opacity, cov, grid_n, grid_dx, count, density) with the border-cell deviation added to the reference's count."""
    k = f"b/{name}/"
    pos, n, dx = g[k + "pos"], int(g[k + "grid_n"]), float(g[k + "grid_dx"])
    count = g[k + "count"].astype(np.int32)
    c0 = cell_of(pos, dx)
    off = np.any((c0 < 0) | (c0 >= n), axis=1)
    cc = np.clip(c0[off], 0, n - 1).astype(np.int64)
    np.add.at(count, (cc[:, 0], cc[:, 1], cc[:, 2]), 1)
    return pos, g[k + "opacity"], g[k + "cov"], n, dx, count, g[k + "density"]


def assert_density(got, want, rtol):
    # densities are compared at the scale of the thresholds (O(1)); tails far below it only need the absolute bound
    np.testing.assert_allclose(got, want, rtol=rtol, atol=1e-6)


def rtol_needed(got, want, atol=1e-6):
    """The smallest rtol with which assert_density(got, want, rtol) passes (assert_allclose's |d| <= atol + rtol |want|)."""
    excess = np.abs(np.asarray(got, np.float64) - want) - atol
    bad = excess > 0
    return float(np.max(excess[bad] / np.abs(want[bad]), initial=0.0))


def density_fp64(pos, opacity, cov, grid_n, grid_dx):
    """densify_grids and compute_density (filling.py:13-87) in float64: exact eigh, eigenvalues clamped at 1e-8, the window
    [c0 - r, c0 + r] unclamped and cells outside the grid skipped one by one. The integer decisions are the reference's
    float32 ones: the cell c0 = floor(x / grid_dx), and r = ceil(sqrt(max sigma) / grid_dx) from the eigenvalue rounded to
    float32 (in float64, a sigma one float32 step above (k dx)^2 would give radius k + 1 instead of k)."""
    pos, dx, n = np.asarray(pos, F32).astype(np.float64), float(F32(grid_dx)), int(grid_n)
    c0 = cell_of(pos, grid_dx)
    cov = np.asarray(cov, F32).astype(np.float64)
    corners = np.array([(a, b, c) for a in range(2) for b in range(2) for c in range(2)])
    density = np.zeros((n, n, n))
    for g in range(len(pos)):
        w, V = np.linalg.eigh(cov[g, [0, 1, 2, 1, 3, 4, 2, 4, 5]].reshape(3, 3))
        w = np.maximum(w, 1e-8)
        P = (V / w) @ V.T
        r = int(np.ceil(np.sqrt(F32(w.max())) / F32(grid_dx)))
        cells = [np.arange(c - r, c + r + 1) for c in c0[g]]
        cells = [a[(a >= 0) & (a < n)].astype(np.int64) for a in cells]
        if not all(len(a) for a in cells):
            continue
        cell = np.stack(np.meshgrid(*cells, indexing="ij"), axis=-1).reshape(-1, 3)
        d = pos[g] - (cell[:, None, :] + corners[None]) * dx                       # (W, 8, 3)
        e = np.einsum("wci,ij,wcj->wc", d, P, d)
        density[cell[:, 0], cell[:, 1], cell[:, 2]] += float(opacity[g]) * np.exp(-0.5 * e).sum(1) / 8.0
    return density


def ray_march(density, thres):
    """collision_search and collision_times (filling.py:117-181) as written: one march per cell and direction. Returns
    hit[d] (a cell beyond along d is denser than thres) and times[d] (false -> true changes beyond, from state false: the
    count grid is 0 at every cell internal_filling tests)."""
    n = density.shape[0]
    t = F32(thres)
    hit = np.zeros((6,) + density.shape, bool)
    times = np.zeros((6,) + density.shape, np.int64)
    for c in np.ndindex(*density.shape):
        for d, step in enumerate(DIRS):
            i, j, k = (c[q] + step[q] for q in range(3))
            state, flag, count = False, False, 0
            while max(i, j, k) < n and min(i, j, k) >= 0:
                new = bool(density[i, j, k] > t)
                flag = flag or new
                if new != state and not state:
                    count += 1
                state = new
                i, j, k = i + step[0], j + step[1], k + step[2]
            hit[d][c], times[d][c] = flag, count
    return hit, times


def cells_of(new, grid_dx, origin, grid_n):
    """Cell of every new particle (float64 arithmetic) and the largest distance outside that cell, in units of grid_dx."""
    q = (np.asarray(new, np.float64) - origin) / grid_dx
    c = np.clip(np.floor(q), 0, grid_n - 1)
    return c.astype(np.int64), float(np.max(np.maximum(c - q, q - (c + 1)), initial=-1.0))


def per_cell(cells, grid_n):
    h = np.zeros(grid_n ** 3, np.int64)
    np.add.at(h, (cells[:, 0] * grid_n + cells[:, 1]) * grid_n + cells[:, 2], 1)
    return h.reshape((grid_n,) * 3)


def rotated_covs(rng, n, lo, hi):
    s = rng.uniform(lo, hi, size=(n, 3))
    Q, _ = np.linalg.qr(rng.standard_normal((n, 3, 3)))
    m = Q @ (s[:, :, None] ** 2 * np.eye(3)) @ Q.transpose(0, 2, 1)
    return np.stack([m[:, 0, 0], m[:, 0, 1], m[:, 0, 2], m[:, 1, 1], m[:, 1, 2], m[:, 2, 2]], axis=1).astype(F32)


def offgrid_scene(seed, n, dx, N=60):
    """Rotated Gaussians spread over [-0.6, 1.6] x the grid's extent: about two thirds outside it, many reaching in, some
    with windows wider than the grid."""
    rng = np.random.default_rng(seed)
    pos = (rng.uniform(-0.6, 1.6, size=(N, 3)) * n * dx).astype(F32)
    return pos, rng.uniform(0.2, 1.0, N).astype(F32), rotated_covs(rng, N, 0.3 * n * dx / 8, 1.5 * n * dx)


# ------------------------------------------------------------------------------------------------------------------ CPU
def test_fixture_covers_the_edges(golden):
    """What the fixture is there for: every pair, grids of 1-3 cells, 12^2 not a multiple of 128, densities on the
    thresholds, held counts up to ppc + 1, and off-grid Gaussians whose windows reach the grid."""
    pairs = set()
    sizes = set()
    for name in A_CASES:
        c = grid_case(golden, name)
        pairs |= set(c["pairs"])
        sizes.add(c["density"].shape[0])
        if "thres" in name:
            for t in (c["dthr"], c["sthr"]):
                for v in (np.nextafter(F32(t), F32(-1)), F32(t), np.nextafter(F32(t), F32(np.inf))):
                    assert np.any(c["density"] == v), (name, t)
        if "held_ppc" in name:
            assert set(np.unique(c["count"])) >= {0, 1, c["ppc"] - 1, c["ppc"], c["ppc"] + 1}
    assert pairs == {(e, r) for e in range(6) for r in range(6)}
    assert {1, 2, 3, 7, 12, 16} <= sizes
    pos, _, _, n, dx, count, density = splat_case(golden, "offgrid")
    c0 = cell_of(pos, dx)
    assert np.all(np.any((c0 < 0) | (c0 >= n), axis=1)) and density.min() > 1
    pos, _, _, n, dx, _, density = splat_case(golden, "offgrid_one")
    assert cell_of(pos, dx)[0, 0] == -4 and np.all(density.sum(axis=(1, 2)) > 1)      # every x-slab, from 4 cells out


@pytest.mark.parametrize("name", A_CASES)
def test_oracle_fill_grids_matches_reference(golden, name):
    c = grid_case(golden, name)
    for p, (e, r) in enumerate(c["pairs"]):
        c1, c2, add_d, add_i = R.fill_grids(c["count"], c["density"], c["dthr"], c["sthr"], c["ppc"], e, r)
        assert np.array_equal(c1, c["c1"]), (e, r)
        assert np.array_equal(c2, c["c2"][p]), (e, r)
        assert (int(add_d.sum()), int(add_d.sum() + add_i.sum())) == (c["n_dense"], c["n_total"][p])


@pytest.mark.parametrize("name", B_CASES)
def test_oracle_densify_matches_reference(golden, name):
    pos, opacity, cov, n, dx, count, density = splat_case(golden, name)
    got_count, got_density = R.densify_grids(pos, opacity, cov, n, dx)
    assert np.array_equal(got_count, count)
    assert_density(got_density, density, 1e-6)


def test_oracle_off_grid_window_reaches_across_the_grid():
    """One isotropic Gaussian (sigma = 2) at x = -0.5, four cells outside an 8-cell grid of 0.125: its window of radius 12
    covers every x-slab. Clamping the radius to grid_n instead left slabs 5-7 at 0."""
    pos, op, cov = [[-0.5, 0.5, 0.5]], [1.0], [[2.0, 0, 0, 2.0, 0, 2.0]]
    count, density = R.densify_grids(pos, op, cov, 8, 0.125)
    want = density_fp64(pos, op, cov, 8, 0.125)
    assert count.sum() == 1 and count[0, 4, 4] == 1
    assert np.all(density.sum(axis=(1, 2)) > 30)
    assert_density(density, want, 2e-6)


@pytest.mark.parametrize("seed", range(6))
def test_oracle_matches_fp64_restatement(seed):
    n, dx = (8, 0.125) if seed % 2 else (10, 0.1)
    pos, opacity, cov = offgrid_scene(seed, n, dx)
    _, density = R.densify_grids(pos, opacity, cov, n, dx)
    want = density_fp64(pos, opacity, cov, n, dx)
    assert want.max() > 0.5
    assert_density(density, want, 1e-5)


def ray_grids():
    rng = np.random.default_rng(77)
    t = F32(0.3)
    vals = np.array([0.0, np.nextafter(t, F32(0)), t, np.nextafter(t, F32(1)), 1.0], F32)
    for n in (1, 2, 5, 9):
        for f in (0.2, 0.5, 0.8):
            yield n, vals[np.where(rng.random((n, n, n)) < f, rng.integers(1, 5, (n, n, n)), 0)]


def test_oracle_classify_matches_literal_ray_march():
    """classify's suffix OR / suffix run count per axis line against the reference's per-cell ray march, all 36 pairs, on
    random grids that hold densities at float32(0.3) and one step either side."""
    for n, density in ray_grids():
        hit, times = ray_march(density, 0.3)
        for e in range(6):
            enclosed = np.all(hit[[d for d in range(6) if d != e]], axis=0)
            for r in range(6):
                got_enclosed, got_odd = R.classify(density, 0.3, e, r)
                assert np.array_equal(got_enclosed, enclosed), (n, e, r)
                assert np.array_equal(got_odd, times[r] % 2 == 1), (n, e, r)


# ------------------------------------------------------------------------------------------------------------------ GPU
def _dev(x, dev):
    return torch.from_numpy(np.ascontiguousarray(x)).to(dev)


@pytest.mark.gpu
def test_device_fill_grids_matches_reference(built_lib, cuda_dev, golden):
    """Every case and pair of part (a): the count grid after both fills, n_dense and n_total exact; every new particle in
    its cell, dense and interior parts counted separately; a second call bit-identical (fill_grids has no atomics)."""
    from pixie_b200 import particle_filling as PF
    for name in A_CASES:
        c = grid_case(golden, name)
        n = c["density"].shape[0]
        dens = _dev(c["density"], cuda_dev)
        cap = n ** 3 * c["ppc"]
        for p, (e, r) in enumerate(c["pairs"]):
            outs = []
            for _ in range(2):
                count = _dev(c["count"], cuda_dev)
                new, n_dense = PF.fill_grids(count, dens, GRID_DX, cap, c["dthr"], c["sthr"], c["ppc"], e, r, seed=9)
                assert np.array_equal(count.cpu().numpy(), c["c2"][p]), (name, e, r)
                assert (n_dense, new.shape[0]) == (c["n_dense"], c["n_total"][p]), (name, e, r)
                outs.append(new)
            assert torch.equal(outs[0], outs[1]), (name, e, r)
            cells, outside = cells_of(outs[0].cpu().numpy(), GRID_DX, np.zeros(3), n)
            assert outside <= 1e-5, (name, e, r, outside)
            assert np.array_equal(per_cell(cells[:n_dense], n), c["c1"] - c["count"]), (name, e, r)
            assert np.array_equal(per_cell(cells[n_dense:], n), c["c2"][p] - c["c1"]), (name, e, r)


@pytest.mark.gpu
def test_device_densify_matches_reference_and_fp64(built_lib, cuda_dev, golden):
    """Every case of part (b): counts exact; densities within 1e-5 of the reference's kernels (the bound of
    test_particle_filling.py), and within 1.2e-5 of the float64 restatement (rtol, with atol 1e-6). Measured on an H100
    80GB HBM3 (700 W): the largest rtol needed was 3.6e-6 against the reference and 2.8e-6 against float64, both in the
    cell holding 5000 Gaussians, where float atomics sum in a different order; every other case needed at most 1.7e-7."""
    from pixie_b200 import particle_filling as PF
    worst_ref, worst_fp64 = {}, {}
    for name in B_CASES:
        pos, opacity, cov, n, dx, want_count, want_density = splat_case(golden, name)
        count, density = PF.densify_grids(_dev(pos, cuda_dev), _dev(opacity, cuda_dev), _dev(cov, cuda_dev), n, dx)
        got = density.cpu().numpy()
        assert np.array_equal(count.cpu().numpy(), want_count), name
        fp64 = density_fp64(pos, opacity, cov, n, dx)
        worst_ref[name], worst_fp64[name] = rtol_needed(got, want_density), rtol_needed(got, fp64)
        print(f"{name}: rtol needed {worst_ref[name]:.3g} vs reference, {worst_fp64[name]:.3g} vs fp64")
    assert max(worst_ref.values()) <= 1e-5, worst_ref
    assert max(worst_fp64.values()) <= 1.2e-5, worst_fp64


@pytest.mark.gpu
def test_device_crop_at_boundary_planes(built_lib, cuda_dev):
    """fill_particles keeps the Gaussians strictly inside the boundary: one Gaussian exactly on each of the six planes is
    dropped, one a float32 step inside is kept. The step inside the upper x plane has (p - x0) / dx rounding to grid_n, so
    it counts in the border cell. Against the oracle, cell for cell."""
    from pixie_b200 import particle_filling as PF
    b, n = [0.07, 0.97, 0.3, 1.1, 0.1, 0.8], 8
    lo, hi = np.array(b[::2], F32), np.array(b[1::2], F32)
    rng = np.random.default_rng(3)
    bulk = lo + rng.uniform(0.1, 0.9, size=(200, 3)).astype(F32) * (hi - lo)
    planes, inside = [], []
    for axis in range(3):
        for v, step in ((lo[axis], np.nextafter(lo[axis], F32(2))), (hi[axis], np.nextafter(hi[axis], F32(-2)))):
            for q, keep in ((v, False), (step, True)):
                p = lo + rng.uniform(0.2, 0.8, 3).astype(F32) * (hi - lo)
                p[axis] = q
                planes.append(p)
                inside.append(keep)
    pos = np.concatenate([bulk, np.array(planes, F32)]).astype(F32)
    dx = max(b[2 * i + 1] - b[2 * i] for i in range(3)) / n
    assert np.floor((np.nextafter(hi[0], F32(-2)) - lo[0]) / F32(dx)) == n
    N = len(pos)
    opacity = np.ones(N, F32)
    cov = np.tile(np.array([1, 0, 0, 1, 0, 1], F32) * F32((0.4 * dx) ** 2), (N, 1))
    kw = dict(grid_n=n, max_samples=10_000, grid_dx=1.0, density_thres=0.02, search_thres=0.5, max_particles_per_cell=2,
              search_exclude_dir=5, ray_cast_dir=4, boundary=b)
    want = R.fill_particles(pos, opacity, cov, **kw)
    assert want["count"].sum() == len(bulk) + sum(inside)
    out = PF.fill_particles(_dev(pos, cuda_dev), _dev(opacity, cuda_dev), _dev(cov, cuda_dev), seed=2, **kw)
    assert torch.equal(out[:N].cpu(), torch.from_numpy(pos)) and out.shape[0] == N + want["n_total"]
    cells, outside = cells_of(out[N:].cpu().numpy(), want["grid_dx"], want["origin"].astype(np.float64), n)
    assert outside <= 1e-5
    assert np.array_equal(per_cell(cells[:want["n_dense"]], n), want["add_dense"])
    assert np.array_equal(per_cell(cells[want["n_dense"]:], n), want["add_interior"])
    # without the twelve plane Gaussians, the Gaussians on the planes and a step inside change the result
    less = R.fill_particles(bulk, opacity[:len(bulk)], cov[:len(bulk)], **kw)
    assert not np.array_equal(less["count_internal"], want["count_internal"])


def shell(n, center, radius, std, seed):
    rng = np.random.default_rng(seed)
    v = rng.standard_normal((n, 3))
    pos = (center + radius * (1 + 0.01 * rng.standard_normal((n, 1))) * v / np.linalg.norm(v, axis=1, keepdims=True)).astype(F32)
    return pos, rng.uniform(0.3, 1.0, n).astype(F32), rotated_covs(rng, n, 0.5 * std, 1.5 * std)


def clear_of(density, thr):
    """A threshold no cell density lies within 1e-5 (relative) of, near `thr`."""
    for k in range(1000):
        t = thr * (1 + 3e-5 * k)
        if not np.any(np.abs(density.astype(np.float64) - t) <= 1e-5 * t):
            return t
    raise AssertionError("no clear threshold")


@pytest.mark.gpu
def test_device_matches_oracle_at_n_grid_200(built_lib, cuda_dev):
    """The default filling grid of the 50-cell configs (4 x n_grid = 200) over the metal boundary: 1M Gaussians on a shell,
    thresholds moved clear of every cell density. Count grid after both fills, n_dense and n_total equal the oracle's."""
    from pixie_b200 import particle_filling as PF
    b, n = [0.86, 1.46, 0.7, 1.3, 0.7, 1.3], 200
    pos, opacity, cov = shell(1_000_000, np.array([1.16, 1.0, 1.0]), 0.22, 0.0015, seed=12)
    lo = np.array(b[::2], F32)
    dx = 0.6 / n
    count, density = R.densify_grids(pos - lo, opacity, cov, n, dx)
    dthr = clear_of(density, float(np.percentile(density[density > 0], 30)))
    sthr = clear_of(density, dthr / 10)
    c1, c2, add_d, add_i = R.fill_grids(count, density, dthr, sthr, 1, 0, 1)
    n_dense, n_total = int(add_d.sum()), int(add_d.sum() + add_i.sum())
    assert n_total - n_dense > 100_000 and n_dense > 1000
    gcount, gdensity = PF.densify_grids(_dev(pos - lo, cuda_dev), _dev(opacity, cuda_dev), _dev(cov, cuda_dev), n, dx)
    assert np.array_equal(gcount.cpu().numpy(), count)
    assert_density(gdensity.cpu().numpy(), density, 1e-5)
    new, got_dense = PF.fill_grids(gcount, gdensity, dx, 2_000_000, dthr, sthr, 1, 0, 1, tuple(float(v) for v in lo))
    assert (got_dense, new.shape[0]) == (n_dense, n_total)
    assert np.array_equal(gcount.cpu().numpy(), c2)


@pytest.mark.gpu
def test_device_empty_inputs(built_lib, cuda_dev):
    """No Gaussians, an all-empty grid (a (0, 3) result) and max_samples = 0."""
    from pixie_b200 import _lib
    from pixie_b200 import particle_filling as PF
    z3, z1, z6 = (torch.zeros((0, k), device=cuda_dev) for k in (3, 1, 6))
    count, density = PF.densify_grids(z3, z1, z6, 5, 0.1)
    assert count.shape == (5, 5, 5) and not count.any() and not density.any()
    new, n_dense = PF.fill_grids(count, density, 0.1, 100)
    assert new.shape == (0, 3) and n_dense == 0
    new, n_dense = PF.fill_grids(count, density, 0.1, 0)
    assert new.shape == (0, 3) and n_dense == 0
    out = PF.fill_particles(z3, z1, z6, 5, 100, 0.1)
    assert out.shape == (0, 3)
    out = PF.fill_particles(z3, z1, z6, 5, 0, 0.1, boundary=[0, 1, 0, 1, 0, 1])
    assert out.shape == (0, 3)
    # one dense cell needs one particle: max_samples = 0 refuses it, 1 takes it
    density[2, 2, 2] = 10.0
    with pytest.raises(_lib.PixieError, match="adds 1 particles"):
        PF.fill_grids(count.clone(), density, 0.1, 0)
    new, n_dense = PF.fill_grids(count, density, 0.1, 1)
    assert new.shape == (1, 3) and n_dense == 1 and int(count[2, 2, 2]) == 1
