"""Generates tests/golden/filling_edges_golden.npz by EXECUTING THE REFERENCE'S OWN particle-filling kernels
(PG/particle_filling/filling.py) on the float32 / int32 `ti` stand-in of _fake_taichi.py, at the edges the scenes of
filling_golden.npz leave open. PIXIE_REFERENCE names a checkout of the reference:

    python tests/golden/make_filling_edges_golden.py

(a) `fill_dense_grids`, then `internal_filling` once per (search_exclude_dir, ray_cast_dir) pair, on hand-built
    (count, density) grids of 1 to 16 cells a side: random fields, hollow boxes whose walls lie on the grid faces, a box with
    a hole in one face, alternating planes and checkerboards, all-dense and all-empty grids, densities at exactly float32(thr)
    and one float32 step either side of both thresholds, and cells already holding 0, 1, ppc - 1, ppc and ppc + 1
    Gaussians. All 36 pairs run at up to 12 cells a side, six pairs at 16. Records the count grid after each kernel.
(b) `densify_grids` on hand-built Gaussians: positions on cell faces and nodes and one float32 step either side, windows
    clipped at faces and corners, diagonal covariances whose window radius is exactly an integer, degenerate covariances,
    5000 Gaussians in one cell, and Gaussians outside the grid beyond each face. Records the count and density grids.

The count write of a Gaussian outside the grid is an out-of-range store in the reference (undefined); cases holding such a
Gaussian run with a lenient count field that drops it. Hand-built density grids need no margin screening, and diagonal
covariances have exact eigenvalues; a seed with rotated covariances is rejected when a window radius sqrt(max sigma) / dx
lies within 1e-4 of an integer, so that eigensolver rounding cannot change a window.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import _fake_taichi as fti  # noqa: E402
from make_filling_golden import covs, load_reference, rand_rot, upper  # noqa: E402

F32 = np.float32
ALL_PAIRS = [(e, r) for e in range(6) for r in range(6)]
# the shipped configs' pairs (5, 4), (0, 1), (2, 4), exclude == ray, and two more
SOME_PAIRS = [(5, 4), (0, 1), (2, 4), (3, 3), (1, 0), (4, 5)]
DENSE = F32(10.0)


def walls(n, lo, hi):
    """The cell faces of the cube [lo, hi]^3 (cell indices)."""
    m = np.zeros((n, n, n), bool)
    m[lo:hi + 1, lo:hi + 1, lo:hi + 1] = True
    m[lo + 1:hi, lo + 1:hi, lo + 1:hi] = False
    return m


def steps(t):
    """float32(t) and one float32 step either side."""
    t = F32(t)
    return [np.nextafter(t, F32(-np.inf)), t, np.nextafter(t, F32(np.inf))]


def grid_cases():
    """[(name, count uint8, density float32, density_thres, search_thres, ppc, pairs)] of part (a)."""
    rng = np.random.default_rng(1234)
    out = []

    def add(name, d, thres=(5.0, 3.0), ppc=1, count=None, pairs=ALL_PAIRS):
        d = np.where(d, DENSE, F32(0.0)) if d.dtype == bool else d.astype(F32)
        c = np.zeros(d.shape, np.uint8) if count is None else count.astype(np.uint8)
        out.append((name, c, d, float(thres[0]), float(thres[1]), int(ppc), np.array(pairs, np.int8)))

    def hole(n, w):                                              # a hole of w x w cells in the -z face of the box on the faces
        m = walls(n, 0, n - 1)
        a = (n - w) // 2
        m[a:a + w, a:a + w, 0] = False
        return m

    ijk = np.indices((12, 12, 12))
    add("n1_dense", np.ones((1, 1, 1), bool))
    add("n1_empty", np.zeros((1, 1, 1), bool))
    add("n1_held", np.ones((1, 1, 1), bool), ppc=2, count=np.ones((1, 1, 1)))
    add("n2_random", rng.random((2, 2, 2)) < 0.5)
    add("n2_dense", np.ones((2, 2, 2), bool))
    add("n3_box", walls(3, 0, 2))
    add("n3_hole", hole(3, 1))
    add("n3_random", rng.random((3, 3, 3)) < 0.6)
    add("n7_box", walls(7, 0, 6))
    add("n7_hole", hole(7, 1))
    add("n7_random", rng.random((7, 7, 7)) < 0.3)
    add("n7_checker", np.indices((7, 7, 7)).sum(0) % 2 == 0)
    for f in (0.1, 0.3, 0.6):
        add(f"n12_random{int(f * 10)}", rng.random((12, 12, 12)) < f)
    add("n12_box", walls(12, 0, 11))
    add("n12_nested", walls(12, 0, 11) | walls(12, 3, 8))
    add("n12_hole", hole(12, 2))
    add("n12_planes", ijk[2] % 2 == 0)                           # every +-z line alternates: 6 runs
    add("n12_lines", (ijk[0] + ijk[2]) % 2 == 0)                 # alternating along x and z, constant along y
    add("n12_checker", ijk.sum(0) % 2 == 0)
    add("n12_all_dense", np.ones((12, 12, 12), bool))
    add("n12_all_empty", np.zeros((12, 12, 12), bool))
    # densities at float32(thr) and one step either side of both thresholds, the search threshold above and below
    for dthr, sthr in ((0.1, 0.3), (0.3, 0.1), (5.0, 40.0), (40.0, 5.0)):
        vals = np.array([0.0] + steps(dthr) + steps(sthr), F32)
        d = vals[rng.choice(len(vals), size=(12, 12, 12), p=[0.3] + [0.7 / 6] * 6)]
        add(f"n12_thres_{dthr:g}_{sthr:g}", d, thres=(dthr, sthr))
    # cells already holding 0, 1, ppc - 1, ppc and ppc + 1 Gaussians; densities above both, between and below the thresholds
    for ppc in (1, 2, 3):
        held = np.array([0, 1, ppc - 1, ppc, ppc + 1])
        c = np.where(rng.random((12, 12, 12)) < 0.5, 0, held[rng.integers(0, 5, (12, 12, 12))])
        d = np.array([0.0, 2.0, 6.0], F32)[rng.choice(3, size=(12, 12, 12), p=[0.4, 0.25, 0.35])]
        add(f"n12_held_ppc{ppc}", d, thres=(5.0, 1.0), ppc=ppc, count=c)
    ijk = np.indices((16, 16, 16))
    add("n16_random", rng.random((16, 16, 16)) < 0.3, pairs=SOME_PAIRS)
    add("n16_nested", walls(16, 0, 15) | walls(16, 4, 11) | walls(16, 6, 9), pairs=SOME_PAIRS)
    add("n16_checker", ijk.sum(0) % 2 == 0, pairs=SOME_PAIRS)
    vals = np.array([0.0] + steps(0.1) + steps(0.3), F32)
    add("n16_thres", vals[rng.choice(7, size=(16, 16, 16), p=[0.3] + [0.7 / 6] * 6)], thres=(0.1, 0.3), pairs=SOME_PAIRS)
    c = np.where(rng.random((16, 16, 16)) < 0.5, 0, rng.integers(0, 4, (16, 16, 16)))
    add("n16_held_ppc2", np.array([0.0, 2.0, 6.0], F32)[rng.choice(3, size=(16, 16, 16))], thres=(5.0, 1.0), ppc=2, count=c,
        pairs=SOME_PAIRS)
    return out


def diag_cov(s2):
    """(N, 6) upper triangles of diag(s2) (N, 3)."""
    c = np.zeros((len(s2), 6), F32)
    c[:, 0], c[:, 3], c[:, 5] = s2[:, 0], s2[:, 1], s2[:, 2]
    return c


def radius_ok(cov, dx):
    """No window radius sqrt(max sigma) / dx within 1e-4 of an integer (rotated covariances only)."""
    m = cov[:, [0, 1, 2, 1, 3, 4, 2, 4, 5]].reshape(-1, 3, 3).astype(np.float64)
    q = np.sqrt(np.maximum(np.linalg.eigvalsh(m), 1e-8).max(axis=1)) / dx
    return not np.any(np.abs(q - np.round(q)) <= 1e-4)


def screened_covs(seed, n, lo, hi, dx):
    for s in range(seed, seed + 100):
        c = covs(np.random.default_rng(s), n, lo, hi)
        if radius_ok(c, dx):
            return c
    raise RuntimeError("no seed passes the radius margin")


def splat_cases():
    """[(name, pos (N, 3), opacity (N,), cov (N, 6), grid_n, grid_dx)] of part (b); 8 cells of 0.125 unless named otherwise."""
    rng = np.random.default_rng(5678)
    n, dx = 8, 0.125
    out = []

    def add(name, pos, cov, grid_n=n, grid_dx=dx):
        pos = np.asarray(pos, F32).reshape(-1, 3)
        out.append((name, pos, rng.uniform(0.2, 1.0, len(pos)).astype(F32), np.asarray(cov, F32).reshape(-1, 6), grid_n, grid_dx))

    # positions on cell faces and nodes, one float32 step either side, and -0.0
    nodes = F32(np.arange(n + 1) * dx)
    vals = np.concatenate([nodes, np.nextafter(nodes, F32(-1)), np.nextafter(nodes, F32(2)), [F32(-0.0)]])
    pos = vals[rng.integers(0, len(vals), (300, 3))]
    pos[:40, 0] = F32(-0.0)
    add("faces", pos, diag_cov(rng.uniform(0.03, 0.2, (300, 3)) ** 2))
    # windows of radius 2-3 clipped at each face, edge and corner of the grid
    dirs = np.array([d for d in np.ndindex(3, 3, 3) if d != (1, 1, 1)]) - 1
    add("clipped", 0.5 + 0.44 * dirs + rng.uniform(-0.03, 0.03, dirs.shape), screened_covs(11, len(dirs), 0.15, 0.3, dx))
    # sqrt(sigma) / dx exactly 1..4 (exact in float32 for a diagonal covariance), and sigma one float32 step either side
    s2 = F32((np.arange(1, 5) * dx) ** 2)
    s2 = np.concatenate([np.nextafter(s2, F32(0)), s2, np.nextafter(s2, F32(1))])
    iso = np.repeat(s2[:, None], 3, axis=1)
    aniso = np.stack([F32(1e-4) * np.ones_like(s2), s2, F32(2e-3) * np.ones_like(s2)], axis=1)   # the largest on one axis
    add("int_radius", rng.uniform(0.05, 0.95, (2 * len(s2), 3)), diag_cov(np.concatenate([iso, aniso])))
    # degenerate covariances: zero, negative definite, isotropic, two equal eigenvalues, rank-1 needles, condition ~1e6
    k = 8
    on_node = nodes[rng.integers(0, n + 1, (k, 3))]
    R = rand_rot(np.random.default_rng(21), k)
    v = R[:, :, 0]
    s = rng.uniform(0.1, 0.25, k)
    two = upper(R @ (np.stack([s, s, 0.3 * s], 1)[:, :, None] ** 2 * np.eye(3)) @ R.transpose(0, 2, 1))
    cond = upper(R @ (np.stack([s, 1e-3 * s, 1e-6 * s], 1)[:, :, None] * np.eye(3)) @ R.transpose(0, 2, 1))
    needle = upper(s[:, None, None] ** 2 * v[:, :, None] * v[:, None, :])
    degen = np.concatenate([np.zeros((k, 6), F32), diag_cov(-rng.uniform(1e-4, 1e-2, (k, 3))),
                            diag_cov(np.repeat(s[:, None] ** 2, 3, 1)), two, cond, needle])
    assert radius_ok(np.concatenate([two, cond, needle]), dx)
    pos = np.concatenate([on_node, rng.uniform(0.1, 0.9, (k, 3))] * 3)
    add("degenerate", pos, degen)
    # 5000 Gaussians in one cell, window radius 1
    add("crowd", (np.array([3, 4, 5]) + rng.uniform(0, 1, (5000, 3))) * dx, covs(rng, 5000, 0.02, 0.08), grid_dx=dx)
    # Gaussians 1, 3 and grid_n + 2 cells beyond each face (other coordinates inside); windows of radius m - 1 (one cell
    # short), m (just reaching the border cell) and m + grid_n + 2 (wider than the grid), from sigma = ((r - 0.5) dx)^2
    pos, s2 = [], []
    for axis in range(3):
        for side in (0, 1):
            for m in (1, 3, n + 2):
                for r in (m - 1, m, m + n + 2):
                    if r < 1:
                        continue
                    p = rng.uniform(0.1, 0.9, 3)
                    p[axis] = ((-m if side == 0 else n - 1 + m) + 0.5) * dx
                    pos.append(p)
                    s2.append(((r - 0.5) * dx) ** 2)
    # corners: outside in two and in three coordinates, wide windows
    for c in ((-3, -3, 4), (n + 2, -1, n + 1), (-n - 2, n + 2, -3), (n + 3, n + 3, n + 3)):
        pos.append((np.array(c) + 0.5) * dx)
        s2.append(((n + 6) * dx) ** 2)
    pos, s2 = np.array(pos), np.array(s2)
    cov = diag_cov(np.repeat(s2[:, None], 3, 1))
    # far outside: an empty window
    far = np.array([[1e6, 0.5, 0.5], [0.5, -1e6, 0.5], [0.5, 0.5, 1e30], [-1e30, -1e30, -1e30]])
    add("offgrid", np.concatenate([pos, far]), np.concatenate([cov, diag_cov(np.full((4, 3), 0.01))]))
    # one isotropic Gaussian (sigma = 2) half a cell beyond the -x face: every x-slab of the grid is in its window
    add("offgrid_one", [[-0.5, 0.5, 0.5]], diag_cov(np.full((1, 3), 2.0)))
    return out


def _field(dtype, shape, value, n=None, lenient=False):
    f = fti.Field(dtype, shape, n, lenient=lenient)
    f.a[...] = value
    return f


def run_grid_case(spec):
    name, count, dens, dthr, sthr, ppc, pairs = spec
    ns, _ = load_reference(0)
    shape = dens.shape
    gd = _field(float, shape, dens)
    parts = fti.Field(float, (dens.size * ppc + 1,), 3)
    g = _field(int, shape, count)
    n_dense = ns["fill_dense_grids"](g, gd, 0.1, dthr, parts, 0, ppc)
    c1 = g.to_numpy()
    c2, totals = [], []
    for e, r in pairs:
        g = _field(int, shape, c1)
        totals.append(ns["internal_filling"](g, gd, 0.1, parts, n_dense, ppc, exclude_dir=int(e), ray_cast_dir=int(r), threshold=sthr))
        c2.append(g.to_numpy())
    c2 = np.stack(c2)
    assert c1.max() <= 255 and c2.max() <= 255
    print(f"(a) {name}: grid {shape[0]}, {len(pairs)} pairs, dense {n_dense}, interior {min(totals) - n_dense}..{max(totals) - n_dense}",
          flush=True)
    k = f"a/{name}/"
    return {k + "count": count, k + "density": dens, k + "thres": np.array([dthr, sthr]), k + "ppc": np.int32(ppc), k + "pairs": pairs,
            k + "count_dense": c1.astype(np.uint8), k + "count_internal": c2.astype(np.uint8), k + "n_dense": np.int32(n_dense),
            k + "n_total": np.array(totals, np.int32)}


def run_splat_case(spec):
    name, pos, opacity, cov, n, dx = spec
    ns, _ = load_reference(0)
    c0 = np.floor(pos / F32(dx))
    off = bool(np.any((c0 < 0) | (c0 >= n)))                    # lenient count field only where a Gaussian lies outside
    N = len(pos)
    grid = fti.Field(int, (n, n, n), lenient=off)
    dens = fti.Field(float, (n, n, n))
    ns["densify_grids"](_field(float, (N,), pos, 3), _field(float, (N,), opacity), _field(float, (N,), cov, 6), grid, dens, dx)
    print(f"(b) {name}: {N} Gaussians, grid {n}, {'lenient' if off else 'strict'} count, count {grid.a.sum()}, "
          f"density max {dens.a.max():.4g}", flush=True)
    k = f"b/{name}/"
    return {k + "pos": pos, k + "opacity": opacity, k + "cov": cov, k + "grid_n": np.int32(n), k + "grid_dx": np.float64(dx),
            k + "count": grid.to_numpy(), k + "density": dens.to_numpy()}


def _run(job):
    part, spec = job
    return run_grid_case(spec) if part == "a" else run_splat_case(spec)


def main():
    from multiprocessing import Pool
    grids, splats = grid_cases(), splat_cases()
    jobs = [("a", s) for s in grids] + [("b", s) for s in splats]
    # slowest first: the 12- and 16-cell grids with every pair, and the 5000-Gaussian cell
    cost = lambda j: (j[1][2].size * len(j[1][6])) if j[0] == "a" else 27 * 8 * len(j[1][1])   # noqa: E731
    order = sorted(range(len(jobs)), key=lambda i: -cost(jobs[i]))
    blob = {"a_cases": np.array([s[0] for s in grids]), "b_cases": np.array([s[0] for s in splats])}
    with Pool(os.cpu_count()) as pool:
        parts = pool.map(_run, [jobs[i] for i in order], chunksize=1)
    for i in np.argsort(order):
        blob.update(parts[i])
    path = os.path.join(HERE, "filling_edges_golden.npz")
    save_npz(path, blob)
    print("wrote", path, len(blob), "arrays,", os.path.getsize(path) // 1024, "KiB")


def save_npz(path, blob):
    """np.savez_compressed with a fixed time stamp on every member, so that a rerun reproduces the file byte for byte."""
    import io
    import zipfile
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as z:
        for k, v in blob.items():
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(v), allow_pickle=False)
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, buf.getvalue())


if __name__ == "__main__":
    main()
