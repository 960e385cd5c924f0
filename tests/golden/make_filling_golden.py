"""Generates tests/golden/filling_golden.npz by EXECUTING THE REFERENCE'S OWN particle-filling kernels
(PG/particle_filling/filling.py: densify_grids, fill_dense_grids, collision_search, collision_times, internal_filling,
fill_particles) on the float32 / int32 `ti` stand-in of _fake_taichi.py. PIXIE_REFERENCE names a checkout of the reference:

    python tests/golden/make_filling_golden.py

The function sources are pulled out of filling.py with `ast` (the module imports taichi and mcubes), their
`ti.atomic_add` calls rewritten for serial execution, and exec'd with the real torch (Tensor.cuda() is a no-op here).
Each case records its inputs, the count / density grids after each kernel, both fill counts and the output.

A seed is rejected when any cell density lies within 1e-4 (relative) of a threshold or any sqrt(max sigma) / dx within 1e-4
of an integer, so that summation order and eigensolver rounding cannot flip a cell or a window.
"""
import ast
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
REF = os.environ["PIXIE_REFERENCE"]
FILLING = REF + "/third_party/PhysGaussian/particle_filling/filling.py"

import _fake_taichi as fti  # noqa: E402

torch.Tensor.cuda = lambda self, *a, **kw: self

KERNELS = ["compute_density", "densify_grids", "fill_dense_grids", "collision_search", "collision_times", "internal_filling",
           "fill_particles"]


def load_reference(seed):
    """The reference's filling functions, exec'd on a fresh `ti` stand-in; kernel calls record grid snapshots."""
    tree = fti.rewrite_atomics(ast.parse(open(FILLING).read()))
    ns = {"ti": fti.make_ti(seed), "torch": torch, "np": np, "mcubes": None}
    seen = set()
    for node in tree.body:
        if isinstance(node, ast.FunctionDef) and node.name in KERNELS:
            exec(compile(ast.Module(body=[node], type_ignores=[]), FILLING, "exec"), ns)
            seen.add(node.name)
    assert seen == set(KERNELS), set(KERNELS) - seen
    snaps = {}

    def recorded(name, fn):
        def run(*a, **kw):
            out = fn(*a, **kw)
            grid, density = (a[3], a[4]) if name == "densify_grids" else (a[0], a[1])
            snaps[name] = (grid.to_numpy(), density.to_numpy())
            return out
        return run
    for k in ("densify_grids", "fill_dense_grids", "internal_filling"):
        ns[k] = recorded(k, ns[k])
    return ns, snaps


def rand_rot(rng, n):
    q = rng.standard_normal((n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    w, x, y, z = q.T
    return np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
                     2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
                     2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], axis=1).reshape(n, 3, 3)


def covs(rng, n, lo, hi):
    """Randomly rotated covariances with standard deviations in [lo, hi)."""
    s = rng.uniform(lo, hi, size=(n, 3))
    R = rand_rot(rng, n)
    return upper(R @ (s[:, :, None] ** 2 * np.eye(3)) @ R.transpose(0, 2, 1))


def upper(m):
    return np.stack([m[:, 0, 0], m[:, 0, 1], m[:, 0, 2], m[:, 1, 1], m[:, 1, 2], m[:, 2, 2]], axis=1).astype(np.float32)


def sphere(rng, n, c, r):
    v = rng.standard_normal((n, 3))
    return c + r * v / np.linalg.norm(v, axis=1, keepdims=True)


def cylinder_cup(rng, n_wall, n_cap, c, r, z0, z1, cap_z):
    t = rng.uniform(0, 2 * np.pi, n_wall)
    wall = np.stack([c[0] + r * np.cos(t), c[1] + r * np.sin(t), rng.uniform(z0, z1, n_wall)], axis=1)
    rr = r * np.sqrt(rng.uniform(0, 1, n_cap))
    t = rng.uniform(0, 2 * np.pi, n_cap)
    cap = np.stack([c[0] + rr * np.cos(t), c[1] + rr * np.sin(t), np.full(n_cap, cap_z)], axis=1)
    return np.concatenate([wall, cap])


C1 = np.array([1.0, 1.0, 1.0])


def case_inputs(name, rng):
    """(pos, opacity (N, 1), cov (N, 6), kwargs of fill_particles) of one case; positions in the simulation frame [0, 2]^3."""
    kw = dict(grid_n=24, max_samples=40000, grid_dx=2.0 / 24, density_thres=1.0, search_thres=0.25, max_particles_per_cell=1,
              search_exclude_dir=5, ray_cast_dir=4, boundary=None)
    if name == "shell":                                       # closed sphere shell, no boundary
        pos = sphere(rng, 2500, C1, 0.6)
        cov = covs(rng, len(pos), 0.015, 0.04)
    elif name == "cups":                                      # cup A open toward -z (excluded: filled), cup B open toward +z (not)
        a = cylinder_cup(rng, 1400, 500, (0.6, 1.0), 0.3, 0.55, 1.45, 1.45)
        b = cylinder_cup(rng, 1400, 500, (1.4, 1.0), 0.3, 0.55, 1.45, 0.55)
        pos = np.concatenate([a, b])
        cov = covs(rng, len(pos), 0.015, 0.035)
    elif name == "nested":                                    # the cavity of the inner shell has even parity: not filled
        pos = np.concatenate([sphere(rng, 3000, C1, 0.75), sphere(rng, 900, C1, 0.35)])
        cov = covs(rng, len(pos), 0.015, 0.035)
    elif name == "flat":                                      # axis-aligned discs whose third eigenvalue hits the 1e-8 clamp
        g = np.arange(-0.55, 0.56, 0.05)
        u, v = [a.ravel() for a in np.meshgrid(g, g)]
        faces = []
        for ax in range(3):
            for side in (-1, 1):
                p = np.zeros((len(u), 3))
                others = [d for d in range(3) if d != ax]
                p[:, others[0]], p[:, others[1]] = u, v
                p[:, ax] = side * 0.5 + 2e-5                  # just off a node plane: finite weights at dz ~ 1e-5
                faces.append((p + C1, ax))
        pos = np.concatenate([f for f, _ in faces])
        flat = rng.choice([0.0, -1e-6, -1e-9, 1e-12], size=len(pos))
        cov = np.zeros((len(pos), 6), np.float32)
        s = rng.uniform(0.02, 0.035, size=(len(pos), 2)) ** 2
        o = 0
        for f, ax in faces:
            sl = slice(o, o + len(f))
            d = np.zeros((len(f), 3))
            others = [q for q in range(3) if q != ax]
            d[:, others[0]], d[:, others[1]], d[:, ax] = s[sl, 0], s[sl, 1], flat[sl]
            cov[sl, 0], cov[sl, 3], cov[sl, 5] = d[:, 0], d[:, 1], d[:, 2]
            o += len(f)
    elif name == "clipped":                                   # r >= 3 windows clipped at the grid border, plus a shell
        big = np.array([[0.05, 0.1, 1.93], [1.95, 1.9, 0.04], [0.1, 1.92, 1.0], [1.0, 0.06, 0.08]])
        pos = np.concatenate([big, sphere(rng, 1500, C1, 0.5)])
        cov = np.concatenate([covs(rng, 4, 0.27, 0.33), covs(rng, 1500, 0.02, 0.04)])
        kw.update(density_thres=1.2, search_thres=0.3)
    elif name == "ppc2":                                      # sparse shell: cells holding one Gaussian get one more
        pos = sphere(rng, 900, C1, 0.6)
        cov = covs(rng, len(pos), 0.03, 0.05)
        kw.update(max_particles_per_cell=2, density_thres=0.6, search_thres=0.4)
    elif name == "boundary":                                  # non-cubic boundary, Gaussians outside it, other directions
        pos = np.concatenate([sphere(rng, 2500, np.array([0.9, 0.95, 1.05]), 0.45), rng.uniform(0.0, 2.0, size=(300, 3))])
        cov = covs(rng, len(pos), 0.01, 0.025)
        kw.update(grid_n=20, boundary=[0.3, 1.5, 0.4, 1.45, 0.45, 1.75], search_exclude_dir=0, ray_cast_dir=1,
                  density_thres=0.5, search_thres=0.15, grid_dx=0.123)
    else:
        raise KeyError(name)
    opacity = rng.uniform(0.5, 1.0, size=(len(pos), 1)).astype(np.float32)
    return pos.astype(np.float32), opacity, np.asarray(cov, np.float32), kw


def margins_ok(pos, cov, kw, density):
    """No density within 1e-4 (relative) of a threshold, no sqrt(max sigma) / dx within 1e-4 of an integer."""
    for thr in (kw["density_thres"], kw["search_thres"]):
        if np.any(np.abs(density.astype(np.float64) - thr) <= 1e-4 * thr):
            return False
    b = kw["boundary"]
    dx = kw["grid_dx"]
    if b is not None:
        keep = np.ones(len(pos), bool)
        for i in range(3):
            keep &= (pos[:, i] > np.float32(b[2 * i])) & (pos[:, i] < np.float32(b[2 * i + 1]))
        cov = cov[keep]
        dx = max(b[1] - b[0], b[3] - b[2], b[5] - b[4]) / kw["grid_n"]
    m = cov[:, [0, 1, 2, 1, 3, 4, 2, 4, 5]].reshape(-1, 3, 3).astype(np.float64)
    w = np.maximum(np.linalg.eigvalsh(m), 1e-8)
    q = np.sqrt(w.max(axis=1)) / dx
    return not np.any(np.abs(q - np.round(q)) <= 1e-4)


CASES = ["shell", "cups", "nested", "flat", "clipped", "ppc2", "boundary"]


def screened(name, seed):
    """The case's inputs if the numpy restatement's densities clear the margins (the reference's serial run is slow)."""
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
    from oracle import particle_filling_ref as R
    pos, opacity, cov, kw = case_inputs(name, np.random.default_rng(seed))
    r = R.fill_particles(pos, opacity, cov, **kw)
    return (pos, opacity, cov, kw) if margins_ok(pos, cov, kw, r["density"]) else None


def run_case(ci):
    name = CASES[ci]
    for seed in range(100 * ci, 100 * ci + 100):
        inputs = screened(name, seed)
        if inputs is None:
            continue
        pos, opacity, cov, kw = inputs
        ns, snaps = load_reference(seed)
        out = ns["fill_particles"](torch.from_numpy(pos), torch.from_numpy(opacity), torch.from_numpy(cov), **kw)
        if margins_ok(pos, cov, kw, snaps["densify_grids"][1]):
            break
    else:
        raise RuntimeError(f"{name}: no seed passes the margins")
    g0, d0 = snaps["densify_grids"]
    g1, _ = snaps["fill_dense_grids"]
    g2, _ = snaps["internal_filling"]
    n_dense = int((g1 - g0).sum())
    n_total = int(out.shape[0]) - len(pos)
    b = kw["boundary"]
    print(f"{name}: seed {seed}, {len(pos)} Gaussians, grid {kw['grid_n']}, dense {n_dense}, interior {n_total - n_dense}, "
          f"density max {d0.max():.3g}", flush=True)
    return {f"{name}/pos": pos, f"{name}/opacity": opacity, f"{name}/cov": cov, f"{name}/seed": np.int64(seed),
            f"{name}/grid_n": np.int32(kw["grid_n"]), f"{name}/max_samples": np.int32(kw["max_samples"]),
            f"{name}/grid_dx": np.float64(kw["grid_dx"]), f"{name}/density_thres": np.float64(kw["density_thres"]),
            f"{name}/search_thres": np.float64(kw["search_thres"]), f"{name}/max_particles_per_cell": np.int32(kw["max_particles_per_cell"]),
            f"{name}/search_exclude_dir": np.int32(kw["search_exclude_dir"]), f"{name}/ray_cast_dir": np.int32(kw["ray_cast_dir"]),
            f"{name}/boundary": np.array(b if b is not None else [], np.float64),
            f"{name}/count_densify": g0, f"{name}/density": d0, f"{name}/count_dense": g1, f"{name}/count_internal": g2,
            f"{name}/n_dense": np.int32(n_dense), f"{name}/n_total": np.int32(n_total), f"{name}/out": out.numpy().copy()}


def main():
    from multiprocessing import Pool
    blob = {"cases": np.array(CASES)}
    with Pool(len(CASES)) as pool:                            # the serial interpreter takes minutes per case
        for part in pool.map(run_case, range(len(CASES))):
            blob.update(part)
    path = os.path.join(HERE, "filling_golden.npz")
    np.savez_compressed(path, **blob)
    print("wrote", path, len(blob), "arrays,", os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
