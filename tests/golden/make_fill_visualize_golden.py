"""Generates tests/golden/fill_visualize_golden.npz by EXECUTING THE REFERENCE'S OWN `get_attr_from_closest` and
`init_filled_particles` (PG/particle_filling/filling.py:383-446, the `particle_filling.visualize` step of gs_simulation.py)
on the float32 `ti` stand-in of _fake_taichi.py. PIXIE_REFERENCE names a checkout of the reference:

    python tests/golden/make_fill_visualize_golden.py

The two functions are pulled out of filling.py with `ast` and exec'd with the real torch (Tensor.cuda() is a no-op here).
The stand-in's vector value gets the one method these functions add to what the filling kernels use, `norm()`: the float32
sqrt (correctly rounded) of the left-to-right float32 dot product with itself, set here so that the stand-in shared with
make_filling_golden.py / make_filling_edges_golden.py stays as it is.

Each case records its inputs (Gaussian positions, SH (N, K, 3), opacity, cov; new particle positions), the nearest-Gaussian
index of every new particle, and the rows the reference appends for the new particles (`out_*`, its outputs past the
first N rows; the first N are checked here to be the inputs, bit for bit). The kernel does not return the index; it is
read back from the copied SH row, which is unique to one Gaussian in every case (checked), and the copied opacity and cov
rows are checked against it too. The attributes are exact functions of the Gaussian's index (unique SH rows, values
that compress), since the search never reads them; only their bits are copied.

Cases (each at most about 2e6 query-Gaussian pairs, so the serial stand-in finishes in well under a minute):
  shell, cups   the Gaussians and (every other / all) filled particles of filling_golden.npz's scenes, SH degree 1 / 0;
                their positions are read from filling_golden.npz (`filling_positions`) and not stored again
  dup           Gaussians stacked 2-6 deep on 40 positions with different attributes: the lowest index wins (index tie)
  mirror        pairs mirrored about exactly representable planes, queries on the bisector: equal d (distance tie)
  sqrt          pairs whose float32 squared distances differ but whose rounded square roots are equal (distance tie)
  exact         queries exactly on Gaussians (d = 0) among random ones
  far           queries 1e2 to 1e6 box sizes outside the Gaussians' box
  one           N = 1
Every SH width (K = 1, 4, 9, 16) occurs. The file is written deterministically: a rerun reproduces it byte for byte.
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
from make_filling_edges_golden import save_npz  # noqa: E402

torch.Tensor.cuda = lambda self, *a, **kw: self
# ti.Vector.norm(): float32 sqrt of the float32 dot product, summed left to right (Taichi's default precision)
fti.Vector.norm = lambda self: F32(np.sqrt(F32(self.dot(self))))

F32 = np.float32
KERNELS = ["get_attr_from_closest", "init_filled_particles"]
CASES = ["shell", "cups", "dup", "mirror", "sqrt", "exact", "far", "one"]
FROM_FILLING = ("shell", "cups")


def filling_positions(filling_golden, name):
    """(Gaussians, queries) of the shell / cups cases: a filling_golden.npz scene's Gaussians and its filled particles
    (every other one for the shell, to keep the serial run short)."""
    pos = filling_golden[f"{name}/pos"]
    new = filling_golden[f"{name}/out"][len(pos):]
    return pos, (new[::2] if name == "shell" else new)


def load_reference():
    tree = fti.rewrite_atomics(ast.parse(open(FILLING).read()))
    ns = {"ti": fti.make_ti(0), "torch": torch, "np": np, "mcubes": None}
    seen = set()
    for node in tree.body:
        if isinstance(node, ast.FunctionDef) and node.name in KERNELS:
            exec(compile(ast.Module(body=[node], type_ignores=[]), FILLING, "exec"), ns)
            seen.add(node.name)
    assert seen == set(KERNELS), set(KERNELS) - seen
    return ns


def attrs(rng, n, k):
    """SH (n, k, 3), opacity (n, 1) and cov (n, 6), float32 and exact functions of the Gaussian index i < 2^12: SH
    i 2^-12 + (3 j + c) / 16 - 1 (rows unique), opacity (i + 1) 2^-12, cov (i + 1) 2^-20 (1, 0, 0, 2, 0, 3).
    `rng` is unused; it keeps the call sites' draws in order."""
    assert n < 4096
    i = np.arange(n, dtype=np.float64)
    shs = (i[:, None, None] * 2.0 ** -12 + np.arange(3 * k).reshape(1, k, 3) / 16.0 - 1.0).astype(F32)
    opacity = ((i[:, None] + 1) * 2.0 ** -12).astype(F32)
    cov = ((i[:, None] + 1) * np.array([1, 0, 0, 2, 0, 3]) * 2.0 ** -20).astype(F32)
    return shs, opacity, cov


def case_inputs(name):
    """(pos (N, 3), shs (N, K, 3), opacity (N, 1), cov (N, 6), new_pos (M, 3)), float32."""
    rng = np.random.default_rng(CASES.index(name) + 17)
    if name in FROM_FILLING:
        pos, new = filling_positions(np.load(os.path.join(HERE, "filling_golden.npz")), name)
        return (pos,) + attrs(rng, len(pos), 4 if name == "shell" else 1) + (new,)
    if name == "dup":
        sites = rng.uniform(0.2, 1.8, (40, 3)).astype(F32)
        pos = np.repeat(sites, rng.integers(2, 7, 40), axis=0)
        pos = pos[rng.permutation(len(pos))]
        new = np.concatenate([rng.uniform(0.0, 2.0, (400, 3)), sites[:20]]).astype(F32)
        return (pos,) + attrs(rng, len(pos), 4) + (new,)
    if name == "mirror":
        # pair (c - h e_a, c + h e_a), c and h on a 2^-6 grid: for a query on the plane through c normal to e_a, both
        # |dx| are h exactly, so both d are equal. Which of the two comes first varies.
        c = rng.integers(32, 96, (150, 3)) / 64.0
        h = rng.integers(1, 24, 150) / 64.0
        a = rng.integers(0, 3, 150)
        e = np.eye(3)[a] * h[:, None]
        lo_first = rng.random(150) < 0.5
        first = np.where(lo_first[:, None], c - e, c + e)
        second = np.where(lo_first[:, None], c + e, c - e)
        pos = np.stack([first, second], axis=1).reshape(-1, 3).astype(F32)
        off = rng.integers(-40, 40, (150, 3)) / 256.0
        off[np.arange(150), a] = 0.0
        new = (c + off).astype(F32)
        return (pos,) + attrs(rng, len(pos), 1) + (new,)
    if name == "sqrt":
        # b = a + t e_y with fl(t^2) ~ 2^-23 |dx|^2: s_b = s_a (1 + 2^-23) but sqrt rounds both to the same d
        q = rng.uniform(0.5, 1.5, (120, 3)).astype(F32)
        scale = (2.0 ** rng.integers(-6, 1, 120)).astype(F32)
        a = q + np.stack([scale, np.zeros(120, F32), np.zeros(120, F32)], axis=1)
        t = (scale * F32(2.0 ** -11.5)).astype(F32)
        b = a + np.stack([np.zeros(120, F32), t, np.zeros(120, F32)], axis=1).astype(F32)
        lo_b = rng.random(120) < 0.5
        pos = np.stack([np.where(lo_b[:, None], b, a), np.where(lo_b[:, None], a, b)], axis=1).reshape(-1, 3).astype(F32)
        return (pos,) + attrs(rng, len(pos), 16) + (q,)
    if name == "exact":
        pos = rng.uniform(0.3, 1.7, (600, 3)).astype(F32)
        new = np.concatenate([pos[rng.choice(600, 300, replace=False)], rng.uniform(0.3, 1.7, (300, 3))]).astype(F32)
        return (pos,) + attrs(rng, len(pos), 9) + (new,)
    if name == "far":
        pos = rng.uniform(0.5, 1.5, (300, 3)).astype(F32)
        v = rng.standard_normal((300, 3))
        v /= np.linalg.norm(v, axis=1, keepdims=True)
        new = (1.0 + v * 10.0 ** rng.uniform(2, 6, (300, 1))).astype(F32)
        return (pos,) + attrs(rng, len(pos), 4) + (new,)
    if name == "one":
        pos = np.array([[1.25, 0.75, 1.0]], F32)
        new = np.concatenate([rng.uniform(0.0, 2.0, (200, 3)), pos]).astype(F32)
        return (pos,) + attrs(rng, 1, 1) + (new,)
    raise KeyError(name)


def run_case(name):
    pos, shs, opacity, cov, new = case_inputs(name)
    k = shs.shape[1]
    rows = shs.reshape(len(pos), -1)
    assert len(np.unique(rows, axis=0)) == len(pos), "SH rows must identify their Gaussian"
    ns = load_reference()
    o_shs, o_op, o_cov = ns["init_filled_particles"](torch.from_numpy(pos), torch.from_numpy(shs.copy()), torch.from_numpy(cov),
                                                   torch.from_numpy(opacity), torch.from_numpy(new))
    o_shs, o_op, o_cov = o_shs.numpy().copy(), o_op.numpy().copy(), o_cov.numpy().copy()
    n = len(pos)
    assert o_shs.shape == (n + len(new), k, 3) and o_op.shape == (n + len(new), 1) and o_cov.shape == (n + len(new), 6)
    for o, x in ((o_shs, shs), (o_op, opacity), (o_cov, cov)):
        assert np.array_equal(o[:n].view(np.uint32), x.view(np.uint32))
    got = o_shs[n:].reshape(len(new), -1)
    match = np.all(got.view(np.uint32)[:, None, :] == rows.view(np.uint32)[None, :, :], axis=2)
    assert np.all(match.sum(1) == 1)
    index = np.argmax(match, axis=1).astype(np.int32)
    assert np.array_equal(o_op[n:].view(np.uint32), opacity[index].view(np.uint32))
    assert np.array_equal(o_cov[n:].view(np.uint32), cov[index].view(np.uint32))
    print(f"{name}: N {n}, M {len(new)}, K {k}", flush=True)
    stored = {} if name in FROM_FILLING else {f"{name}/pos": pos, f"{name}/new_pos": new}
    return {**stored, f"{name}/shs": shs, f"{name}/opacity": opacity, f"{name}/cov": cov,
            f"{name}/index": index, f"{name}/out_shs": o_shs[n:], f"{name}/out_opacity": o_op[n:], f"{name}/out_cov": o_cov[n:]}


def main():
    from multiprocessing import Pool
    blob = {"cases": np.array(CASES)}
    with Pool(len(CASES)) as pool:
        for part in pool.map(run_case, CASES):
            blob.update(part)
    path = os.path.join(HERE, "fill_visualize_golden.npz")
    save_npz(path, blob)
    print("wrote", path, len(blob), "arrays,", os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
