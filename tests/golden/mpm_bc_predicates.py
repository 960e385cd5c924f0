"""numpy restatement of the MPM boundary-condition decisions (GOLDEN-VECTOR TOOLING, shared by
make_mpm_bc_edges_golden.py and tests/test_mpm_bc_edges.py).

Every predicate is evaluated in two forms:
  * `fused=False`: the reference's float32 arithmetic, one rounding per operation (what the stand-in of
    _fake_warp.py computes, and what oracle/mpm_ref.c built with -ffp-contract=off computes);
  * `fused=True`: the same statements contracted the way nvcc contracts them by default, i.e. `a * b + c` as one
    fused multiply-add with a single rounding. Dot products become fma(z, nz, fma(y, ny, x * nx)).
The generator asserts that every case meant to separate the two forms does, and the tests check that the fused
form disagrees with the fixture on each of those cases, so a device that contracts these statements fails them.

Grid decisions are reported as classes per node: a bitmask of zeroed components (PASS = 0, ZERO = 7), CUBOID
(set to the cuboid's velocity) or CUT (the cut collider's 0.3 scaling).
"""
from __future__ import annotations

from fractions import Fraction

import numpy as np

f32 = np.float32
PASS, ZERO, CUBOID, CUT, UNKNOWN = 0, 7, 8, 9, -1
BC_SURFACE, BC_CUBOID, BC_BBOX = 0, 1, 2          # oracle/mpm_ref.py numbering


def round_f32(q: Fraction) -> np.float32:
    """Correctly rounded float32 of an exact rational (ties to even)."""
    r = f32(float(q))
    best = None
    for c in (np.nextafter(r, f32(-np.inf)), r, np.nextafter(r, f32(np.inf))):
        if not np.isfinite(c):
            continue
        d = abs(Fraction(float(c)) - q)
        key = (d, int(np.array(c, f32).view(np.uint32)) & 1)
        if best is None or key < best[0]:
            best = (key, c)
    return f32(best[1])


def fma32(a, b, c) -> np.float32:
    """fmaf(a, b, c): the exact a * b + c rounded once to float32."""
    return round_f32(Fraction(float(f32(a))) * Fraction(float(f32(b))) + Fraction(float(f32(c))))


def mul(a, b):
    return f32(f32(a) * f32(b))


def offset(g, dx, p, fused):
    """float(g) * dx - p"""
    return fma32(f32(g), dx, -f32(p)) if fused else f32(mul(f32(g), dx) - f32(p))


def dot(a, b, fused):
    """wp.dot: ((a0 b0 + a1 b1) + a2 b2)"""
    if fused:
        return fma32(a[2], b[2], fma32(a[1], b[1], mul(a[0], b[0])))
    return f32(f32(mul(a[0], b[0]) + mul(a[1], b[1])) + mul(a[2], b[2]))


def reset_threshold(end_time, dt, fused):
    """end_time + 15.0 * dt"""
    return fma32(f32(15.0), dt, end_time) if fused else f32(f32(end_time) + mul(f32(15.0), dt))


def grid_bcs(nodes, u, bcs, n_grid, dx, time, dt, fused=False):
    """Velocities after every grid BC (registration order) for nodes [M, 3] that all start at velocity u.
    bcs: dicts with float32 point / normal / size / velocity / start_time / end_time and kind, surface_type, reset."""
    dx, time, dt = f32(dx), f32(time), f32(dt)
    out = np.empty((len(nodes), 3), f32)
    for i, (gx, gy, gz) in enumerate(np.asarray(nodes)):
        v = np.array(u, f32)
        for bc in bcs:
            active = time >= bc["start_time"] and time < bc["end_time"]
            kind = bc["kind"]
            if kind == BC_SURFACE:
                if active:
                    off = [offset(g, dx, p, fused) for g, p in zip((gx, gy, gz), bc["point"])]
                    if dot(off, bc["normal"], fused) < 0:
                        zz = mul(f32(gz), dx)
                        if bc["surface_type"] == 11 and not (zz < f32(0.4) or zz > f32(0.53)):
                            v = np.array([mul(v[0], 0.3), mul(0.0, 0.3), mul(v[2], 0.3)], f32)
                        else:
                            v = np.zeros(3, f32)
            elif kind == BC_CUBOID:
                if active:
                    off = [offset(g, dx, p, fused) for g, p in zip((gx, gy, gz), bc["point"])]
                    if all(abs(o) < s for o, s in zip(off, bc["size"])):
                        v = np.array(bc["velocity"], f32)
                elif bc["reset"] == 1 and time < reset_threshold(bc["end_time"], dt, fused):
                    v = np.zeros(3, f32)
            elif kind == BC_BBOX and active:
                for a, g in enumerate((gx, gy, gz)):
                    if (g < 3 and v[a] < 0) or (g >= n_grid - 3 and v[a] > 0):
                        v[a] = 0
        out[i] = v
    return out


def clock(dt, k):
    """The reference's host clock after k substeps: `self.time = self.time + dt` in Python floats (:637)."""
    t = 0.0
    for _ in range(k):
        t = t + dt
    return t


def box_nodes(lo, hi):
    """Node indices [M, 3] of the box [lo, hi), x slowest."""
    return np.stack(np.meshgrid(*[np.arange(a, b) for a, b in zip(lo, hi)], indexing="ij"), -1).reshape(-1, 3)


def restate_case(c, records, fused, window="f32"):
    """Classes [steps, nodes] of a fixture grid case: its substeps from the sentinel grid, the moving cuboid advanced
    between them like `modify` (Python floats, stored as float32). `modify`'s window compares the Python-float clock
    with the float32 start / end times: in float32 (window="f32", the stand-in under NumPy 2) or in double
    (window="f64", the device and the oracle); the two differ only for times that round onto a substep's clock."""
    n, lim, dt = c["n_grid"], c["grid_lim"], c["dt"]
    dx = f32(lim / n)
    recs = [dict(r) for r in records]
    nodes = box_nodes(c["lo"], c["hi"])
    t = clock(dt, c["k"])
    out = []
    for _ in range(c["steps"]):
        out.append(classify(grid_bcs(nodes, c["u"], recs, n, dx, t, dt, fused=fused), c["u"], velocity=c["vel"]))
        for r in recs:
            if window == "f32":
                on = f32(t) >= f32(r["start_time"]) and f32(t) < f32(r["end_time"])
            else:
                on = t >= float(f32(r["start_time"])) and t < float(f32(r["end_time"]))
            if r["kind"] == BC_CUBOID and on:
                r["point"] = [float(f32(p + dt * v)) for p, v in zip(r["point"], r["velocity"])]
        t = t + dt
    return np.stack(out)


def classify(v, u, velocity=None, ulps=0):
    """Class of each node velocity (see module doc). `ulps` > 0 accepts u and the cut value within that many float32
    steps (device grids hold m u / m, not u); zeros and the cuboid velocity are always exact."""
    v = np.asarray(v, f32).reshape(-1, 3)
    u = np.asarray(u, f32)
    cut = np.array([mul(u[0], 0.3), 0.0, mul(u[2], 0.3)], f32)

    def near(a, b):
        if ulps == 0:
            return a == b
        ia, ib = np.asarray(a, f32).view(np.int32).astype(np.int64), np.asarray(b, f32).view(np.int32).astype(np.int64)
        return (np.sign(a) == np.sign(b)) & (np.abs(ia - ib) <= ulps)

    out = np.full(len(v), UNKNOWN, np.int8)
    for i, w in enumerate(v):
        if velocity is not None and (w == np.asarray(velocity, f32)).all():
            out[i] = CUBOID
        elif w[1] == 0 and near(w[0], cut[0]) and near(w[2], cut[2]) and u[0] != 0:
            out[i] = CUT
        else:
            bits = 0
            for a in range(3):
                if w[a] == 0:
                    bits |= 1 << a
                elif not near(w[a], u[a]):
                    bits = UNKNOWN
                    break
            out[i] = bits
    return out


def select_box(x, point, size):
    """selection_add_impulse_on_particles / _translation: |x - p| < size on every axis (subtractions only)."""
    x = np.asarray(x, f32)
    off = np.abs((x - np.asarray(point, f32)).astype(f32))
    return (off < np.asarray(size, f32)).all(axis=1).astype(np.int32)


def additional_params_material(x, boxes, material0):
    """apply_additional_params, one launch per box in order: p - size < x < p + size; later boxes win."""
    x = np.asarray(x, f32)
    mat = np.full(len(x), material0, np.int32)
    for b in boxes:
        p, s = np.asarray(b["point"], f32), np.asarray(b["size"], f32)
        inside = ((x > (p - s).astype(f32)) & (x < (p + s).astype(f32))).all(axis=1)
        mat[inside] = b["material"]
    return mat


def select_cylinder(x, point, normal, half_height, radius, fused=False):
    """selection_enforce_particle_velocity_cylinder: |dot(o, n)| < hh and |o - dot(o, n) n| < r."""
    n = np.asarray(normal, f32)
    out = np.zeros(len(x), np.int32)
    for i, xi in enumerate(np.asarray(x, f32)):
        o = (xi - np.asarray(point, f32)).astype(f32)
        on = dot(o, n, fused)
        if fused:
            h = [fma32(-on, n[a], o[a]) for a in range(3)]
        else:
            h = [f32(o[a] - mul(on, n[a])) for a in range(3)]
        hd = f32(np.sqrt(dot(h, h, fused)))
        out[i] = int(abs(on) < f32(half_height) and hd < f32(radius))
    return out


def rotation_theta_positive(x, point, h2, fused=False):
    """The rotation modifier's half-plane test: theta keeps its sign where dot(x - point, h2) > 0 (:1160-1163)."""
    out = np.zeros(len(x), bool)
    for i, xi in enumerate(np.asarray(x, f32)):
        o = (xi - np.asarray(point, f32)).astype(f32)
        out[i] = dot(o, np.asarray(h2, f32), fused) > 0
    return out
