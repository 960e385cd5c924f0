"""Generates tests/golden/mpm_bc_edges_golden.npz by EXECUTING THE REFERENCE'S OWN BOUNDARY-CONDITION CODE
($PIXIE_REFERENCE/third_party/PhysGaussian/mpm_solver_warp/mpm_solver_warp.py and mpm_utils.py) on the float32
`warp` stand-in of tests/golden/_fake_warp.py:

    PIXIE_REFERENCE=/path/to/checkout python tests/golden/make_mpm_bc_edges_golden.py

The BCs are registered through the reference's own methods. Its collide closures and `modify` closures then run in
the order of `p2g2p` (:607-621) on a grid whose velocity is a sentinel `u` at every node, and its selection kernels
run on particles placed on the faces they test. What they decide is recorded per node and per particle. The cases sit
where a float32 comparison flips a node or a particle: planes and faces through node coordinates and one float32 step
either side, reset windows that end on a substep, points and particles found by search where a fused multiply-add
would decide differently (asserted here against mpm_bc_predicates.py), and a moving cuboid sweeping across nodes.
A rerun reproduces the file byte for byte. Nothing of the reference is copied: it is imported.
"""
import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
REF = os.path.join(os.environ["PIXIE_REFERENCE"], "third_party", "PhysGaussian", "mpm_solver_warp")

import _fake_warp as wp  # noqa: E402

wp.install()
for missing in ("h5py", "plyfile"):               # imported by engine_utils.py for file I/O only
    if missing not in sys.modules:
        m = types.ModuleType(missing)
        m.PlyData = m.PlyElement = m.File = None
        sys.modules[missing] = m
sys.path.insert(0, REF)
import mpm_solver_warp as REFMOD  # noqa: E402  (the reference)

import mpm_bc_predicates as P  # noqa: E402

f32 = np.float32
GRIDS = ((16, 2.0), (37, 2.0), (64, 2.0), (100, 2.0), (50, 1.0))
U_POS = (0.625, -0.375, 0.875)             # sentinel node velocity: exact, every component well away from 0
U_NEG = (-0.625, 0.375, -0.875)
CUBE_V = (0.25, 0.5, -0.75)                # cuboid velocity, distinct from u, -u and the cut value


def up(x, k=1):
    x = f32(x)
    for _ in range(abs(k)):
        x = np.nextafter(x, f32(np.inf) if k > 0 else f32(-np.inf))
    return f32(x)


def node(g, dx):
    return f32(f32(g) * f32(dx))


# ------------------------------------------------------------------------------------------ running the reference
def launch_nodes(kernel, nodes, inputs):
    """wp.launch restricted to the given thread ids (argument conversion as in _fake_warp.launch)."""
    args = []
    for t, v in zip(kernel.ann, inputs):
        if t is float and not isinstance(v, (wp._Vec, wp.mat33, wp.array)):
            v = f32(v)
        elif t is int and isinstance(v, (bool, int, np.integer)):
            v = int(v)
        args.append(v)
    for idx in nodes:
        wp._tid = tuple(int(i) for i in idx)
        kernel.fn(*args)
    wp._tid = None


def bc_record(kind, p):
    """The parameters as the reference stored them (float32)."""
    rec = dict(kind=kind, point=[0.0] * 3, normal=[0.0] * 3, size=[0.0] * 3, velocity=[0.0] * 3,
               start_time=float(f32(p.start_time)), end_time=float(f32(p.end_time)), surface_type=0, reset=0)
    if kind in (P.BC_SURFACE, P.BC_CUBOID):
        rec["point"] = [float(v) for v in p.point.a]
    if kind == P.BC_SURFACE:
        rec["normal"] = [float(v) for v in p.normal.a]
        rec["surface_type"] = int(p.surface_type)
    if kind == P.BC_CUBOID:
        rec["size"] = [float(f32(v)) for v in p.size]
        rec["velocity"] = [float(v) for v in p.velocity.a]
        rec["reset"] = int(p.reset)
    return rec


def run_grid_case(c):
    """Registers c["bcs"] on the reference solver and runs its grid BC closures for c["steps"] substeps starting at
    substep c["k"]; every substep starts from the sentinel grid. Returns classes [steps, nodes] and the BC records."""
    n, lim, dt = c["n_grid"], c["grid_lim"], c["dt"]
    s = REFMOD.MPM_Simulator_WARP(1, n_grid=n, grid_lim=lim, device="cpu")
    kinds = []
    for method, kw in c["bcs"]:
        getattr(s, method)(**kw)
        kinds.append({"add_surface_collider": P.BC_SURFACE, "set_velocity_on_cuboid": P.BC_CUBOID,
                      "add_bounding_box": P.BC_BBOX}[method])
    s.time = P.clock(dt, c["k"])
    nodes = P.box_nodes(c["lo"], c["hi"])
    records = [bc_record(k, p) for k, p in zip(kinds, s.collider_params)]
    cls = []
    for _ in range(c["steps"]):
        s.mpm_state.grid_v_out.data[...] = np.asarray(c["u"], f32)
        for k in range(len(s.grid_postprocess)):               # p2g2p's BC loop (:607-621)
            launch_nodes(s.grid_postprocess[k], nodes, [s.time, dt, s.mpm_state, s.mpm_model, s.collider_params[k]])
            if s.modify_bc[k] is not None:
                s.modify_bc[k](s.time, dt, s.collider_params[k])
        v = s.mpm_state.grid_v_out.data[nodes[:, 0], nodes[:, 1], nodes[:, 2]]
        cls.append(P.classify(v, c["u"], velocity=c["vel"]))
        s.time = s.time + dt                                   # :637
    return np.stack(cls), records


# ------------------------------------------------------------------------------------------ grid cases
def collider(point, normal, surface="sticky", **kw):
    return ("add_surface_collider", dict(point=[float(v) for v in point], normal=list(normal), surface=surface,
                                         friction=0.0, **kw))


def cuboid(point, size, **kw):
    return ("set_velocity_on_cuboid", dict(point=[float(v) for v in point], size=[float(v) for v in size],
                                           velocity=list(CUBE_V), **kw))


def ref_normal(normal):
    s = REFMOD.MPM_Simulator_WARP(1, n_grid=16, grid_lim=2.0, device="cpu")
    s.add_surface_collider([1.0, 1.0, 1.0], list(normal))
    return s.collider_params[0].normal.a.copy()


def grid_cases():
    cases = []

    def add(name, n, lim, bcs, lo, hi, u=U_POS, k=3, dt=1e-4, steps=1, disc=False):
        cases.append(dict(name=name, n_grid=n, grid_lim=lim, dt=dt, k=k, steps=steps, bcs=bcs, lo=list(lo), hi=list(hi),
                          u=list(u), vel=list(CUBE_V), disc=disc))

    # axis-aligned planes through a node plane (dot = +-0 is not < 0) and one float32 step either side, every
    # surface type, every grid; the cut type on y planes with z boxes over its 0.4 / 0.53 band
    for n, lim in GRIDS:
        dx = lim / n
        c = n // 2
        for surface in ("sticky", "slip", "separate", "cut"):
            for step in (-1, 0, 1):
                if surface == "cut":
                    pz = up(node(c, dx), step)
                    z0, z1 = int(0.38 / dx), int(np.ceil(0.55 / dx)) + 1
                    add(f"plane_{surface}_n{n}_{step:+d}", n, lim, [collider((1.0, pz, 1.0), (0.0, 1.0, 0.0), surface)],
                        (c - 1, c - 2, max(z0, 1)), (c + 1, c + 3, min(z1, n - 1)))
                else:
                    pz = up(node(c, dx), step)
                    add(f"plane_{surface}_n{n}_{step:+d}", n, lim, [collider((1.0, 1.0, pz), (0.0, 0.0, 1.0), surface)],
                        (c - 1, c - 1, c - 2), (c + 1, c + 1, c + 3))
            # a -x facing plane through a node plane
        add(f"plane_negx_n{n}", n, lim, [collider((node(c, dx), 1.0, 1.0), (-1.0, 0.0, 0.0))], (c - 2, c - 1, c - 1), (c + 3, c + 1, c + 1))

    # tilted normals: points searched so that the fused dot product decides a node differently, both directions
    for n, lim in ((100, 2.0), (37, 2.0), (50, 1.0)):
        dx = f32(lim / n)
        c = n // 2
        for normal in ((0.0, 0.3, 1.0), (-1.0, 0.0, 0.1), (0.3, -0.7, 0.2), (1.0, 1.0, 1.0)):
            nf = ref_normal(normal)
            found = {}
            for kx in range(-2, 3):
                for ky in range(-2, 3):
                    for kz in range(-2, 3):
                        for a in range(4):
                            g = (c + a, c - a, c + 2 * a)
                            p = [up(node(gi, dx), ki) for gi, ki in zip(g, (kx, ky, kz))]
                            off_u = [P.offset(gi, dx, pi, False) for gi, pi in zip(g, p)]
                            off_f = [P.offset(gi, dx, pi, True) for gi, pi in zip(g, p)]
                            du, df = P.dot(off_u, nf, False) < 0, P.dot(off_f, nf, True) < 0
                            if du != df and du not in found:
                                found[du] = (g, p)
                if len(found) == 2:
                    break
            assert found, ("no fused-sensitive point", n, normal)
            for du, (g, p) in sorted(found.items()):
                add(f"tilted_n{n}_{'_'.join(f'{v:g}' for v in normal)}_{'in' if du else 'out'}", n, lim,
                    [collider(p, normal)], [gi - 2 for gi in g], [gi + 3 for gi in g], disc=True)
    # nodes whose z coordinate is exactly float32 0.4 or 0.53, under a cut plane (the band edges)
    for n, lim in GRIDS:
        dx = lim / n
        for zb in (0.4, 0.53):
            gz = int(round(zb / dx))
            if node(gz, dx) == f32(zb) and 1 <= gz < n - 2:
                c = n // 2
                add(f"cut_band_n{n}_{zb:g}", n, lim, [collider((1.0, node(c, dx), 1.0), (0.0, 1.0, 0.0), "cut")],
                    (c - 1, c - 2, gz - 1), (c + 1, c + 2, gz + 2))

    # cuboids: faces on node coordinates (|off| == size is outside) and one step either side, per axis
    for n, lim in GRIDS:
        dx = lim / n
        c = n // 2
        p = [node(c, dx)] * 3
        for axis in range(3):
            for step in (-1, 0, 1):
                size = [f32(3.5 * dx)] * 3
                size[axis] = up(P.offset(c + 2, dx, p[axis], False), step)
                add(f"cuboid_face_n{n}_a{axis}_{step:+d}", n, lim, [cuboid(p, size)], (c - 3, c - 3, c - 3), (c + 4, c + 4, c + 4))
    # (point, size) pairs where the fused node offset lands on the other side of the face
    for n, lim in ((100, 2.0), (37, 2.0), (50, 1.0)):
        dx = f32(lim / n)
        c = n // 2
        for axis in range(3):
            done = set()
            for k in range(-6, 7):
                for gface in (c + 2, c - 2, c + 3):
                    pa = up(node(c, dx) + f32(0.3) * dx, k)
                    ou, of = P.offset(gface, dx, pa, False), P.offset(gface, dx, pa, True)
                    if abs(ou) == abs(of):
                        continue
                    inside_u = abs(ou) < abs(of)           # size = the larger magnitude: only the smaller one is inside
                    if inside_u in done:
                        continue
                    done.add(inside_u)
                    p = [node(c, dx) + f32(0.3) * dx] * 3
                    p[axis] = pa
                    size = [f32(4.5 * dx)] * 3
                    size[axis] = f32(max(abs(ou), abs(of)))
                    add(f"cuboid_fused_n{n}_a{axis}_{'in' if inside_u else 'out'}", n, lim, [cuboid(p, size)],
                        (c - 4, c - 4, c - 4), (c + 5, c + 5, c + 5), disc=True)
            assert done, ("no fused-sensitive cuboid", n, axis)
    for n, lim in ((16, 2.0), (100, 2.0)):
        c = n // 2
        add(f"cuboid_zero_n{n}", n, lim, [cuboid([node(c, lim / n)] * 3, [0.0, 0.0, 0.0])], (c - 1,) * 3, (c + 2,) * 3)
        add(f"cuboid_huge_n{n}", n, lim, [cuboid([1.0, 1.0, 1.0], [5.0, 5.0, 5.0])], (0, 0, 0), (4, 4, 4))

    # bounding box: every padding plane, both signs of u
    for n, lim in GRIDS:
        for sgn, u in (("pos", U_POS), ("neg", U_NEG)):
            add(f"bbox_lo_n{n}_{sgn}", n, lim, [("add_bounding_box", {})], (0, 0, 0), (5, 5, 5), u=u)
            add(f"bbox_hi_n{n}_{sgn}", n, lim, [("add_bounding_box", {})], (n - 5,) * 3, (n,) * 3, u=u)

    # time windows starting / ending exactly at a substep's float32 clock, for every grid BC kind
    dt, k = 1e-4, 7
    tk = float(f32(P.clock(dt, k)))
    for tag, win in (("start", dict(start_time=tk, end_time=999.0)), ("end", dict(start_time=0.0, end_time=tk))):
        for kk in (k - 1, k):
            add(f"window_collider_{tag}_k{kk}", 16, 2.0, [collider((1.0, 1.0, 1.9), (0.0, 0.0, 1.0), **win)],
                (7, 7, 7), (9, 9, 9), k=kk)
            add(f"window_cuboid_{tag}_k{kk}", 16, 2.0, [cuboid((1.0, 1.0, 1.0), (0.4, 0.4, 0.4), **win)],
                (7, 7, 7), (9, 9, 9), k=kk)
            add(f"window_bbox_{tag}_k{kk}", 16, 2.0, [("add_bounding_box", dict(win))], (0, 0, 0), (3, 3, 3), k=kk, u=U_NEG)

    # reset windows: (dt, end_time, substep) where end + 15 dt rounds differently when fused, and the neighbours
    picked = []
    for dtv in (1e-4, 5e-5, 2e-4, 3e-5):
        got = 0
        for m in range(2, 80):
            end = m * 1e-4 if dtv != 3e-5 else m * 3e-5
            if dtv == 1e-4 and m == 6:
                end = 6e-4
            for kk in range(int(end / dtv) + 10, int(end / dtv) + 20):
                t32 = f32(P.clock(dtv, kk))
                if t32 < f32(end):
                    continue
                if (t32 < P.reset_threshold(f32(end), f32(dtv), False)) != (t32 < P.reset_threshold(f32(end), f32(dtv), True)):
                    picked.append((dtv, end, kk))
                    got += 1
                    break
            if got == 3:
                break
    assert (1e-4, 6e-4, 21) in picked, picked
    for dtv, end, kk in picked:
        for k2 in sorted({kk, int(round(end / dtv)) + 14, int(round(end / dtv)) + 15, int(round(end / dtv)) + 16}):
            add(f"reset_dt{dtv:g}_end{end:g}_k{k2}", 16, 2.0, [cuboid((0.3, 0.3, 0.3), (0.05, 0.05, 0.05), end_time=end, reset=1)],
                (7, 7, 7), (9, 9, 9), k=k2, dt=dtv, disc=(k2 == kk))

    # a moving cuboid whose faces sweep across the nodes of a dx = 0.02 grid, then its reset window
    end = 0.00605                            # between two substeps' clocks
    for kk in range(80):                      # `modify` compares the Python-float clock: keep it on the kernel's side
        t = P.clock(1e-4, kk)
        assert (t < end) == (f32(t) < f32(end)) and (t < float(f32(end))) == (f32(t) < f32(end)), kk
    cases.append(dict(name="moving_cuboid_n100", n_grid=100, grid_lim=2.0, dt=1e-4, k=0, steps=80,
                      bcs=[("set_velocity_on_cuboid", dict(point=[1.01, 0.99, 1.003], size=[0.05, 0.05, 0.05],
                                                           velocity=[20.0, -12.0, 6.5], start_time=0.0, end_time=end,
                                                           reset=1))],
                      lo=[47, 42, 46], hi=[60, 53, 56], u=list(U_POS), vel=[20.0, -12.0, 6.5], disc=False))
    # the open modelling point, recorded: `modify` compares the Python-float clock with the float32 start time. The stand-in
    # (NumPy 2) compares in float32, the device and the oracle in double. A start time that rounds up from a substep's clock
    # starts the kernel's window at that substep while the double window starts one substep later, so from then on the
    # double-window cuboid lags one step behind. The fixture keeps the stand-in's classes and the double-window classes.
    ks = next(k for k in range(10, 40) if float(f32(P.clock(1e-4, k))) > P.clock(1e-4, k))
    cases.append(dict(name="moving_cuboid_window_open_point", n_grid=100, grid_lim=2.0, dt=1e-4, k=ks - 2, steps=24,
                      bcs=[("set_velocity_on_cuboid", dict(point=[1.01, 0.99, 1.003], size=[0.05, 0.05, 0.05],
                                                           velocity=[20.0, -12.0, 6.5],
                                                           start_time=float(f32(P.clock(1e-4, ks))), end_time=999.0))],
                      lo=[47, 44, 46], hi=[57, 53, 56], u=list(U_POS), vel=[20.0, -12.0, 6.5], disc=False, open_point=True))
    return cases


# ------------------------------------------------------------------------------------------ particle selections
def selection_cases(rng):
    out = {}
    # boxes: particles on each face and up to 3 float32 steps either side
    boxes = [((1.0, 1.0, 1.0), (0.25, 0.25, 0.25)), ((0.83, 1.17, 0.91), (0.07, 0.13, 0.0301))]
    xs = []
    for p, s in boxes:
        for axis in range(3):
            for sign in (-1, 1):
                face = f32(f32(p[axis]) + f32(sign * s[axis]))
                for k in range(-3, 4):
                    x = [f32(v) for v in p]
                    x[axis] = up(face, k)
                    xs.append(x)
    xs += list(rng.uniform(0.7, 1.3, size=(40, 3)).astype(f32))
    out["box_x"] = np.asarray(xs, f32)
    out["box_params"] = boxes
    # apply_additional_params: a different rule (p - s < x < p + s); two overlapping boxes, the later one wins
    mboxes = [dict(point=[1.0, 1.0, 1.0], size=[0.25, 0.25, 0.25], E=1e5, nu=0.3, density=900.0, material=2),
              dict(point=[1.2, 1.0, 1.0], size=[0.07, 0.13, 0.11], E=2e5, nu=0.25, density=1100.0, material=5)]
    xs = []
    for b in mboxes:
        for axis in range(3):
            for sign in (-1, 1):
                face = f32(f32(b["point"][axis]) + f32(sign) * f32(b["size"][axis]))
                for k in range(-2, 3):
                    x = [f32(v) for v in b["point"]]
                    x[axis] = up(face, k)
                    xs.append(x)
    xs += list(rng.uniform(0.7, 1.35, size=(40, 3)).astype(f32))
    out["mat_x"] = np.asarray(xs, f32)
    out["mat_boxes"] = mboxes
    # cylinder: caps and wall one step either side, and particles found by search where the fused form differs
    cyl = dict(point=[1.0, 1.0, 1.0], normal=[0.3, -0.7, 0.2], half_height_and_radius=[0.12, 0.15])
    from_ref = REFMOD.MPM_Simulator_WARP(1, n_grid=16, grid_lim=2.0, device="cpu")
    from_ref.load_initial_data_from_torch(__import__("torch").zeros(1, 3), __import__("torch").ones(1), n_grid=16, grid_lim=2.0,
                                          device="cpu")
    from_ref.enforce_particle_velocity_rotation(point=cyl["point"], normal=cyl["normal"],
                                                half_height_and_radius=cyl["half_height_and_radius"], rotation_scale=1.0,
                                                translation_scale=0.0, start_time=0.0, end_time=1.0, device="cpu")
    prm = from_ref.particle_velocity_modifier_params[0]
    n, h1 = prm.normal.a.copy(), prm.horizontal_axis_1.a.copy()
    hh, r = cyl["half_height_and_radius"]
    xs, disc = [], []
    for t in np.linspace(-1.3, 1.3, 9):
        for ang in np.linspace(0, 2 * np.pi, 7, endpoint=False):
            h2 = np.cross(h1, n)
            for kind in ("cap", "wall"):
                if kind == "cap":
                    base = np.asarray(cyl["point"]) + np.sign(t + 1e-9) * hh * n + 0.5 * r * (np.cos(ang) * h1 + np.sin(ang) * h2)
                else:
                    base = np.asarray(cyl["point"]) + 0.8 * t * hh * n + r * (np.cos(ang) * h1 + np.sin(ang) * h2)
                for k in (-2, -1, 0, 1, 2):
                    x = np.asarray([up(f32(v), k) for v in base], f32)
                    xs.append(x)
    xs = np.asarray(xs, f32)
    # search: perturb wall / cap particles until the fused and unfused masks differ
    cand = []
    for i in range(4000):
        b = xs[rng.integers(len(xs))]
        x = np.asarray([up(v, int(rng.integers(-6, 7))) for v in b], f32)
        mu_ = P.select_cylinder(x[None], cyl["point"], n, hh, r, fused=False)[0]
        mf = P.select_cylinder(x[None], cyl["point"], n, hh, r, fused=True)[0]
        if mu_ != mf:
            cand.append((x, int(mu_)))
        if len(cand) >= 24 and len({c[1] for c in cand}) == 2:
            break
    assert len({c[1] for c in cand}) == 2, "no fused-sensitive cylinder particles in both directions"
    out["cyl_x"] = np.concatenate([xs, np.asarray([c[0] for c in cand], f32)])
    # rotation modifier: particles on the half-plane dot(x - point, h2) = 0 (offset along h1 and n), where theta's sign is
    # decided by a float32 zero or by a last-bit difference that a fused dot product would round the other way
    h2r = prm.horizontal_axis_2.a.copy()
    zero, flip = [], []
    pt = np.asarray(cyl["point"], f32)
    ks = np.stack(np.meshgrid(*[np.arange(-3, 4)] * 3, indexing="ij"), -1).reshape(-1, 3)
    for _ in range(3000):
        a = rng.choice([-1.0, 1.0]) * rng.uniform(0.02, 0.14)
        b = rng.uniform(-0.1, 0.1)
        base = (pt.astype(np.float64) + a * h1.astype(np.float64) + b * n.astype(np.float64)).astype(f32)
        xs_ = np.stack([np.asarray([up(base[d], int(k[d])) for d in range(3)], f32) for k in ks])
        o = (xs_ - pt).astype(f32)
        pr = (o * h2r).astype(f32)                                  # the unfused dot product, vectorised
        du = ((pr[:, 0] + pr[:, 1]).astype(f32) + pr[:, 2]).astype(f32)
        for j in np.flatnonzero(np.abs(du) < 1e-8):
            x, oj = xs_[j], o[j]
            on = P.dot(oj, n, False)
            h = np.array([f32(oj[d] - P.mul(on, n[d])) for d in range(3)], f32)
            cosine = f32(P.dot(oj, h1, False) / f32(np.sqrt(P.dot(h, h, False))))
            if not abs(cosine) < f32(1.0):          # theta = 0 or pi: its sign cannot show in the velocity
                continue
            if du[j] == 0 and len(zero) < 12:
                zero.append(x)
            elif du[j] != 0 and (du[j] > 0) != (P.dot(oj, h2r, True) > 0) and len(flip) < 30:
                flip.append(x)
        if len(zero) >= 12 and len(flip) >= 30:
            break
    assert len(zero) >= 4 and len(flip) >= 10, (len(zero), len(flip))
    out["rot_x"] = np.concatenate([np.asarray(zero, f32), np.asarray(flip, f32)])
    out["rot_disc"] = np.concatenate([np.zeros(len(zero), bool), np.ones(len(flip), bool)])
    out["rot"] = dict(cyl, rotation_scale=2.0, translation_scale=0.1, start_time=0.0, end_time=1.0)
    out["cyl_disc"] = np.concatenate([np.zeros(len(xs), bool), np.ones(len(cand), bool)])
    out["cyl"] = cyl
    # release_particles_sequentially: particles on the 50 nested faces along z, one step either side
    rel = dict(normal=[0, 0, 1], start_position=0.3, end_position=1.1, num_layers=10, start_time=0.0, end_time=0.37)
    half = f32(f32(np.abs(f32(rel["start_position"] - rel["end_position"]))) / f32(50))
    xs = []
    for i in range(0, 50, 3):
        size = f32(half * f32(50 - i))
        for sign in (-1, 1):
            face = f32(f32(rel["end_position"]) + f32(sign) * size)
            for k in (-1, 0, 1):
                xs.append([f32(1.0), f32(1.0), up(face, k)])
    out["rel_x"] = np.asarray(xs, f32)
    out["rel"] = rel
    return out


def run_selections(sel):
    import torch
    rec = {}

    def solver(x):
        s = REFMOD.MPM_Simulator_WARP(len(x), n_grid=16, grid_lim=2.0, device="cpu")
        s.load_initial_data_from_torch(torch.from_numpy(x.copy()), torch.ones(len(x)), n_grid=16, grid_lim=2.0, device="cpu")
        return s

    s = solver(sel["box_x"])
    for p, sz in sel["box_params"]:
        s.add_impulse_on_particles(force=[1.0, 0.0, 0.0], dt=1e-4, point=list(p), size=list(sz), num_dt=3, device="cpu")
        s.enforce_particle_velocity_translation(point=list(p), size=list(sz), velocity=[0.0, 0.0, 0.0], start_time=0.0,
                                                end_time=1.0, device="cpu")
    rec["box_masks"] = np.stack([np.array(q.mask.numpy(), np.int32) for q in list(s.impulse_params) + list(s.particle_velocity_modifier_params)])
    s = solver(sel["mat_x"])
    s.set_parameters_dict(dict(material="jelly", E=3e5, nu=0.2, density=1000.0,
                               additional_material_params=[dict(b) for b in sel["mat_boxes"]]), device="cpu")
    rec["mat_material"] = np.array(s.mpm_state.particle_material.numpy(), np.int32)
    s = solver(sel["cyl_x"])
    c = sel["cyl"]
    s.enforce_particle_velocity_rotation(point=c["point"], normal=c["normal"], half_height_and_radius=c["half_height_and_radius"],
                                         rotation_scale=1.0, translation_scale=0.0, start_time=0.0, end_time=1.0, device="cpu")
    rec["cyl_mask"] = np.array(s.particle_velocity_modifier_params[0].mask.numpy(), np.int32)
    rec["cyl_normal"] = s.particle_velocity_modifier_params[0].normal.a.copy()
    hh, r = c["half_height_and_radius"]
    unf = P.select_cylinder(sel["cyl_x"], c["point"], rec["cyl_normal"], hh, r, fused=False)
    fus = P.select_cylinder(sel["cyl_x"], c["point"], rec["cyl_normal"], hh, r, fused=True)
    assert (unf == rec["cyl_mask"]).all(), "unfused cylinder restatement differs from the reference"
    assert (fus != rec["cyl_mask"])[sel["cyl_disc"]].all(), "a fused-sensitive cylinder particle does not separate"
    assert (P.select_box(sel["box_x"], *sel["box_params"][0]) == rec["box_masks"][0]).all()
    assert (P.additional_params_material(sel["mat_x"], sel["mat_boxes"], 0) == rec["mat_material"]).all()
    s = solver(sel["rot_x"])
    c = sel["rot"]
    s.enforce_particle_velocity_rotation(**c, device="cpu")
    prm = s.particle_velocity_modifier_params[0]
    assert np.asarray(prm.mask.numpy()).all(), "every half-plane particle lies inside the cylinder"
    rec["rot_h1"], rec["rot_h2"], rec["rot_normal"] = prm.horizontal_axis_1.a.copy(), prm.horizontal_axis_2.a.copy(), prm.normal.a.copy()
    wp.launch(kernel=s.particle_velocity_modifiers[0], dim=len(sel["rot_x"]), inputs=[0.5, s.mpm_state, prm], device="cpu")
    rec["rot_v"] = np.array(s.mpm_state.particle_v.numpy(), f32)
    pos = P.rotation_theta_positive(sel["rot_x"], c["point"], rec["rot_h2"], fused=False)
    a1 = rec["rot_v"].astype(np.float64) @ rec["rot_h1"].astype(np.float64)      # -hd sin(theta) rotation_scale
    assert ((a1 < 0) == pos).all() and (a1 != 0).all(), "the stand-in's velocity does not show theta's sign"
    fus = P.rotation_theta_positive(sel["rot_x"], c["point"], rec["rot_h2"], fused=True)
    assert (fus != pos)[sel["rot_disc"]].all()
    rec["rot_theta_pos"] = pos
    s = solver(sel["rel_x"])
    s.release_particles_sequentially(**sel["rel"])
    rec["rel_masks"] = np.stack([np.array(q.mask.numpy(), np.int32) for q in s.particle_velocity_modifier_params])
    rec["rel_size"] = np.stack([q.size.a.copy() for q in s.particle_velocity_modifier_params])
    rec["rel_end_time"] = np.array([f32(q.end_time) for q in s.particle_velocity_modifier_params], f32)
    return rec


# ------------------------------------------------------------------------------------------ host-side parameters
def parameter_cases(rng):
    normals = [[0.0, 0.0, 1.0], [0.0, 0.3, 1.0], [-1.0, 0.0, 0.1], [0.0, 0.0, 2.0], [0.0, 1.0, 0.0], [1.0, 1.0, 1.0],
               [0.3, -0.7, 0.2], [0.0, 0.0, 3.0], [1, 2, 2], [-3, 0, 4]]
    normals += [list(map(float, v)) for v in np.round(rng.uniform(-2, 2, size=(150, 3)), 3)]
    normals += [list(map(int, v)) for v in rng.integers(-5, 6, size=(40, 3)) if np.any(v)]
    out = {"normals_in": np.asarray(normals, np.float64)}
    s = REFMOD.MPM_Simulator_WARP(1, n_grid=16, grid_lim=2.0, device="cpu")
    for nv in normals:
        s.add_surface_collider([1.0, 1.0, 1.0], nv)
    out["collider_normal"] = np.stack([p.normal.a.copy() for p in s.collider_params])
    for nv in normals:
        s.enforce_particle_velocity_rotation(point=[1.0, 1.0, 1.0], normal=nv, half_height_and_radius=[0.1, 0.1],
                                             rotation_scale=1.0, translation_scale=0.0, start_time=0.0, end_time=1.0,
                                             device="cpu")
    prm = s.particle_velocity_modifier_params
    out["rot_normal"] = np.stack([p.normal.a.copy() for p in prm])
    out["rot_h1"] = np.stack([p.horizontal_axis_1.a.copy() for p in prm])
    out["rot_h2"] = np.stack([p.horizontal_axis_2.a.copy() for p in prm])
    rels = [(0.3, 1.1, 0.37), (1.7, 0.2, 1.0), (0.05, 1.95, 3e-3), (1.0, 1.0 + 1e-7, 0.123456)]
    out["release_in"] = np.asarray(rels, np.float64)
    sizes, ends = [], []
    for a, b, e in rels:
        s2 = REFMOD.MPM_Simulator_WARP(1, n_grid=16, grid_lim=2.0, device="cpu")
        s2.release_particles_sequentially([0, 1, 0], a, b, 10, 0.0, e)
        sizes.append(np.stack([q.size.a.copy() for q in s2.particle_velocity_modifier_params]))
        ends.append(np.array([f32(q.end_time) for q in s2.particle_velocity_modifier_params], f32))
    out["release_size"], out["release_end_time"] = np.stack(sizes), np.stack(ends)
    imps = [(0.0, 1e-4, 8), (2e-4, 1e-4, 8), (3e-5, 3e-5, 7), (0.1, 2e-4, 33)]
    out["impulse_in"] = np.asarray(imps, np.float64)
    ends = []
    for st, dtv, nd in imps:
        s.add_impulse_on_particles(force=[1.0, 0.0, 0.0], dt=dtv, point=[1, 1, 1], size=[1, 1, 1], num_dt=nd, start_time=st,
                                   device="cpu")
        ends.append(f32(s.impulse_params[-1].end_time))
    out["impulse_end_time"] = np.asarray(ends, f32)
    return out


def main():
    rng = np.random.default_rng(20261017)
    blob, meta = {}, {"grid": [], "selection": {}}
    for i, c in enumerate(grid_cases()):
        cls, records = run_grid_case(c)
        unf = P.restate_case(c, records, fused=False)
        assert (unf == cls).all(), (c["name"], "unfused restatement differs from the reference", np.argwhere(unf != cls)[:5])
        assert (cls != P.UNKNOWN).all(), c["name"]
        fus = P.restate_case(c, records, fused=True)
        if c["disc"]:
            assert (fus != cls).any(), (c["name"], "meant to separate fused from unfused, but does not")
        f64w = P.restate_case(c, records, fused=False, window="f64")
        if c.get("open_point"):
            assert (f64w != cls).any(), (c["name"], "the open-point case does not separate the two windows")
            blob[f"grid/{i}/cls_f64_window"] = f64w
        else:
            assert (f64w == cls).all(), (c["name"], "depends on the float32 / double window of `modify`")
        m = dict(c, records=records, fused_differs=bool((fus != cls).any()))
        m["bcs"] = [[meth, kw] for meth, kw in c["bcs"]]
        meta["grid"].append(m)
        blob[f"grid/{i}/cls"] = cls
        print(f"{c['name']:40s} nodes {cls.shape[1]:5d} x {cls.shape[0]:2d}  classes {sorted(set(cls.ravel().tolist()))}"
              f"  fused differs {m['fused_differs']}", flush=True)
    sel = selection_cases(rng)
    rec = run_selections(sel)
    for k in ("box_x", "mat_x", "cyl_x", "cyl_disc", "rel_x", "rot_x", "rot_disc"):
        blob[f"sel/{k}"] = sel[k]
    for k, v in rec.items():
        blob[f"sel/{k}"] = v
    meta["selection"] = {k: sel[k] for k in ("box_params", "mat_boxes", "cyl", "rel", "rot")}
    for k, v in parameter_cases(rng).items():
        blob[f"param/{k}"] = v
    blob["meta"] = np.frombuffer(json.dumps(meta, default=float).encode(), dtype=np.uint8)
    np.savez_compressed(os.path.join(HERE, "mpm_bc_edges_golden.npz"), **blob)
    print("wrote", os.path.join(HERE, "mpm_bc_edges_golden.npz"), len(blob), "arrays")


if __name__ == "__main__":
    main()
