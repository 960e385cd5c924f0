"""Scenarios of the MPM golden fixtures (GOLDEN-VECTOR TOOLING, shared by the generator and the tests).

A scenario is pure data: seeded particle arrays, a `set_parameters_dict` dictionary, a list of boundary-condition
calls (method name + kwargs of the reference's `MPM_Simulator_WARP`) and checkpoints.  `replay()` drives ANY object
with the reference's call surface through it:
  * the reference class itself, imported from a checkout of the reference and executed on tests/golden/_fake_warp.py
    (make_mpm_golden.py -> tests/golden/mpm_golden.npz),
  * tests/oracle_solver.OracleSolver (oracle/mpm_ref.c behind the same surface)          -> CPU test,
  * pixie_b200.mpm_solver_warp.MPM_Simulator_WARP (the CUDA path through the C ABI)       -> `-m gpu` test.

Geometry: 16^3 grid over [0,2]^3 (dx = 0.125), 96-120 particles; every stencil stays inside the grid (the reference
indexes out of bounds otherwise).  Box faces and planes are kept off the grid nodes and off the particles.
"""
from __future__ import annotations

import copy

import numpy as np

N_GRID, GRID_LIM, DT = 16, 2.0, 1e-4
CHECKPOINTS = (1, 20)      # substeps after which the state is recorded
PARTICLE_FIELDS = ("particle_x", "particle_v", "particle_C", "particle_F", "particle_F_trial", "particle_stress",
                   "particle_cov")
MODEL_FIELDS = ("yield_stress", "mu", "lam", "E", "nu")


def _particles(seed, n, lo=(0.75, 0.75, 0.75), hi=(1.25, 1.25, 1.25), f_amp=0.12, v_amp=0.6):
    rng = np.random.default_rng(seed)
    x = rng.uniform(lo, hi, size=(n, 3)).astype(np.float32)
    vol = (rng.uniform(0.5, 1.5, size=n) * (GRID_LIM / N_GRID) ** 3 / 6).astype(np.float32)
    cov = np.abs(rng.standard_normal((n, 6))).astype(np.float32) * 1e-3
    v = (v_amp * rng.standard_normal((n, 3))).astype(np.float32)
    C = (2.0 * rng.standard_normal((n, 3, 3))).astype(np.float32)
    F = (np.eye(3)[None] + f_amp * rng.standard_normal((n, 3, 3))).astype(np.float32)
    return dict(x=x, vol=vol, cov=cov, v=v, C=C, F_trial=F)


_BASE = dict(E=2e5, nu=0.3, density=1000.0, g=[0.0, 0.0, -9.8], yield_stress=3e3, bulk_modulus=1e5,
             grid_v_damping_scale=0.9999, rpic_damping=0.0, friction_angle=30.0, hardening=1, xi=0.2, softening=0.1,
             plastic_viscosity=8.0)

_COMMON_BCS = [
    ("add_bounding_box", {}),
    ("set_velocity_on_cuboid", dict(point=[1.0, 1.0, 0.81], size=[0.3, 0.3, 0.07], velocity=[0.0, 0.0, 0.0])),
    ("add_surface_collider", dict(point=[1.0, 1.0, 0.70], normal=[0.0, 0.0, 2.0], surface="sticky", friction=0.0,
                                  start_time=0.0, end_time=1e3)),
    ("add_impulse_on_particles", dict(force=[0.02, 0.0, -0.01], dt=DT, point=[1.0, 1.0, 1.1], size=[0.2, 0.2, 0.1],
                                      num_dt=8, start_time=2 * DT)),
    ("enforce_particle_velocity_translation", dict(point=[1.15, 1.15, 0.95], size=[0.08, 0.08, 0.08],
                                                   velocity=[0.0, 0.2, 0.0], start_time=5 * DT, end_time=12 * DT)),
]


def scenarios():
    out = []
    for name, mat in (("jelly", "jelly"), ("metal", "metal"), ("sand", "sand"), ("snow", "snow"), ("stationary", "stationary")):
        out.append(dict(name=name, seed=11 + len(out), n=96, params=dict(_BASE, material=mat), bcs=copy.deepcopy(_COMMON_BCS),
                        f_amp=0.25 if mat in ("metal", "snow") else 0.12))
    # visplas (id 3) and fluid (id 4) are excluded from NAME_TO_MATERIAL_ID (mpm_solver_warp.py:20-26): they are only
    # reachable through numeric ids in additional_material_params, which is how the mixed scenario sets them.
    boxes = []
    for i, (mid, E, nu, rho) in enumerate(((0, 1.5e5, 0.25, 900.0), (1, 3e5, 0.3, 1500.0), (2, 1e5, 0.28, 1300.0),
                                           (3, 8e4, 0.35, 1100.0), (4, 5e4, 0.4, 1000.0), (5, 2e5, 0.22, 400.0),
                                           (6, 1e5, 0.3, 1000.0))):
        lo = 0.75 + 0.5 * i / 7.0
        boxes.append(dict(point=[lo + 0.25 / 7.0, 1.0, 1.0], size=[0.25 / 7.0, 0.3, 0.3], E=E, nu=nu, density=rho, material=mid))
    boxes.append(dict(point=[1.0, 1.2, 1.2], size=[0.1, 0.04, 0.04], E=4e5, nu=0.2, density=2000.0, material="sand"))
    out.append(dict(name="mixed", seed=31, n=120, params=dict(_BASE, material="jelly", additional_material_params=boxes),
                    bcs=copy.deepcopy(_COMMON_BCS), f_amp=0.2))
    # every other code path: rpic damping, update_cov_with_F, no grid damping, moving cuboid with reset, the three
    # non-sticky surface types, rotation modifier, a wall cluster that reaches the bounding-box padding
    out.append(dict(name="paths", seed=41, n=110, update_cov_with_F=True,
                    params=dict(_BASE, material="jelly", rpic_damping=0.3, grid_v_damping_scale=1.1, spawn_offset=[0.01, -0.02, 0.0]),
                    wall_cluster=True,
                    bcs=[("add_bounding_box", dict(start_time=0.0, end_time=15 * DT)),
                         ("set_velocity_on_cuboid", dict(point=[0.83, 1.0, 1.21], size=[0.07, 0.3, 0.07], velocity=[40.0, 0.0, 0.0],
                                                         start_time=0.0, end_time=6 * DT, reset=1)),
                         ("add_surface_collider", dict(point=[1.0, 1.0, 0.80], normal=[0.0, 0.3, 1.0], surface="slip", friction=0.2,
                                                       start_time=10 * DT, end_time=999.0)),
                         ("add_surface_collider", dict(point=[1.0, 0.78, 1.0], normal=[0.0, 1.0, 0.0], surface="cut", friction=0.0)),
                         ("add_surface_collider", dict(point=[1.24, 1.0, 1.0], normal=[-1.0, 0.0, 0.1], surface="separate", friction=0.5,
                                                       start_time=3 * DT, end_time=9 * DT)),
                         ("enforce_particle_velocity_rotation", dict(point=[1.0, 1.0, 1.0], normal=[0.0, 0.0, 3.0],
                                                                     half_height_and_radius=[0.12, 0.15], rotation_scale=2.0,
                                                                     translation_scale=0.1, start_time=0.0, end_time=7 * DT))]))
    out.append(dict(name="pic", seed=51, n=96, params=dict(_BASE, material="jelly", rpic_damping=-1.0), bcs=[], f_amp=0.05))
    return out


def inputs(sc):
    p = _particles(sc["seed"], sc["n"], f_amp=sc.get("f_amp", 0.12))
    if sc.get("wall_cluster"):
        k = sc["n"] // 4          # a cluster near the -x wall, moving outward: nodes 1..3 meet the bounding box padding
        rng = np.random.default_rng(sc["seed"] + 1000)
        # (z in the 0.4..0.53 band hard-coded in the "cut" collider, y below its plane: mpm_solver_warp.py:809-820)
        p["x"][:k] = rng.uniform((0.27, 0.6, 0.42), (0.40, 0.9, 0.62), size=(k, 3)).astype(np.float32)
        p["v"][:k, 0] = -np.abs(p["v"][:k, 0]) - 0.5
    return p


def replay(solver_cls, sc, be, checkpoints=CHECKPOINTS, data=None):
    """Drive `solver_cls` (reference call surface) through scenario `sc`.  `be` adapts what differs between the
    back ends: tensor placement and direct array assignment (`wp.from_torch(...)` in the reference,
    material_field.py:322 / gs_simulation.py:528; a torch tensor in the product).  Returns {checkpoint: {field: ndarray}}
    plus the selection masks and the post-setup per-particle parameters."""
    d = data if data is not None else inputs(sc)
    n = sc["n"]
    s = solver_cls(n, n_grid=N_GRID, grid_lim=GRID_LIM, device=be.device)
    s.load_initial_data_from_torch(be.tensor(d["x"]), be.tensor(d["vol"]), be.tensor(d["cov"]), n_grid=N_GRID,
                                   grid_lim=GRID_LIM, device=be.device)
    if sc.get("update_cov_with_F"):
        # initialize() resets the flag (mpm_solver_warp.py:74), so it is set after loading and the covariance is seeded by hand
        s.mpm_model.update_cov_with_F = True
        be.set_state(s, "particle_cov", d["cov"].reshape(-1).copy())
    s.set_parameters_dict(copy.deepcopy(sc["params"]), device=be.device)
    s.finalize_mu_lam(device=be.device)
    s.import_particle_v_from_torch(be.tensor(d["v"]), device=be.device)
    s.import_particle_C_from_torch(be.tensor(d["C"]), device=be.device)
    be.set_state(s, "particle_F_trial", d["F_trial"].copy())
    for method, kw in sc["bcs"]:
        kw = dict(kw)
        if method in ("add_impulse_on_particles", "enforce_particle_velocity_translation", "enforce_particle_velocity_rotation"):
            kw["device"] = be.device
        getattr(s, method)(**kw)
    out = {"setup": dict(be.get_model(s, ("E", "nu", "mu", "lam")), **be.get_state(s, ("particle_mass", "particle_density",
                                                                                        "particle_material", "particle_x")))}
    out["masks"] = be.get_masks(s)
    done = 0
    for cp in checkpoints:
        for i in range(done, cp):
            s.p2g2p(i, DT, device=be.device)
        done = cp
        rec = dict(be.get_state(s, PARTICLE_FIELDS), **be.get_model(s, MODEL_FIELDS))
        rec["time"] = np.float64(s.time)
        if cp == checkpoints[0]:
            rec.update(be.get_grid(s))
        out[cp] = rec
    # export kernels (compute_cov_from_F only runs when update_cov_with_F is off: mpm_solver_warp.py:726-741)
    exp = {"R": np.asarray(be.to_numpy(s.export_particle_R_to_torch(device=be.device))).reshape(n, 9).copy(),
           "cov": np.asarray(be.to_numpy(s.export_particle_cov_to_torch(device=be.device))).reshape(n, 6).copy()}
    out["export"] = exp
    return out
