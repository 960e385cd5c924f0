"""MPM rollouts through the host/device state machine of pixie_b200/csrc/mpm.cu, against the C oracle.

The substep kernels are tied to fp64 references one substep at a time elsewhere (test_gpu_mpm_constitutive.py,
test_gpu_mpm_transfer.py). What decides which state, parameters and boundary-condition table those kernels see over a
rollout is the host side: the cell-sorted private copy of the particles (written back by every export, gathered and
sorted again by the next step, re-sorted every kResortEvery substeps), the CUDA-graph cache keyed by (count, clock
parity, dt), the clock and moving-cuboid points kept in two parity slots, and the inline / device-table paths of the
particle BCs. A bug there changes the trajectory, not the per-substep numerics.

A scenario is a setup plus a script of operations (step, export, in-place edit, BC, parameters, clock, rebind) that is
applied in lockstep to the CUDA shim and to the oracle in fp32 and fp64. Particle-BC selections of the first back end
(the device when there is one) are handed to the others, so a particle on a selection boundary cannot make them diverge;
box selections must be identical anyway. Positions and other fields are recorded at the script's exports (an export is a
write-back, so recording after every step would hide the unsynchronised paths); the clock after every step.

Judging, as the rest of the suite does: against the fp32 oracle everywhere (moving cuboids cross grid nodes at a step
that depends on the precision, see test_gpu_mpm.py); scenes without a moving cuboid also against fp64, drift below
20 x (fp32 oracle vs fp64 oracle) + 1e-6. Clock equal to the oracle's to 1e-12 after every step.

Bounds: `_TOL` below, set from the maxima measured on one H100 80GB HBM3 (700 W) with the headroom stated there.
"""
import copy
import os
import re
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, HERE)

import mpm_scenarios as S  # noqa: E402
from mpm_backends import OracleSolver  # noqa: E402
from oracle import mpm_ref as R  # noqa: E402

DEV = "cuda:0"
DT = S.DT
ROOT = os.path.dirname(HERE)

# max |CUDA - fp32 oracle| per recorded field, by test family. Measured maxima on one H100 80GB HBM3 (700 W power limit),
# bounds about 3-5x above them:
#   chop  (paths / mixed / 5000-particle synthetic, 240 substeps): X 5.1e-6, V 4.4e-4, F 2.2e-4, C 6.2e-3, cov 4.3e-7, R 2.2e-5
#   frame (6 frames of 333 / 400 substeps, every material):       X 2.7e-4, V 2.9e-3, F 1.6e-3, C 1.6e-2, cov 1.8e-8, R 6.8e-4
#   pbc   (3..101 particle BCs, 200 substeps, jelly):             X 1.2e-6, V 4.9e-5, F 9.7e-6, C 6.7e-4, R 1.8e-6
#   mid   (metal / snow / jelly, 270 substeps):                   X 1.8e-5, V 1.5e-3, F 1.2e-4, C 1.0e-2, R 7.5e-5, yield 10, mu / lam 0
#         (the largest are the "plastic" case, where every snow particle's mu and lam reach 0 on the device)
# Drift vs fp64 next to the fp32-vs-fp64 floor where there is no moving cuboid: mixed 7.9e-6 / 7.9e-6, pbc 5.1e-6 / 5.1e-6.
_TOL = {
    "chop": {"X": 2e-5, "V": 2e-3, "F": 1e-3, "F_TRIAL": 1e-3, "C": 3e-2, "COV": 2e-6, "R": 1e-4},
    "frame": {"X": 1e-3, "V": 1e-2, "F": 5e-3, "F_TRIAL": 5e-3, "C": 5e-2, "COV": 1e-7, "R": 3e-3},
    "pbc": {"X": 5e-6, "V": 2e-4, "F": 4e-5, "F_TRIAL": 4e-5, "C": 3e-3, "COV": 1e-9, "R": 1e-5},
    "mid": {"X": 6e-5, "V": 5e-3, "F": 5e-4, "F_TRIAL": 5e-4, "C": 5e-2, "COV": 1e-9, "R": 3e-4, "YIELD": 40.0, "MU": 1.0, "LAM": 1.0},
}


# ------------------------------------------------------------------------------------------------ scenes
def _stretched_paths(bbox_end=163 * DT):
    """The golden `paths` setup with its BC windows stretched over graph replays and the re-sort at substep 100: windows
    37..163 DT, the reset=1 cuboid ending at the odd substep 117 (slowed down so it keeps particles inside the grid)."""
    sc = copy.deepcopy(next(s for s in S.scenarios() if s["name"] == "paths"))
    d = S.inputs(sc)
    w0, w1 = 37 * DT, 163 * DT
    bcs = [("add_bounding_box", dict(start_time=0.0, end_time=bbox_end)),
           ("set_velocity_on_cuboid", dict(point=[0.83, 1.0, 1.21], size=[0.07, 0.3, 0.07], velocity=[4.0, 0.0, 0.0],
                                           start_time=0.0, end_time=117 * DT, reset=1)),
           ("add_surface_collider", dict(point=[1.0, 1.0, 0.80], normal=[0.0, 0.3, 1.0], surface="slip", friction=0.2,
                                         start_time=w0, end_time=999.0)),
           ("add_surface_collider", dict(point=[1.0, 0.78, 1.0], normal=[0.0, 1.0, 0.0], surface="cut", friction=0.0)),
           ("add_surface_collider", dict(point=[1.24, 1.0, 1.0], normal=[-1.0, 0.0, 0.1], surface="separate", friction=0.5,
                                         start_time=w0, end_time=w1)),
           ("enforce_particle_velocity_rotation", dict(point=[1.0, 1.0, 1.0], normal=[0.0, 0.0, 3.0], half_height_and_radius=[0.12, 0.15],
                                                       rotation_scale=2.0, translation_scale=0.1, start_time=w0, end_time=w1))]
    return dict(name="paths", n=sc["n"], n_grid=S.N_GRID, grid_lim=S.GRID_LIM, x=d["x"], vol=d["vol"], cov=d["cov"], v=d["v"], C=d["C"],
                F_trial=d["F_trial"], params=sc["params"], ucov=True, bcs=bcs, moving=True)


def _stretched_mixed():
    """The golden `mixed` setup (every material through additional_material_params) with the impulse open over 37..163 DT
    and the velocity translation over 63..137 DT."""
    sc = copy.deepcopy(next(s for s in S.scenarios() if s["name"] == "mixed"))
    d = S.inputs(sc)
    bcs = copy.deepcopy(sc["bcs"])
    bcs[3] = ("add_impulse_on_particles", dict(force=[0.02, 0.0, -0.01], dt=DT, point=[1.0, 1.0, 1.1], size=[0.2, 0.2, 0.1],
                                               num_dt=126, start_time=37 * DT))
    bcs[4] = ("enforce_particle_velocity_translation", dict(point=[1.15, 1.15, 0.95], size=[0.08, 0.08, 0.08], velocity=[0.0, 0.2, 0.0],
                                                            start_time=63 * DT, end_time=137 * DT))
    return dict(name="mixed", n=sc["n"], n_grid=S.N_GRID, grid_lim=S.GRID_LIM, x=d["x"], vol=d["vol"], cov=d["cov"], v=d["v"], C=d["C"],
                F_trial=d["F_trial"], params=sc["params"], bcs=bcs, moving=False)


_SYN_PARAMS = {"material": "jelly", "g": [0.0, 0.0, -9.8], "density": 1000.0, "E": 1e5, "nu": 0.3, "yield_stress": 2e3,
               "grid_v_damping_scale": 0.9999, "rpic_damping": 0.0, "friction_angle": 30.0, "hardening": 1, "xi": 0.1,
               "softening": 0.1, "plastic_viscosity": 10.0, "bulk_modulus": 1e5}


def _synthetic(n=5000, ng=32, materials=(0, 1, 2, 3, 4, 5, 6), seed=3, bcs="windows"):
    """synthetic_scene (per-particle E, nu, density, material) on a 2.0 box. `bcs`: "windows" = bounding box, a static
    floor cuboid, a reset=1 cuboid moving until the odd substep 117, a sticky plane, an impulse over 37..63 DT and a
    velocity translation over 63..137 DT; "bbox" = the bounding box only."""
    sc = R.synthetic_scene(n, ng, seed=seed, materials=materials)
    out = dict(name="synthetic", n=n, n_grid=ng, grid_lim=2.0, x=sc["x"], vol=sc["vol"], v=sc["v"], params=dict(_SYN_PARAMS),
               per=dict(E=sc["E"], nu=sc["nu"], material=sc["material"], density=sc["density"]), moving=False)
    out["bcs"] = [("add_bounding_box", {})]
    if bcs == "windows":
        out["bcs"] += [
            ("set_velocity_on_cuboid", dict(point=[1.0, 1.0, 0.62], size=[0.51, 0.51, 0.04], velocity=[0.0, 0.0, 0.0])),
            ("set_velocity_on_cuboid", dict(point=[0.7, 1.0, 1.3], size=[0.05, 0.2, 0.05], velocity=[0.5, 0.0, 0.0], start_time=0.0,
                                            end_time=117 * DT, reset=1)),
            ("add_surface_collider", dict(point=[1.0, 1.0, 0.1], normal=[0.0, 0.0, 2.0], surface="sticky", friction=0.0, end_time=1e3)),
            ("add_impulse_on_particles", dict(force=[0.5, 0.0, -0.2], dt=DT, point=[1.0, 1.0, 1.2], size=[0.2, 0.2, 0.1], num_dt=26,
                                              start_time=37 * DT)),
            ("enforce_particle_velocity_translation", dict(point=[1.3, 1.3, 0.9], size=[0.1, 0.1, 0.1], velocity=[0.0, 0.2, 0.0],
                                                           start_time=63 * DT, end_time=137 * DT))]
        out["moving"] = True
    return out


def _particle_bcs(k):
    """k particle BCs with staggered windows and overlapping selections: impulses, translations and rotations in turn
    (the last of 5 and of 8 is a translation, so the last entry of the device table decides velocities)."""
    out = []
    for i in range(k):
        t0 = (7 + 11 * i) * DT
        t1 = t0 + (60 + 9 * i) * DT
        c = [1.0 + 0.09 * (i % 3 - 1), 1.0 + 0.07 * (i % 2) - 0.035, 1.0 + 0.05 * (i % 4 - 1.5)]
        if i % 3 == 0:
            out.append(("add_impulse_on_particles", dict(force=[2.0 - 0.3 * i, 0.5, 1.0], dt=DT, point=c, size=[0.25, 0.25, 0.2],
                                                         num_dt=60 + 9 * i, start_time=t0)))
        elif i % 3 == 1:
            out.append(("enforce_particle_velocity_translation", dict(point=c, size=[0.2, 0.3, 0.25], velocity=[0.1 * i, -0.2, 0.05 * i],
                                                                      start_time=t0, end_time=t1)))
        else:
            # a narrow cylinder and a short window: the reference's acos of a cosine that rounds above 1 is NaN
            out.append(("enforce_particle_velocity_rotation", dict(point=c, normal=[0.0, 0.0, 1.0], half_height_and_radius=[0.1, 0.12],
                                                                   rotation_scale=1.5, translation_scale=0.1, start_time=t0,
                                                                   end_time=t0 + 20 * DT)))
    return out


# ------------------------------------------------------------------------------------------------ harness
class _Oracle(OracleSolver):
    """OracleSolver that can take the selection masks of another back end (`add`)."""

    def __init__(self, sc, precision):
        super().__init__(sc["n"], sc["n_grid"], sc["grid_lim"], precision=precision)

    def add(self, method, kw, masks=None):
        """Calls BC `method`; with `masks`, its selections are replaced by them in order. Returns [(kind, own selection)]."""
        own = []
        if masks is not None:
            it = iter(masks)
            box, cyl = self.o.select_box, self.o.select_cylinder
            self.o.select_box = lambda *a: (own.append(("box", box(*a))), np.asarray(next(it), dtype=np.int32))[1]
            self.o.select_cylinder = lambda *a: (own.append(("cyl", cyl(*a))), np.asarray(next(it), dtype=np.int32))[1]
        try:
            getattr(self, method)(**copy.deepcopy(kw))
        finally:
            if masks is not None:
                del self.o.select_box, self.o.select_cylinder
        return own


def _setup_cuda(sc):
    from pixie_b200.mpm_solver_warp import MPM_Simulator_WARP

    def T(a):
        return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)

    s = MPM_Simulator_WARP(sc["n"], n_grid=sc["n_grid"], grid_lim=sc["grid_lim"], device=DEV)
    s.load_initial_data_from_torch(T(sc["x"]), T(sc["vol"]), T(sc["cov"]) if "cov" in sc else None, n_grid=sc["n_grid"],
                                   grid_lim=sc["grid_lim"], device=DEV)
    if sc.get("ucov"):
        s.mpm_model.update_cov_with_F = True
        s.mpm_state.particle_cov = T(sc["cov"].reshape(-1))
    s.set_parameters_dict(copy.deepcopy(sc["params"]), device=DEV)
    per = sc.get("per", {})
    if "E" in per:
        s.mpm_model.E = T(per["E"])
        s.mpm_model.nu = T(per["nu"])
        s.mpm_state.particle_material = T(per["material"])
        s.reset_densities_and_update_masses(T(per["density"]))
    s.finalize_mu_lam(device=DEV)
    s.import_particle_v_from_torch(T(sc["v"]))
    if "C" in sc:
        s.import_particle_C_from_torch(T(sc["C"]))
    if "F_trial" in sc:
        s.mpm_state.particle_F_trial = T(sc["F_trial"])
    return s


def _setup_oracle(sc, precision):
    o = _Oracle(sc, precision)
    t = torch.from_numpy
    o.load_initial_data_from_torch(t(sc["x"]), t(sc["vol"]), t(sc["cov"]) if "cov" in sc else None, n_grid=sc["n_grid"],
                                   grid_lim=sc["grid_lim"])
    if sc.get("ucov"):
        o.mpm_model.update_cov_with_F = True
        o.o.set("COV", sc["cov"])
    o.set_parameters_dict(copy.deepcopy(sc["params"]))
    per = sc.get("per", {})
    if "E" in per:
        o.o.set("E", per["E"]); o.o.set("NU", per["nu"]); o.o.set("MATERIAL", per["material"]); o.o.set("DENSITY", per["density"])
        o.o.compute_mass()
    o.finalize_mu_lam()
    o.o.set("V", sc["v"])
    if "C" in sc:
        o.o.set("C", sc["C"])
    if "F_trial" in sc:
        o.o.set("F_TRIAL", sc["F_trial"])
    return o


_EXPORT = {"x": ("X", "export_particle_x_to_torch"), "v": ("V", "export_particle_v_to_torch"), "F": ("F", "export_particle_F_to_torch"),
           "cov": ("COV", "export_particle_cov_to_torch"), "R": ("R", "export_particle_R_to_torch")}


class Rollout:
    """One scenario on several back ends in lockstep: 'cuda' (the shim), 'f32' and 'f64' (the oracle)."""

    def __init__(self, sc, sides=("cuda", "f32", "f64"), stream=None):
        self.sc, self.n = sc, sc["n"]
        self.stream = stream
        self.sides = {}
        for k in sides:
            self.sides[k] = self._cuda(lambda: _setup_cuda(sc)) if k == "cuda" else _setup_oracle(sc, k)
        self.rec = {k: [] for k in sides}          # [(label, field, array)]
        self.clock = {k: [] for k in sides}
        self.mask_diff = {"box": 0, "cyl": 0}
        for method, kw in sc["bcs"]:
            self.do(("bc", method, kw))

    def _cuda(self, fn):
        if self.stream is None:
            return fn()
        with torch.cuda.stream(self.stream):
            return fn()

    def run(self, script):
        for op in script:
            self.do(op)
        return self

    def do(self, op):
        kind = op[0]
        masks = None                               # selections of the first back end, for the others
        for name, x in self.sides.items():
            if name == "cuda":
                self._cuda(lambda: self._do_cuda(x, op))
                if kind == "bc":
                    masks = self._new_masks
                continue
            if kind == "step":
                x.o.step(op[1], op[2])
            elif kind == "export":
                fid = _EXPORT[op[1]][0]
                a = x.o.get(fid) if fid in ("X", "V", "F") else getattr(x, _EXPORT[op[1]][1])().numpy()
                self.rec[name].append((op[1], fid, np.asarray(a, dtype=np.float64).reshape(self.n, -1)))
            elif kind == "fields":
                for fid in op[1]:
                    self.rec[name].append(("fields", fid, np.asarray(x.o.get(fid), dtype=np.float64).reshape(self.n, -1)))
            elif kind == "mutate":
                a = torch.from_numpy(x.o.get(op[1]).astype(np.float32 if x.precision == "f32" else np.float64))
                op[2](a)
                x.o.set(op[1], a.numpy())
            elif kind == "rebind":
                a = torch.from_numpy(x.o.get(op[1]).astype(np.float32))
                x.o.set(op[1], op[2](a).numpy())
                x.finalize_mu_lam()
            elif kind == "bc":
                k0 = len(x.masks)
                own = x.add(op[1], op[2], masks)
                if masks is None:
                    masks = list(x.masks[k0:])
                elif x.precision == "f32":
                    for (sel, mine), theirs in zip(own, masks):
                        self.mask_diff[sel] = max(self.mask_diff[sel], int((mine != np.asarray(theirs)).sum()))
            elif kind == "params":
                x.set_parameters_dict(copy.deepcopy(op[1]))
            elif kind == "time":
                x.o.time = op[1]
            else:
                raise ValueError(op)
            if kind == "step":
                self.clock[name].append(x.time)

    def _do_cuda(self, s, op):
        kind = op[0]
        if kind == "step":
            if op[1] == 1:
                s.p2g2p(0, op[2])
            else:
                s.p2g2p_n(op[1], op[2])
            self.clock["cuda"].append(s.time)
        elif kind == "export":
            fid, meth = _EXPORT[op[1]]
            a = getattr(s, meth)()
            self.rec["cuda"].append((op[1], fid, a.detach().cpu().numpy().astype(np.float64).reshape(self.n, -1)))
        elif kind == "fields":
            for fid in op[1]:
                self.rec["cuda"].append(("fields", fid, s._t[fid].detach().cpu().numpy().astype(np.float64).reshape(self.n, -1)))
        elif kind == "mutate":
            t = s.export_particle_v_to_torch() if op[1] == "V" else s._t[op[1]]
            op[2](t)
        elif kind == "rebind":
            setattr(s.mpm_model, {"E": "E", "NU": "nu"}[op[1]], op[2](s._t[op[1]].clone()).contiguous())
            s.finalize_mu_lam()
        elif kind == "bc":
            k0 = len(s._masks)
            getattr(s, op[1])(**copy.deepcopy(op[2]))
            self._new_masks = [m.cpu().numpy() for m in s._masks[k0:]]
        elif kind == "params":
            s.set_parameters_dict(copy.deepcopy(op[1]))
        elif kind == "time":
            s.time = op[1]
        else:
            raise ValueError(op)

    # ---- judging
    def compare(self, a, b):
        """max |a - b| per field over every recorded point (the two records must have the same labels)."""
        ra, rb = self.rec[a], self.rec[b]
        assert [(l, f) for l, f, _ in ra] == [(l, f) for l, f, _ in rb]
        out = {}
        for (_, fid, x), (_, _, y) in zip(ra, rb):
            assert np.isfinite(x).all(), (a, fid)
            out[fid] = max(out.get(fid, 0.0), float(np.abs(x - y).max()))
        return out

    def drift_pairs(self):
        """(drift vs fp64, fp32-vs-fp64 floor) of the positions at every recorded point."""
        out = []
        for (_, fid, c), (_, _, p32), (_, _, p64) in zip(self.rec["cuda"], self.rec["f32"], self.rec["f64"]):
            if fid == "X":
                out.append((float(np.abs(c - p64).max()), float(np.abs(p32 - p64).max())))
        return out


def judge(ro, tag, family, moving=None):
    """Asserts the CUDA run against the oracle (see the module docstring) and records a table row."""
    moving = ro.sc.get("moving", False) if moving is None else moving
    err = ro.compare("cuda", "f32")
    for k, c in enumerate(ro.clock["cuda"]):
        assert abs(c - ro.clock["f32"][k]) < 1e-12 and ro.clock["f32"][k] == ro.clock["f64"][k], (tag, k, c, ro.clock["f32"][k])
    assert ro.mask_diff["box"] == 0 and ro.mask_diff["cyl"] <= 2, (tag, ro.mask_diff)
    pairs = ro.drift_pairs()
    drift = max(d for d, _ in pairs)
    floor = max(f for _, f in pairs)
    row = f"{tag:<44s} " + " ".join(f"{k}={v:.1e}" for k, v in sorted(err.items())) + f" | drift64={drift:.1e} floor={floor:.1e}"
    print("[rollout]", row)
    tol = _TOL[family]
    for fid, e in err.items():
        assert e < tol[fid], f"{tag}: {fid} vs fp32 oracle {e:.2e} > {tol[fid]:.0e}"
    if not moving:
        for d, f in pairs:
            assert d < 20 * f + 1e-6, f"{tag}: drift vs fp64 {d:.2e} > 20 x floor {f:.2e} + 1e-6"
    return err


# ------------------------------------------------------------------------------------------------ scripts
CHOPS = {"single": [1] * 240, "whole": [240], "irregular": [1, 2, 3, 4, 5, 7, 49, 50, 51, 1, 3, 64]}
_CHOP_EXPORTS = {3: ("x",), 6: ("cov",), 9: ("v", "R")}            # after these chunks of the irregular chopping
_FINAL = [("export", "x"), ("export", "v"), ("export", "F"), ("export", "cov"), ("export", "R"), ("fields", ("F_TRIAL", "C"))]


def chop_script(chunks, dt=DT):
    out = []
    for i, k in enumerate(chunks):
        out.append(("step", k, dt))
        if chunks is CHOPS["irregular"]:
            out += [("export", e) for e in _CHOP_EXPORTS.get(i, ())]
    return out + _FINAL


def frame_script(step_per_frame, dts, frames=6):
    """scene_driver's frame loop: every frame exports x, cov and R, then steps `step_per_frame` substeps."""
    out = []
    for f in range(frames):
        out += [("export", "x"), ("export", "cov"), ("export", "R"), ("step", step_per_frame, dts[f % len(dts)])]
    return out + _FINAL


# Frame-loop schedules. mpm_step_fused chops a call of n substeps into chunks of
#   count = min(remaining, kFusedGraphSteps, max(1, kResortEvery - steps_since_sort))
# (kFusedGraphSteps = 50, kResortEvery = 100; the gather after an export restarts steps_since_sort at 0), replays chunks of
# at least kMinGraphSteps = 4 from a graph keyed (count, clock parity, dt), and flips the parity after every odd chunk.
# 333 substeps per frame: 50,50 | 50,50 | 50,50 | 33 -> keys (50, p, dt), (33, p, dt), and the odd 33 flips p for the
# next frame; 400: 50 x 8 -> (50, p, dt) only. With dt alternating DT, DT/2, DT/2, DT, DT, DT/2 over six 333-substep
# frames (parity 0,1,0,1,0,1) the keys are (50|33, 0, DT), (50|33, 1, DT/2), (50|33, 0, DT/2), (50|33, 1, DT), ...: 8
# distinct keys for kGraphSlots = 4 slots, so slots are evicted and keys captured again. test_graph_key_model checks this
# derivation against the constants in mpm.cu.
FRAME_RUNS = {"333": (333, [DT]), "400": (400, [DT]), "333-two-dt": (333, [DT, DT / 2, DT / 2, DT, DT, DT / 2])}


def _constants():
    src = open(os.path.join(ROOT, "pixie_b200", "csrc", "mpm.cu")).read()
    get = lambda name: int(re.search(rf"\b{name}\s*=\s*(\d+)", src).group(1))   # noqa: E731
    return dict(steps=get("kFusedGraphSteps"), min=get("kMinGraphSteps"), resort=get("kResortEvery"), slots=get("kGraphSlots"))


def graph_keys(calls, k=None):
    """The (count, parity, dt) keys, in order, of `calls` = [(n_substeps, dt)] each after a write-back, as mpm_step_fused
    produces them; returns (keys, captures) where captures counts graph builds under round-robin replacement."""
    k = k or _constants()
    par, keys = 0, []
    for n, dt in calls:
        since = done = 0
        while done < n:
            if since >= k["resort"]:
                since = 0
            c = min(n - done, k["steps"], max(1, k["resort"] - since))
            if c >= k["min"]:
                keys.append((c, par, dt))
            par ^= c & 1
            done += c
            since += c
    slots, nxt, captures = [None] * k["slots"], 0, 0
    for key in keys:
        if key not in slots:
            slots[nxt] = key
            nxt = (nxt + 1) % k["slots"]
            captures += 1
    return keys, captures


def _mid_script(change):
    """150 substeps as two calls of 75 (chunks 50, 25 | 25, re-sort, 50: graphs of three keys are cached), then `change`,
    then 120 more substeps."""
    pre = [("step", 75, DT), ("step", 75, DT)]
    post = [("step", 61, DT), ("export", "x"), ("step", 59, DT)]
    ops = {
        "bcs": [("bc", "set_velocity_on_cuboid", dict(point=[1.2, 1.0, 0.93], size=[0.1, 0.3, 0.05], velocity=[0.0, 0.0, 1.0])),
                ("bc", "add_surface_collider", dict(point=[1.0, 1.0, 0.71], normal=[0.0, 0.3, 1.0], surface="slip", friction=0.2)),
                ("bc", "add_impulse_on_particles", dict(force=[0.0, 2.0, 0.5], dt=DT, point=[0.9, 0.9, 1.0], size=[0.2, 0.2, 0.2],
                                                        num_dt=80, start_time=150 * DT))],
        "params": [("params", {"g": [0.0, -3.0, -9.8], "grid_v_damping_scale": 0.999})],
        "dt": [],
        "time": [("time", 40 * DT)],
        "inplace": [("mutate", "V", lambda t: t.mul_(0.5)), ("mutate", "F_TRIAL", lambda t: t[:, 0, 0].mul_(1.01))],
        "rebind": [("rebind", "E", lambda t: t * 1.5)],
        "plastic": [("fields", ("X", "YIELD", "MU", "LAM"))],
    }[change]
    if change == "dt":
        post = [("step", 61, DT / 2), ("export", "x"), ("step", 59, DT)]
    return pre + ops + post + _FINAL + [("fields", ("YIELD", "MU", "LAM"))]


MID = ("bcs", "params", "dt", "time", "inplace", "rebind", "plastic")


def _mid_scene(change, n=5000):
    """The synthetic scene with its BC windows. "plastic": metal and snow only, with a yield stress of 1 Pa, no hardening
    and a softening of 1e5, so that every snow particle's yield stress falls through 0 within the first substeps it yields
    and the return map sets its mu and lam to 0 on the device (mpm_utils.py:165-171); metal keeps its mu and lam."""
    if change != "plastic":
        return _synthetic(n=n, materials=(0, 1, 5))
    sc = _synthetic(n=n, materials=(1, 5))
    sc["params"].update(yield_stress=1.0, hardening=0, softening=1e5)
    return sc
PBC = ("3", "4", "5", "8", "release1", "release2")


def _pbc_scene(case):
    sc = _synthetic(materials=(0,), seed=7, bcs="bbox")
    if case.startswith("release"):
        rel = ("release_particles_sequentially", dict(normal=[0, 0, 1], start_position=0.7, end_position=1.3, num_layers=50,
                                                        start_time=0.0, end_time=0.01))
        sc["bcs"] += [rel] * int(case[-1]) + _particle_bcs(1)
    else:
        sc["bcs"] += _particle_bcs(int(case))
    return sc


_PBC_SCRIPT = [("step", 97, DT), ("export", "x"), ("step", 103, DT)] + _FINAL


# ------------------------------------------------------------------------------------------------ CPU part
def _oracle_pair(sc):
    """The fp32 and fp64 oracles in lockstep (masks of the fp32 one handed to the fp64 one)."""
    return Rollout(sc, sides=("f32", "f64"))


@pytest.mark.parametrize("scene", ["paths", "mixed"])
@pytest.mark.parametrize("chop", ["whole", "irregular"])
def test_harness_chopped_on_oracles(scene, chop):
    sc = _stretched_paths() if scene == "paths" else _stretched_mixed()
    ro = _oracle_pair(sc).run(chop_script(CHOPS[chop]))
    assert len(ro.clock["f32"]) == len(CHOPS[chop]) and ro.clock["f32"] == ro.clock["f64"]
    assert abs(ro.clock["f32"][-1] - 240 * DT) < 1e-12
    err = ro.compare("f32", "f64")
    print(scene, chop, err)
    assert err["X"] < 1e-4


@pytest.mark.parametrize("case", ["5", "release2"])
def test_harness_particle_bcs_on_oracles(case):
    ro = _oracle_pair(_pbc_scene(case)).run(_PBC_SCRIPT)
    err = ro.compare("f32", "f64")
    assert err["X"] < 1e-4 and len(ro.sides["f32"].masks) == len(ro.sides["f64"].masks)
    assert all((a == b).all() for a, b in zip(ro.sides["f32"].masks, ro.sides["f64"].masks))


@pytest.mark.parametrize("change", MID)
def test_harness_mid_rollout_on_oracles(change):
    ro = _oracle_pair(_mid_scene(change, n=1500)).run(_mid_script(change))
    assert ro.clock["f32"] == ro.clock["f64"]
    want = 150 * DT + 120 * DT if change not in ("dt", "time") else None
    if change == "time":
        want = 40 * DT + 120 * DT
    if want is not None:
        assert abs(ro.clock["f32"][-1] - want) < 1e-12
    err = ro.compare("f32", "f64")
    assert err["X"] < 1e-2                     # a moving cuboid: fp32 and fp64 part where its faces cross nodes


def test_oracle_chopping_is_bitwise():
    """The oracle's serial scatter is deterministic: any chopping of 240 substeps gives the same bits."""
    for sc in (_stretched_paths(), _stretched_mixed()):
        whole = _setup_oracle(sc, "f32")
        chopped = _setup_oracle(sc, "f32")
        for o in (whole, chopped):
            for method, kw in sc["bcs"]:
                o.add(method, kw)
        whole.o.step(240, DT)
        for k in CHOPS["irregular"]:
            chopped.o.step(k, DT)
        assert whole.time == chopped.time
        for fid in ("X", "V", "C", "F_TRIAL", "F", "COV", "YIELD"):
            assert np.array_equal(whole.o.get(fid), chopped.o.get(fid)), fid


def test_graph_key_model():
    k = _constants()
    assert (k["steps"], k["min"], k["resort"], k["slots"]) == (50, 4, 100, 4)
    keys, captures = graph_keys([(333, DT)] * 6, k)
    assert set(keys) == {(50, 0, DT), (33, 0, DT), (50, 1, DT), (33, 1, DT)} and captures == 4
    keys, _ = graph_keys([(400, DT)] * 6, k)
    assert set(keys) == {(50, 0, DT)}
    spf, dts = FRAME_RUNS["333-two-dt"]
    keys, captures = graph_keys([(spf, dts[f]) for f in range(6)], k)
    assert len(set(keys)) >= 5 and len(set(keys)) > k["slots"] and captures > len(set(keys))
    # the mid-rollout scripts cache graphs of several keys before their change
    keys, _ = graph_keys([(75, DT)], k)
    assert keys == [(50, 0, DT), (25, 0, DT)]


# ------------------------------------------------------------------------------------------------ GPU part
@pytest.mark.gpu
@pytest.mark.parametrize("scene", ["paths", "mixed", "synthetic"])
def test_chopping_invariance(built_lib, cuda_dev, scene):
    """240 substeps as 240 x p2g2p, one p2g2p_n(240) and an irregular chopping with exports between chunks: every run
    matches the oracle, and the runs match each other."""
    make = {"paths": _stretched_paths, "mixed": _stretched_mixed, "synthetic": _synthetic}[scene]
    finals = {}
    for chop, chunks in CHOPS.items():
        ro = Rollout(make()).run(chop_script(chunks))
        judge(ro, f"chop/{scene}/{chop}", "chop")
        finals[chop] = [a for _, f, a in ro.rec["cuda"] if f == "X"][-1]
    for a in finals:
        for b in finals:
            assert np.abs(finals[a] - finals[b]).max() < _TOL["chop"]["X"], (scene, a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("run", list(FRAME_RUNS) + ["paths-cov"])
def test_frame_loop(built_lib, cuda_dev, run):
    """scene_driver's loop (export x, cov, R; p2g2p_n(step_per_frame)) for 6 frames; "paths-cov" evolves cov with F on the
    device, so it goes through the write-back and the gather every frame."""
    if run == "paths-cov":
        sc, spf, dts = _stretched_paths(bbox_end=999.0), 333, [DT]
    else:
        (spf, dts), sc = FRAME_RUNS[run], _synthetic()
    ro = Rollout(sc).run(frame_script(spf, dts))
    judge(ro, f"frames/{run}", "frame")


@pytest.mark.gpu
@pytest.mark.parametrize("case", PBC)
def test_particle_bc_table(built_lib, cuda_dev, case):
    """3 and 4 particle BCs travel in the kernel parameters, 5 and 8 (and 51 / 101) are walked in the device table."""
    ro = Rollout(_pbc_scene(case)).run(_PBC_SCRIPT)
    judge(ro, f"pbc/{case}", "pbc")


@pytest.mark.gpu
@pytest.mark.parametrize("change", MID)
def test_mid_rollout_change(built_lib, cuda_dev, change):
    """A change after 150 substeps, with graphs of several keys cached, is seen by every later substep."""
    sc = _mid_scene(change)
    ro = Rollout(sc).run(_mid_script(change))
    judge(ro, f"mid/{change}", "mid")
    if change == "plastic":
        # the state written back after 150 substeps (before the change point's re-gather) already holds what the device
        # changed: negative yield stresses and mu = lam = 0 of the snow particles, the metal's mu and lam untouched
        got = {f: a[:, 0] for _, f, a in ro.rec["cuda"][:4]}
        snow = sc["per"]["material"] == 5
        print(f"[rollout] mid/plastic after 150: snow {int(snow.sum())}, mu = 0: {int((got['MU'] == 0).sum())}, "
              f"lam = 0: {int((got['LAM'] == 0).sum())}, min yield {got['YIELD'].min():.1f}")
        assert (got["YIELD"][snow] < 0).mean() > 0.9, "snow must soften through 0 on the device"
        assert (got["MU"][snow] == 0).mean() > 0.9 and (got["LAM"][snow] == 0).mean() > 0.9
        assert (got["MU"][~snow] > 0).all() and (got["LAM"][~snow] > 0).all()


@pytest.mark.gpu
def test_side_stream_ordering(built_lib, cuda_dev):
    """The chopped script on a torch side stream matches the default-stream run; on a 100k-particle scene, add_bc,
    set_parameters_dict and the clock right after p2g2p_n(400) see the queued substeps."""
    side = torch.cuda.Stream()
    base = Rollout(_stretched_mixed()).run(chop_script(CHOPS["irregular"]))
    ro = Rollout(_stretched_mixed(), stream=side).run(chop_script(CHOPS["irregular"]))
    torch.cuda.synchronize()
    judge(ro, "stream/mixed/irregular", "chop")
    assert ro.clock["cuda"] == base.clock["cuda"]
    xa = [a for _, f, a in ro.rec["cuda"] if f == "X"][-1]
    xb = [a for _, f, a in base.rec["cuda"] if f == "X"][-1]
    assert np.abs(xa - xb).max() < _TOL["chop"]["X"]

    sc = _synthetic(n=100_000, ng=64, materials=(0,), seed=0, bcs="bbox")
    results = []
    for stream in (None, side):
        ctx = torch.cuda.stream(stream) if stream is not None else torch.cuda.stream(torch.cuda.current_stream())
        s = _setup_cuda(sc)
        torch.cuda.synchronize()
        with ctx:
            s.p2g2p_n(400, DT)
            t1 = s.time
            s.add_impulse_on_particles(force=[0.0, 0.0, 5.0], dt=DT, point=[1.0, 1.0, 1.0], size=[0.2, 0.2, 0.2], num_dt=50, start_time=t1)
            s.add_surface_collider(point=[1.0, 1.0, 0.7], normal=[0.0, 0.0, 1.0], surface="slip", friction=0.1)
            s.set_parameters_dict({"g": [0.0, 1.0, -9.8], "grid_v_damping_scale": 0.999})
            t2 = s.time
            s.p2g2p_n(100, DT)
            t3 = s.time
            x = s.export_particle_x_to_torch().cpu().numpy().astype(np.float64)
            mask = s._masks[-1].cpu().numpy()
        results.append((t1, t2, t3, x, mask))
    (a1, a2, a3, xa, ma), (b1, b2, b3, xb, mb) = results
    print(f"[rollout] stream/100k clocks {a1!r} {a3!r} | {b1!r} {b3!r}; x diff {np.abs(xa - xb).max():.1e}")
    assert (a1, a2, a3) == (b1, b2, b3) and abs(a1 - 400 * DT) < 1e-12 and abs(a3 - 500 * DT) < 1e-12
    assert (ma == mb).all() and ma.sum() > 100
    assert np.abs(xa - xb).max() < _TOL["chop"]["X"]


@pytest.mark.gpu
def test_slab_grid_bcs_across_faces(built_lib, cuda_dev):
    """3 slabs on one device through the phase API, with a reset=1 cuboid moving across the interface at plane 6, a slip
    plane and a cut plane: each rank applies them on its owned and overlap planes and advances the cuboid itself. Same
    trajectory as the undivided CUDA run and as the fp32 oracle, and each of the three BCs changes that trajectory."""
    from pixie_b200.mpm_slab import FusedSlabBackend, LocalSlabCluster, SlabRank
    from slab_backends import load_scene, make_scene
    import test_slab_mpm as T

    N, G, LIM, SDT = T.N, T.G, T.LIM, T.DT
    # faces off the grid nodes, and an end time between two clock ticks: the reset zeroes the grid while
    # time < end_time + 15 dt, and a bound that lands on a tick is decided by the last bit of that sum (the kernel's fused
    # multiply-add and the oracle's separate product and sum round it differently)
    bcs = [("set_velocity_on_cuboid", dict(point=[0.37, 0.5, 0.45], size=[0.05, 0.12, 0.047], velocity=[0.5, 0.0, 0.0],
                                           start_time=0.0, end_time=21.5 * SDT, reset=1)),
           ("add_surface_collider", dict(point=[0.5, 0.5, 0.28], normal=[0.0, 0.0, 1.0], surface="slip", friction=0.3)),
           ("add_surface_collider", dict(point=[0.5, 0.34, 0.5], normal=[0.0, 1.0, 0.0], surface="cut", friction=0.0))]
    fields = make_scene(N, G, LIM)
    bounds = [(0, 6), (6, 10), (10, 16)]
    base = (fields["X"][:, 0].astype(np.float32) * np.float32(G / LIM) - np.float32(0.5)).astype(np.int32)

    def finish(s):
        from pixie_b200 import _lib
        lib = _lib.load()
        _lib.check(lib.pixie_mpm_compute_mass(s._handle, s._stream()))
        _lib.check(lib.pixie_mpm_compute_mu_lam(s._handle, s._stream()))
        s.add_bounding_box()
        for method, kw in bcs:
            getattr(s, method)(**kw)

    ranks = []
    for r in range(3):
        lo = -10 ** 9 if r == 0 else bounds[r][0]
        hi = 10 ** 9 if r == 2 else bounds[r][1]
        idx = np.where((base >= lo) & (base < hi))[0]
        s = T._cuda_solver(fields, idx, N)
        finish(s)
        ranks.append(SlabRank(FusedSlabBackend(s, len(idx)), r, 3, slack=1, migrate_every=2, ids=torch.from_numpy(idx.astype(np.int64)),
                              bounds=bounds[r]))
    whole = T._cuda_solver(fields, np.arange(N), N)
    finish(whole)
    steps = 60
    whole.p2g2p_n(steps, SDT)
    x_whole = whole._t["X"].view(N, 3).cpu().numpy().astype(np.float64)
    before = [r.b.active for r in ranks]
    cl = LocalSlabCluster(ranks)
    for _ in range(steps):
        cl.substep(SDT)
    torch.cuda.synchronize()
    for r in ranks:
        r.check_device_error()
    assert sum(r.b.active for r in ranks) == N and [r.b.active for r in ranks] != before
    x_slab = cl.gather("X").numpy().reshape(N, 3)
    oracle_bcs = [dict(kind=R.BC_CUBOID, point=[0.37, 0.5, 0.45], size=[0.05, 0.12, 0.047], velocity=[0.5, 0.0, 0.0],
                       end_time=21.5 * SDT, reset=1),
                  dict(kind=R.BC_SURFACE, point=[0.5, 0.5, 0.28], normal=[0.0, 0.0, 1.0], friction=0.3, surface_type=1),
                  dict(kind=R.BC_SURFACE, point=[0.5, 0.34, 0.5], normal=[0.0, 1.0, 0.0], surface_type=11)]

    def oracle(drop=None):
        ref = R.MpmRef(N, G, LIM, "f32")
        load_scene(ref, fields)
        for k, bc in enumerate(oracle_bcs):
            if k != drop:
                ref.add_bc(**bc)
        ref.step(steps, SDT)
        return np.asarray(ref.get("X"))

    x_ref = oracle()
    # every one of the three BCs changes the trajectory (the cuboid spans the slab interface at x = 6 / 16 = 0.375)
    effect = [np.abs(x_ref - oracle(drop=k)).max() for k in range(len(oracle_bcs))]
    d_sw, d_sr, d_wr = np.abs(x_slab - x_whole).max(), np.abs(x_slab - x_ref).max(), np.abs(x_whole - x_ref).max()
    print(f"[rollout] slabs: slab-whole {d_sw:.1e} slab-f32 {d_sr:.1e} whole-f32 {d_wr:.1e}; "
          f"effect of cuboid / slip / cut {effect[0]:.1e} / {effect[1]:.1e} / {effect[2]:.1e}")
    assert min(effect) > 1e-2, effect          # measured 0.13 / 0.031 / 0.064 on the fp32 oracle
    # measured 1.2e-7 to 1.8e-7 (float atomics)
    assert d_sw < 2e-6 and d_sr < 2e-6 and d_wr < 2e-6
