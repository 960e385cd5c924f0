"""Back ends for tests/golden/mpm_scenarios.replay (TEST INFRASTRUCTURE).

OracleSolver puts oracle/mpm_ref.c behind the call surface of the reference's `MPM_Simulator_WARP`
(mpm_solver_warp.py:47-1210) — only the host-side bookkeeping of that class is restated here (key handling of
`set_parameters_dict`, normal normalisation, rotation axes); every kernel runs in the C oracle.  The golden fixture
(tests/golden/mpm_golden.npz, produced by executing the reference's own source) is what pins both.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from oracle import mpm_ref as R

NAME_TO_ID = {"jelly": 0, "metal": 1, "sand": 2, "snow": 5, "stationary": 6, "elastic": 0, "rigid": 6}
_STATE = {"particle_x": "X", "particle_v": "V", "particle_C": "C", "particle_F": "F", "particle_F_trial": "F_TRIAL",
          "particle_stress": "STRESS", "particle_cov": "COV", "particle_mass": "MASS", "particle_density": "DENSITY",
          "particle_material": "MATERIAL", "particle_init_cov": "INIT_COV", "particle_vol": "VOL"}
_MODEL = {"E": "E", "nu": "NU", "mu": "MU", "lam": "LAM", "yield_stress": "YIELD", "bulk": "BULK"}


class _Model:
    pass


class OracleSolver:
    def __init__(self, n_particles, n_grid=100, grid_lim=1.0, device="cpu", precision="f32"):
        self.precision = precision
        self.initialize(n_particles, n_grid, grid_lim)

    def initialize(self, n, n_grid, grid_lim):
        self.n_particles = n
        self.o = R.MpmRef(n, n_grid, grid_lim, self.precision)
        self.mpm_model = _Model()
        self.mpm_model.update_cov_with_F = False
        self.mpm_model.material = 0
        self.masks = []

    @property
    def time(self):
        return self.o.time

    def load_initial_data_from_torch(self, x, vol, cov=None, n_grid=100, grid_lim=1.0, device="cpu"):
        self.initialize(x.shape[0], n_grid, grid_lim)
        self.o.set("X", x.numpy())
        self.o.set("VOL", vol.numpy())
        if cov is not None:
            self.o.set("INIT_COV", cov.numpy())

    def set_parameters_dict(self, kw, device="cpu"):
        o, n = self.o, self.n_particles
        if "material" in kw:
            self.mpm_model.material = NAME_TO_ID.get(kw["material"], -1)
            if self.mpm_model.material == -1:
                raise TypeError("Undefined material type")
        o.set("MATERIAL", np.full(n, self.mpm_model.material))
        for key, f in (("E", "E"), ("nu", "NU"), ("bulk_modulus", "BULK"), ("yield_stress", "YIELD")):
            if key in kw:
                o.set(f, np.full(n, np.float32(kw[key])))
        p = {}
        for key in ("hardening", "xi", "rpic_damping", "plastic_viscosity", "softening", "grid_v_damping_scale"):
            if key in kw:
                p[key] = float(kw[key])
        if "friction_angle" in kw:
            p["alpha"] = R.friction_alpha(kw["friction_angle"])
        if "g" in kw:
            p["g"] = tuple(kw["g"])
        p["update_cov_with_F"] = int(bool(self.mpm_model.update_cov_with_F))
        o.set_params(**p)
        if "spawn_offset" in kw:
            x = o.get("X").astype(np.float32)
            x += np.asarray(kw["spawn_offset"], dtype=np.float32)      # in-place float32 add on the exported view
            o.set("X", x)
        if "density" in kw:
            o.set("DENSITY", np.full(n, np.float32(kw["density"])))
            o.compute_mass()
        if "additional_material_params" in kw:
            for b in kw["additional_material_params"]:
                mat = NAME_TO_ID.get(b["material"], -1) if isinstance(b["material"], str) else b["material"]
                o.apply_additional_params(b["point"], b["size"], b["E"], b["nu"], b["density"], mat)
            o.compute_mass()

    def finalize_mu_lam(self, device="cpu"):
        self.o.compute_mu_lam()

    def import_particle_v_from_torch(self, t, clone=True, device="cpu"):
        self.o.set("V", t.numpy())

    def import_particle_C_from_torch(self, t, clone=True, device="cpu"):
        self.o.set("C", t.numpy())

    def p2g2p(self, step, dt, device="cpu"):
        self.o.step(1, dt)

    # ---- boundary conditions (host-side argument handling of mpm_solver_warp.py:749-1179)
    def add_bounding_box(self, start_time=0.0, end_time=999.0):
        self.o.add_bc(R.BC_BBOX, start_time=start_time, end_time=end_time)

    def set_velocity_on_cuboid(self, point, size, velocity, start_time=0.0, end_time=999.0, reset=0):
        self.o.add_bc(R.BC_CUBOID, point=point, size=size, velocity=velocity, start_time=start_time, end_time=end_time, reset=reset)

    def add_surface_collider(self, point, normal, surface="sticky", friction=0.0, start_time=0.0, end_time=999.0):
        scale = np.float32(1.0) / np.sqrt(np.float32(sum(x ** 2 for x in normal)))
        normal = [scale * x for x in normal]
        st = {"sticky": 0, "slip": 1, "cut": 11}.get(surface, 2)
        self.o.add_bc(R.BC_SURFACE, point=point, normal=normal, friction=friction, surface_type=st, start_time=start_time, end_time=end_time)

    def add_impulse_on_particles(self, force, dt, point=(1, 1, 1), size=(1, 1, 1), num_dt=1, start_time=0.0, device="cpu"):
        mask = self.o.select_box(point, size)
        self.masks.append(mask)
        self.o.add_bc(R.BC_IMPULSE, velocity=force, start_time=start_time, end_time=start_time + dt * num_dt, mask=mask)

    def enforce_particle_velocity_translation(self, point, size, velocity, start_time, end_time, device="cpu"):
        mask = self.o.select_box(point, size)
        self.masks.append(mask)
        self.o.add_bc(R.BC_VTRANS, velocity=velocity, start_time=start_time, end_time=end_time, mask=mask)

    def enforce_particle_velocity_rotation(self, point, normal, half_height_and_radius, rotation_scale, translation_scale,
                                           start_time, end_time, device="cpu"):
        f32 = np.float32
        scale = f32(1.0) / np.sqrt(f32(normal[0] ** 2 + normal[1] ** 2 + normal[2] ** 2))
        n = np.asarray([scale * x for x in normal], dtype=f32)
        h1 = np.asarray([1.0, 1.0, 1.0], dtype=f32)
        if abs(float(np.dot(n, h1))) < 0.01:
            h1 = np.asarray([0.72, 0.37, -0.67], dtype=f32)
        h1 = (h1 - np.dot(h1, n) * n).astype(f32)
        h1 = (h1 * (f32(1.0) / np.sqrt(np.dot(h1, h1)))).astype(f32)
        h2 = np.cross(h1, n).astype(f32)
        mask = self.o.select_cylinder(point, n, half_height_and_radius[0], half_height_and_radius[1])
        self.masks.append(mask)
        self.o.add_bc(R.BC_VROT, point=point, normal=list(n), h1=list(h1), h2=list(h2), hhr=half_height_and_radius,
                      rotation_scale=rotation_scale, translation_scale=translation_scale, start_time=start_time,
                      end_time=end_time, mask=mask)

    def export_particle_R_to_torch(self, device="cpu"):
        self.o.compute_R_from_F()
        return torch.from_numpy(self.o.get("R").reshape(-1, 9))

    def export_particle_cov_to_torch(self, device="cpu"):
        if not self.mpm_model.update_cov_with_F:
            self.o.compute_cov_from_F()
        return torch.from_numpy(self.o.get("COV").reshape(-1))


class OracleBackend:
    device = "cpu"

    def tensor(self, a):
        return torch.from_numpy(np.ascontiguousarray(a))

    def to_numpy(self, t):
        return t.numpy()

    def set_state(self, s, name, arr):
        s.o.set(_STATE[name], arr)

    def get_state(self, s, names):
        return {k: s.o.get(_STATE[k]) for k in names}

    def get_model(self, s, names):
        return {k: s.o.get(_MODEL[k]) for k in names}

    def get_masks(self, s):
        return list(s.masks)

    def get_grid(self, s):
        m, vi, vo = s.o.grid()
        return {"grid_m": m, "grid_v_in": vi, "grid_v_out": vo}


class _DeviceArray:
    """A device pointer presented through __cuda_array_interface__, so torch can copy from it."""

    def __init__(self, ptr, shape, typestr="<f4"):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (int(ptr), False), "version": 3,
                                         "strides": None}


def device_grid_v(s) -> np.ndarray:
    """Grid velocities of the last substep, [n, n, n, 3], read through pixie_mpm_grid_ptrs. Only nodes inside the
    particles' node box are swept; the solver leaves the others as they were."""
    import ctypes as C
    from pixie_b200 import _lib
    mv, v = C.c_void_p(), C.c_void_p()
    _lib.check(_lib.load().pixie_mpm_grid_ptrs(s._handle, C.byref(mv), C.byref(v)))
    n = int(s.mpm_model.n_grid)
    torch.cuda.synchronize()
    g = torch.as_tensor(_DeviceArray(v.value, (n, n, n, 4)), device=s._device).clone()
    return g[..., :3].cpu().numpy()


class CudaBackend:
    """pixie_b200.mpm_solver_warp.MPM_Simulator_WARP on cuda:0 (every call goes through the C ABI)."""
    device = "cuda:0"

    def tensor(self, a):
        return torch.from_numpy(np.ascontiguousarray(a)).to(self.device)

    def to_numpy(self, t):
        return t.detach().cpu().numpy()

    def set_state(self, s, name, arr):
        setattr(s.mpm_state, name, self.tensor(arr))

    def get_state(self, s, names):
        return {k: getattr(s.mpm_state, k).numpy() for k in names}

    def get_model(self, s, names):
        return {k: getattr(s.mpm_model, k).numpy() for k in names}

    def get_masks(self, s):
        return [m.cpu().numpy() for m in s._masks]

    def get_grid(self, s):
        return {"grid_v_out": device_grid_v(s)}
