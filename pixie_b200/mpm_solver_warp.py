"""Drop-in `MPM_Simulator_WARP` (third_party/PhysGaussian/mpm_solver_warp/mpm_solver_warp.py:47-1210).

Same constructor, methods, argument meaning and error behaviour as the reference class, as used by
gs_simulation.py:68-72, 483-489, 528-531, 591-594, 634, material_field.py:232-363, 452, 531 and
utils/decode_param.py:277-396 — but every kernel runs in libpixie_b200.so (hand-written sm_90a CUDA,
pixie_b200/csrc/mpm.cu) instead of Warp, substeps are replayed from a CUDA graph with the simulation
clock on the device, and nothing synchronises with the host inside the substep loop.

State arrays are torch tensors owned here (Warp arrays alias torch memory in the reference too,
warp_utils.py:244-324); `mpm_state.<field>` / `mpm_model.<field>` return thin views with `.numpy()`,
and assigning a torch tensor (e.g. `solver.mpm_model.E = tensor`, gs_simulation.py:528) rebinds the
device pointer.

Additions (not in the reference): `p2g2p_n(n_substeps, dt)` runs many substeps in one call.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Optional

import numpy as np
import torch

from . import _lib

MATERIAL_ID_TO_NAME = {0: "jelly", 1: "metal", 2: "sand", 3: "visplas", 4: "fluid", 5: "snow", 6: "stationary"}
EXCLUDED_MATERIAL_NAMES = ["visplas", "fluid"]
NAME_TO_MATERIAL_ID = {name: i for i, name in MATERIAL_ID_TO_NAME.items() if name not in EXCLUDED_MATERIAL_NAMES}
NAME_TO_MATERIAL_ID.update({"elastic": 0, "rigid": 6})
#: boundary conditions one solver can hold (kMaxBC in csrc/mpm.cu); grid and particle BCs share the table
MAX_BCS = 256


# ---- host-side BC parameter arithmetic of the reference (:749-1210). The reference evaluates it at Python scope, where
# `wp.sqrt` / `wp.abs` / `wp.length` return float32 scalars and wp.vec3 arithmetic is float32 with one rounding per
# operation; a Python float combined with a float32 scalar is rounded to float32 first. The BC kernels then compare node
# and particle coordinates against these values, so they are reproduced bit for bit (tests/test_mpm_bc_edges.py).
_f32 = np.float32


def _dot_f32(a, b):
    """wp.dot of two float32 3-vectors: ((a0 b0 + a1 b1) + a2 b2), one rounding per operation."""
    acc = _f32(0.0)
    for k in range(3):
        acc = _f32(acc + _f32(_f32(a[k]) * _f32(b[k])))
    return acc


def _unit_normal_f32(normal):
    """`normal_scale = 1.0 / wp.sqrt(float(...))`, then `normal_scale * x` per component (:760-761, :1092-1095)."""
    scale = _f32(_f32(1.0) / _f32(np.sqrt(_f32(float(normal[0] ** 2 + normal[1] ** 2 + normal[2] ** 2)))))
    return np.array([_f32(scale * _f32(x)) for x in normal], dtype=_f32)


def collider_normal(normal) -> np.ndarray:
    """The float32 normal `add_surface_collider` stores (:758-768)."""
    return _unit_normal_f32(normal)


def rotation_axes(normal):
    """(normal, horizontal_axis_1, horizontal_axis_2) as `enforce_particle_velocity_rotation` stores them (:1092-1117)."""
    n = _unit_normal_f32(normal)
    h1 = np.array([1.0, 1.0, 1.0], dtype=_f32)
    if _f32(np.abs(_dot_f32(n, h1))) < _f32(0.01):
        h1 = np.array([0.72, 0.37, -0.67], dtype=_f32)
    d = _dot_f32(h1, n)
    h1 = np.array([_f32(h1[k] - _f32(d * n[k])) for k in range(3)], dtype=_f32)
    inv = _f32(_f32(1.0) / _f32(np.sqrt(_dot_f32(h1, h1))))
    h1 = np.array([_f32(h1[k] * inv) for k in range(3)], dtype=_f32)
    h2 = np.cross(h1, n).astype(_f32)              # float32 a_i b_j - a_j b_i, like wp.cross
    return n, h1, h2


def release_layers(normal, start_position, end_position, end_time, num_layers=50):
    """(point, size, end_time) of the translation modifiers `release_particles_sequentially` registers (:1185-1210):
    the layer half-length is float32 (`wp.abs(...) / num_layers`), the end times are Python floats."""
    point, size, axis = [0, 0, 0], [0, 0, 0], -1
    for i in range(3):
        if normal[i] == 0:
            point[i] = 1
            size[i] = 1
        else:
            axis = i
            point[i] = end_position
    half_length_portion = _f32(_f32(np.abs(_f32(start_position - end_position))) / _f32(num_layers))
    end_time_portion = end_time / num_layers
    out = []
    for i in range(num_layers):
        size[axis] = _f32(half_length_portion * _f32(num_layers - i))
        out.append((list(point), list(size), end_time_portion * (i + 1)))
    return out


def impulse_end_time(start_time, dt, num_dt):
    """`start_time + dt * num_dt` in Python floats, stored as float32 (:993-994)."""
    return start_time + dt * num_dt


def get_material_name(material_id):
    """Reference quirk kept: despite its name this maps a material NAME to its id (:29-39)."""
    return NAME_TO_MATERIAL_ID.get(material_id, -1)


def get_material_id(material_name):
    return NAME_TO_MATERIAL_ID.get(material_name, -1)


class _Arr:
    """Stand-in for a wp.array aliasing a torch tensor: `.numpy()`, `.shape`, `.tensor`."""

    def __init__(self, t: torch.Tensor):
        self.tensor = t

    def numpy(self):
        return self.tensor.detach().cpu().numpy()

    @property
    def shape(self):
        return tuple(self.tensor.shape)

    def __len__(self):
        return self.tensor.shape[0]


def _as_tensor(v) -> torch.Tensor:
    return v.tensor if isinstance(v, _Arr) else v


class _Struct:
    """MPMStateStruct / MPMModelStruct facade: array attributes are bound to C-ABI field ids."""

    def __init__(self, solver, fields):
        object.__setattr__(self, "_solver", solver)
        object.__setattr__(self, "_fields", fields)      # attr name -> (field id name, dtype, width)

    def __getattr__(self, name):
        fields = object.__getattribute__(self, "_fields")
        if name in fields:
            return _Arr(object.__getattribute__(self, "_solver")._t[fields[name][0]])
        raise AttributeError(name)

    def __setattr__(self, name, value):
        fields = object.__getattribute__(self, "_fields")
        if name in fields:
            fid, dtype, width = fields[name]
            solver = object.__getattribute__(self, "_solver")
            t = _as_tensor(value)
            if t.dtype != dtype or not t.is_cuda or not t.is_contiguous():
                raise RuntimeError("Error aliasing Torch tensor: must be a contiguous CUDA float32/int32 tensor")
            if t.numel() != solver.n_particles * width:
                raise RuntimeError(f"{name}: expected {solver.n_particles * width} elements, got {t.numel()}")
            solver._bind(fid, t)
        else:
            object.__setattr__(self, name, value)


_STATE_FIELDS = {
    "particle_x": ("X", torch.float32, 3), "particle_v": ("V", torch.float32, 3),
    "particle_F": ("F", torch.float32, 9), "particle_F_trial": ("F_TRIAL", torch.float32, 9),
    "particle_C": ("C", torch.float32, 9), "particle_stress": ("STRESS", torch.float32, 9),
    "particle_R": ("R", torch.float32, 9), "particle_cov": ("COV", torch.float32, 6),
    "particle_init_cov": ("INIT_COV", torch.float32, 6), "particle_vol": ("VOL", torch.float32, 1),
    "particle_mass": ("MASS", torch.float32, 1), "particle_density": ("DENSITY", torch.float32, 1),
    "particle_material": ("MATERIAL", torch.int32, 1), "particle_selection": ("SELECTION", torch.int32, 1),
}
_MODEL_FIELDS = {
    "E": ("E", torch.float32, 1), "nu": ("NU", torch.float32, 1), "mu": ("MU", torch.float32, 1),
    "lam": ("LAM", torch.float32, 1), "bulk": ("BULK", torch.float32, 1), "yield_stress": ("YIELD", torch.float32, 1),
}
_SHAPES = {"X": (3,), "V": (3,), "F": (3, 3), "F_TRIAL": (3, 3), "C": (3, 3), "STRESS": (3, 3), "R": (3, 3)}


class MPM_Simulator_WARP:
    def __init__(self, n_particles, n_grid=100, grid_lim=1.0, device="cuda:0"):
        self._handle = None
        self._masks = []
        self.initialize(n_particles, n_grid, grid_lim, device=device)
        self.time_profile = {}

    # ------------------------------------------------------------------------------ life cycle
    def initialize(self, n_particles, n_grid=100, grid_lim=1.0, device="cuda:0"):
        """mpm_solver_warp.py:52-180."""
        lib = _lib.require_device()
        self._destroy()
        self.n_particles = int(n_particles)
        self._device = torch.device(device)
        n = self.n_particles
        dev = self._device
        self._tensors = {}
        with torch.cuda.device(dev):
            h = C.c_void_p()
            _lib.check(lib.pixie_mpm_create(n, int(n_grid), float(grid_lim), C.byref(h)))
            self._handle = h
        self.mpm_state = _Struct(self, _STATE_FIELDS)
        self.mpm_model = _Struct(self, _MODEL_FIELDS)
        for fields in (_STATE_FIELDS, _MODEL_FIELDS):
            for _, (fid, dtype, width) in fields.items():
                shape = ((n,) + _SHAPES[fid]) if fid in _SHAPES else (n * width,)
                # particle_x is wp.empty in the reference; zeros is a harmless superset
                self._bind(fid, torch.zeros(shape, dtype=dtype, device=dev))
        m = self.mpm_model
        m.grid_lim, m.n_grid = grid_lim, int(n_grid)
        m.grid_dim_x = m.grid_dim_y = m.grid_dim_z = int(n_grid)
        m.dx, m.inv_dx = m.grid_lim / m.n_grid, float(m.n_grid / m.grid_lim)
        m.update_cov_with_F = False
        m.material = 0
        m.plastic_viscosity = 0.0
        m.softening = 0.1
        m.friction_angle = 25.0
        sin_phi = math.sin(m.friction_angle / 180.0 * 3.14159265)
        m.alpha = math.sqrt(2.0 / 3.0) * 2.0 * sin_phi / (3.0 - sin_phi)
        m.gravitational_accelaration = (0.0, 0.0, 0.0)
        m.rpic_damping = 0.0
        m.grid_v_damping_scale = 1.1
        m.hardening = 0.0
        m.xi = 0.0
        self._masks = []
        self.n_bcs = 0                                   # entries used in the native BC table (MAX_BCS)
        self.grid_postprocess, self.collider_params, self.modify_bc = [], [], []
        self.pre_p2g_operations, self.impulse_params = [], []
        self.particle_velocity_modifiers, self.particle_velocity_modifier_params = [], []
        self._push_params()
        self.time = 0.0

    def _destroy(self):
        if getattr(self, "_handle", None) is not None:
            _lib.load().pixie_mpm_destroy(self._handle)
            self._handle = None

    def __del__(self):
        try:
            self._destroy()
        except Exception:
            pass

    def _stream(self):
        return _lib.stream(self._device)

    def _fence(self, write_back=True):
        """Puts a call that changes bindings, parameters, boundary conditions or the clock behind the substeps queued on
        the caller's stream. Those C calls copy on the legacy default stream, which does not wait for torch's side
        streams (they are non-blocking), so pending results are written back on the caller's stream and the host waits
        for it first. Once the write-back is done, binding a field or setting parameters only changes host state, so the
        wait is stricter than those two need; it is kept as the one rule for every such call, which only runs at set-up
        and between rollouts."""
        if write_back:
            _lib.check(_lib.load().pixie_mpm_sync(self._handle, self._stream()))
        torch.cuda.current_stream(self._device).synchronize()

    @property
    def _t(self):
        """Particle / model tensors in the caller's order. The default native path keeps a cell-sorted private copy
        between steps, so any access goes through a sync (results written back, and — since the caller may now modify
        the tensors in place like the reference's zero-copy exports allow — re-read at the next step). The sync is a
        no-op when nothing was stepped since the last access, and on the direct (slab) path."""
        if self._handle is not None:
            _lib.check(_lib.load().pixie_mpm_sync(self._handle, self._stream()))
        return self._tensors

    def _bind(self, fid: str, t: torch.Tensor):
        self._tensors[fid] = t
        self._fence()
        _lib.check(_lib.load().pixie_mpm_bind(self._handle, _lib.FIELDS[fid], _lib.ptr(t)))

    def _push_params(self):
        m = self.mpm_model
        p = _lib.MpmParams()
        p.n_grid, p.grid_lim = int(m.n_grid), float(m.grid_lim)
        for i in range(3):
            p.gravity[i] = float(m.gravitational_accelaration[i])
        p.rpic_damping, p.grid_v_damping_scale = float(m.rpic_damping), float(m.grid_v_damping_scale)
        p.alpha, p.hardening, p.xi = float(m.alpha), float(m.hardening), float(m.xi)
        p.plastic_viscosity, p.softening = float(m.plastic_viscosity), float(m.softening)
        p.update_cov_with_F = int(bool(m.update_cov_with_F))
        self._fence()
        _lib.check(_lib.load().pixie_mpm_set_params(self._handle, C.byref(p)))

    # simulation clock: `self.time` is a host float in the reference (:167, :637); here it lives on the
    # device so that substeps need no host round trip.
    @property
    def time(self) -> float:
        t = C.c_double()
        self._fence(write_back=False)
        _lib.check(_lib.load().pixie_mpm_get_time(self._handle, C.byref(t)))
        return t.value

    @time.setter
    def time(self, value: float):
        self._fence(write_back=False)
        _lib.check(_lib.load().pixie_mpm_set_time(self._handle, float(value)))

    # ------------------------------------------------------------------------------ loading
    def load_initial_data_from_torch(self, tensor_x, tensor_volume, tensor_cov=None, n_grid=100, grid_lim=1.0,
                                     device="cuda:0"):
        """mpm_solver_warp.py:234-281."""
        self.dim, self.n_particles = tensor_x.shape[1], tensor_x.shape[0]
        assert tensor_x.shape[0] == tensor_volume.shape[0]
        self.initialize(self.n_particles, n_grid, grid_lim, device=device)
        self.import_particle_x_from_torch(tensor_x, device=device)
        self._t["VOL"].copy_(tensor_volume.detach().reshape(-1).to(self._device, torch.float32))
        if tensor_cov is not None:
            self._t["INIT_COV"].copy_(tensor_cov.detach().reshape(-1).to(self._device, torch.float32))
            if self.mpm_model.update_cov_with_F:
                self._bind("COV", self._t["INIT_COV"])
        self._t["V"].zero_()
        ft = self._t["F_TRIAL"]
        ft.zero_()
        ft[:, 0, 0] = 1.0
        ft[:, 1, 1] = 1.0
        ft[:, 2, 2] = 1.0
        print("Particles initialized from torch data.")
        print("Total particles: ", self.n_particles)

    def set_parameters(self, device="cuda:0", **kwargs):
        self.set_parameters_dict(kwargs, device)

    def set_parameters_dict(self, kwargs={}, device="cuda:0"):
        """mpm_solver_warp.py:287-463 (same key handling and order)."""
        lib = _lib.load()
        m = self.mpm_model
        if "material" in kwargs:
            print("Setting material to ", kwargs["material"])
            m.material = get_material_name(kwargs["material"])
            print("Material ID: ", m.material)
            if m.material == -1:
                raise TypeError("Undefined material type")
        if "grid_lim" in kwargs:
            m.grid_lim = kwargs["grid_lim"]
        if "n_grid" in kwargs:
            m.n_grid = int(kwargs["n_grid"])
        m.grid_dim_x = m.grid_dim_y = m.grid_dim_z = m.n_grid
        m.dx, m.inv_dx = m.grid_lim / m.n_grid, float(m.n_grid / m.grid_lim)
        # the reference re-creates particle_material on every call and fills it with model.material
        self._bind("MATERIAL", torch.full((self.n_particles,), int(m.material), dtype=torch.int32, device=self._device))
        if "E" in kwargs:
            self._t["E"].fill_(float(kwargs["E"]))
        if "nu" in kwargs:
            self._t["NU"].fill_(float(kwargs["nu"]))
        if "bulk_modulus" in kwargs:
            self._t["BULK"].fill_(float(kwargs["bulk_modulus"]))
        if "yield_stress" in kwargs:
            self._t["YIELD"].fill_(float(kwargs["yield_stress"]))
        if "hardening" in kwargs:
            m.hardening = kwargs["hardening"]
        if "xi" in kwargs:
            m.xi = kwargs["xi"]
        if "friction_angle" in kwargs:
            m.friction_angle = kwargs["friction_angle"]
            sin_phi = math.sin(m.friction_angle / 180.0 * 3.14159265)
            m.alpha = math.sqrt(2.0 / 3.0) * 2.0 * sin_phi / (3.0 - sin_phi)
        if "g" in kwargs:
            m.gravitational_accelaration = (kwargs["g"][0], kwargs["g"][1], kwargs["g"][2])
        if "spawn_offset" in kwargs:
            offset = kwargs["spawn_offset"]
            pos_torch = self.export_particle_x_to_torch()
            pos_torch[:, 0] += offset[0]
            pos_torch[:, 1] += offset[1]
            pos_torch[:, 2] += offset[2]
            self.import_particle_x_from_torch(pos_torch)
        if "rpic_damping" in kwargs:
            m.rpic_damping = kwargs["rpic_damping"]
        if "plastic_viscosity" in kwargs:
            m.plastic_viscosity = kwargs["plastic_viscosity"]
        if "softening" in kwargs:
            m.softening = kwargs["softening"]
        if "grid_v_damping_scale" in kwargs:
            m.grid_v_damping_scale = kwargs["grid_v_damping_scale"]
        self._push_params()
        if "density" in kwargs:
            self._t["DENSITY"].fill_(float(kwargs["density"]))
            _lib.check(lib.pixie_mpm_compute_mass(self._handle, self._stream()))
        if "additional_material_params" in kwargs:
            boxes = []
            for params in kwargs["additional_material_params"]:
                if isinstance(params["material"], str):
                    params["material"] = get_material_name(params["material"])
                boxes.append(list(params["point"]) + list(params["size"]) +
                             [params["E"], params["nu"], params["density"], float(params["material"])])
            if boxes:
                b = np.ascontiguousarray(np.asarray(boxes, dtype=np.float32))
                # one launch for the whole list (the reference launches once per box, i.e. O(N^2)
                # threads when material_field.py:343-363 passes one box per particle)
                _lib.check(lib.pixie_mpm_apply_additional_params(self._handle, C.c_void_p(b.ctypes.data), len(boxes),
                                                                 self._stream()))
            _lib.check(lib.pixie_mpm_compute_mass(self._handle, self._stream()))

    def _apply_additional_params_boxes(self, boxes: torch.Tensor):
        """`additional_material_params` as an (n_boxes, 10) float32 device tensor (point, size, E, nu, density, material):
        the per-box `apply_additional_params` launches (:436-452) + the mass update (:454-463) without a Python dict per box."""
        lib = _lib.load()
        b = boxes.detach().to(self._device, torch.float32).contiguous()
        _lib.check(lib.pixie_mpm_apply_additional_params(self._handle, _lib.ptr(b), int(b.shape[0]), self._stream()))
        _lib.check(lib.pixie_mpm_compute_mass(self._handle, self._stream()))

    def finalize_mu_lam(self, device="cuda:0"):
        _lib.check(_lib.load().pixie_mpm_compute_mu_lam(self._handle, self._stream()))

    def finalize_mu_lam_bulk(self, device="cuda:0"):
        lib = _lib.load()
        _lib.check(lib.pixie_mpm_compute_mu_lam(self._handle, self._stream()))
        _lib.check(lib.pixie_mpm_compute_bulk(self._handle, self._stream()))

    # ------------------------------------------------------------------------------ stepping
    def p2g2p(self, step, dt, device="cuda:0"):
        """One explicit substep (mpm_solver_warp.py:514-637). `step` is unused, as in the reference."""
        _lib.check(_lib.load().pixie_mpm_step(self._handle, 1, float(dt), self._stream()))

    def p2g2p_n(self, n_substeps, dt):
        """`n_substeps` x p2g2p without returning to Python (CUDA-graph replay)."""
        _lib.check(_lib.load().pixie_mpm_step(self._handle, int(n_substeps), float(dt), self._stream()))

    def launch_count(self) -> int:
        """Kernels of libpixie_b200 launched for this solver so far (graph replays count their nodes)."""
        return int(_lib.load().pixie_mpm_launch_count(self._handle))

    def reset_densities_and_update_masses(self, all_particle_densities, device="cuda:0"):
        d = all_particle_densities.clone().detach().to(self._device, torch.float32).contiguous()
        self._bind("DENSITY", d)
        _lib.check(_lib.load().pixie_mpm_compute_mass(self._handle, self._stream()))

    # ------------------------------------------------------------------------------ import / export
    def _import(self, fid, tensor, clone, shape):
        if tensor is None:
            return
        if clone:
            tensor = tensor.clone().detach()
        tensor = torch.reshape(tensor, shape)
        if tensor.dtype != torch.float32 or not tensor.is_contiguous():
            raise RuntimeError("Error aliasing Torch tensor to Warp array. Torch tensor must be float32 or int32 type")
        self._bind(fid, tensor.to(self._device))

    def import_particle_x_from_torch(self, tensor_x, clone=True, device="cuda:0"):
        self._import("X", tensor_x, clone, (-1, 3))

    def import_particle_v_from_torch(self, tensor_v, clone=True, device="cuda:0"):
        self._import("V", tensor_v, clone, (-1, 3))

    def import_particle_F_from_torch(self, tensor_F, clone=True, device="cuda:0"):
        self._import("F", tensor_F, clone, (-1, 3, 3))

    def import_particle_C_from_torch(self, tensor_C, clone=True, device="cuda:0"):
        self._import("C", tensor_C, clone, (-1, 3, 3))

    def export_particle_x_to_torch(self):
        return self._t["X"]

    def export_particle_stress_to_torch(self):
        return self._t["STRESS"]

    def export_particle_v_to_torch(self):
        return self._t["V"]

    def export_particle_F_to_torch(self):
        return self._t["F"].reshape(-1, 9)

    def export_particle_R_to_torch(self, device="cuda:0"):
        _lib.check(_lib.load().pixie_mpm_compute_R_from_F(self._handle, self._stream()))
        return self._t["R"].reshape(-1, 9)

    def export_particle_C_to_torch(self):
        return self._t["C"].reshape(-1, 9)

    def export_particle_cov_to_torch(self, device="cuda:0"):
        if not self.mpm_model.update_cov_with_F:
            _lib.check(_lib.load().pixie_mpm_compute_cov_from_F(self._handle, self._stream()))
        return self._t["COV"]

    def print_time_profile(self):
        print("MPM Time profile:")
        for key, value in self.time_profile.items():
            print(key, sum(value))

    # ------------------------------------------------------------------------------ boundary conditions
    def _add_bc(self, kind, mask: Optional[torch.Tensor] = None, **kw):
        bc = _lib.MpmBC()
        bc.kind = kind
        for name in ("point", "normal", "size", "velocity", "horizontal_axis_1", "horizontal_axis_2"):
            v = kw.get(name, (0.0, 0.0, 0.0))
            for i in range(3):
                getattr(bc, name)[i] = float(v[i])
        hhr = kw.get("half_height_and_radius", (0.0, 0.0))
        bc.half_height_and_radius[0], bc.half_height_and_radius[1] = float(hhr[0]), float(hhr[1])
        bc.start_time, bc.end_time = float(kw.get("start_time", 0.0)), float(kw.get("end_time", 999.0))
        bc.friction = float(kw.get("friction", 0.0))
        bc.surface_type, bc.reset = int(kw.get("surface_type", 0)), int(kw.get("reset", 0))
        bc.rotation_scale = float(kw.get("rotation_scale", 0.0))
        bc.translation_scale = float(kw.get("translation_scale", 0.0))
        if mask is not None:
            self._masks.append(mask)
            bc.mask_dev = _lib.ptr(mask)
        self._fence()
        _lib.check(_lib.load().pixie_mpm_add_bc(self._handle, C.byref(bc)))
        self.n_bcs += 1
        return bc

    def _select_box(self, point, size) -> torch.Tensor:
        mask = torch.zeros(self.n_particles, dtype=torch.int32, device=self._device)
        p3, s3 = (C.c_float * 3)(*[float(v) for v in point]), (C.c_float * 3)(*[float(v) for v in size])
        _lib.check(_lib.load().pixie_mpm_select_box(self._handle, p3, s3, _lib.ptr(mask), self._stream()))
        return mask

    def add_surface_collider(self, point, normal, surface="sticky", friction=0.0, start_time=0.0, end_time=999.0):
        """:749-843."""
        point = list(point)
        normal = collider_normal(normal)
        if surface == "sticky" and friction != 0:
            raise ValueError("friction must be 0 on sticky surfaces.")
        surface_type = {"sticky": 0, "slip": 1, "cut": 11}.get(surface, 2)
        bc = self._add_bc(_lib.BC_SURFACE_COLLIDER, point=point, normal=normal, friction=friction,
                          surface_type=surface_type, start_time=start_time, end_time=end_time)
        self.collider_params.append(bc)
        self.grid_postprocess.append("surface_collider")
        self.modify_bc.append(None)

    def set_velocity_on_cuboid(self, point, size, velocity, start_time=0.0, end_time=999.0, reset=0):
        """:852-908 (the moving-box update `modify` runs on the device)."""
        bc = self._add_bc(_lib.BC_CUBOID, point=list(point), size=size, velocity=velocity, start_time=start_time,
                          end_time=end_time, reset=reset)
        self.collider_params.append(bc)
        self.grid_postprocess.append("cuboid")
        self.modify_bc.append("device")

    def add_bounding_box(self, start_time=0.0, end_time=999.0):
        """:910-977."""
        bc = self._add_bc(_lib.BC_BOUNDING_BOX, start_time=start_time, end_time=end_time)
        self.collider_params.append(bc)
        self.grid_postprocess.append("bounding_box")
        self.modify_bc.append(None)

    def add_impulse_on_particles(self, force, dt, point=[1, 1, 1], size=[1, 1, 1], num_dt=1, start_time=0.0,
                                 device="cuda:0"):
        """:982-1029."""
        mask = self._select_box(point, size)
        bc = self._add_bc(_lib.BC_IMPULSE, mask=mask, point=point, size=size, velocity=force, start_time=start_time,
                          end_time=impulse_end_time(start_time, dt, num_dt))
        self.impulse_params.append(bc)
        self.pre_p2g_operations.append("apply_force")

    def enforce_particle_velocity_translation(self, point, size, velocity, start_time, end_time, device="cuda:0"):
        """:1031-1075."""
        mask = self._select_box(point, size)
        bc = self._add_bc(_lib.BC_VELOCITY_TRANSLATION, mask=mask, point=point, size=size, velocity=velocity,
                          start_time=start_time, end_time=end_time)
        self.particle_velocity_modifier_params.append(bc)
        self.particle_velocity_modifiers.append("translation")

    def enforce_particle_velocity_rotation(self, point, normal, half_height_and_radius, rotation_scale,
                                           translation_scale, start_time, end_time, device="cuda:0"):
        """:1080-1179 (axes built in fp32 like the wp.vec3 arithmetic of the reference)."""
        n, h1, h2 = rotation_axes(normal)
        mask = torch.zeros(self.n_particles, dtype=torch.int32, device=self._device)
        p3, n3 = (C.c_float * 3)(*[float(v) for v in point]), (C.c_float * 3)(*[float(v) for v in n])
        _lib.check(_lib.load().pixie_mpm_select_cylinder(self._handle, p3, n3, float(half_height_and_radius[0]),
                                                         float(half_height_and_radius[1]), _lib.ptr(mask), self._stream()))
        bc = self._add_bc(_lib.BC_VELOCITY_ROTATION, mask=mask, point=point, normal=n, horizontal_axis_1=h1,
                          horizontal_axis_2=h2, half_height_and_radius=half_height_and_radius,
                          rotation_scale=rotation_scale, translation_scale=translation_scale, start_time=start_time,
                          end_time=end_time)
        self.particle_velocity_modifier_params.append(bc)
        self.particle_velocity_modifiers.append("rotation")

    def release_particles_sequentially(self, normal, start_position, end_position, num_layers, start_time, end_time):
        """:1183-1210 (num_layers is overridden to 50, as in the reference)."""
        for point, size, layer_end in release_layers(normal, start_position, end_position, end_time):
            self.enforce_particle_velocity_translation(point=point, size=size, velocity=[0, 0, 0],
                                                       start_time=start_time, end_time=layer_end)
