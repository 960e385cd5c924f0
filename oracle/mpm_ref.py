"""ORACLE (test infrastructure, not product code): ctypes wrapper of oracle/mpm_ref.c, the CPU
restatement of the reference's Warp MPM kernels, pinned to the reference's own source through
tests/golden/mpm_golden.npz (see the header of mpm_ref.c and tests/test_mpm_golden.py).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs import this.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from typing import Dict, Optional, Sequence

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_BUILD = os.path.join(_HERE, "_build")

FIELDS = dict(X=0, V=1, F=2, F_TRIAL=3, C=4, STRESS=5, R=6, COV=7, INIT_COV=8, VOL=9, MASS=10, DENSITY=11,
              E=12, NU=13, MU=14, LAM=15, BULK=16, YIELD=17, MATERIAL=18, SELECTION=19)
WIDTH = [3, 3, 9, 9, 9, 9, 9, 6, 6, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1]
BC_SURFACE, BC_CUBOID, BC_BBOX, BC_IMPULSE, BC_VTRANS, BC_VROT = range(6)

_libs: Dict[str, C.CDLL] = {}


def build():
    subprocess.check_call(["make", "-s", "-C", _HERE])


def _lib(precision: str) -> C.CDLL:
    if precision in _libs:
        return _libs[precision]
    path = os.path.join(_BUILD, f"libmpm_ref_{precision}.so")
    if not os.path.exists(path):
        build()
    lib = C.CDLL(path)
    D = C.POINTER(C.c_double)
    lib.mpmref_create.restype = C.c_void_p
    lib.mpmref_create.argtypes = [C.c_int, C.c_int, C.c_double]
    lib.mpmref_destroy.argtypes = [C.c_void_p]
    lib.mpmref_set.argtypes = [C.c_void_p, C.c_int, D]
    lib.mpmref_get.argtypes = [C.c_void_p, C.c_int, D]
    lib.mpmref_get_grid.argtypes = [C.c_void_p, D, D, D]
    lib.mpmref_set_params.argtypes = [C.c_void_p, D] + [C.c_double] * 7 + [C.c_int, C.c_int]
    lib.mpmref_set_time.argtypes = [C.c_void_p, C.c_double]
    lib.mpmref_get_time.restype = C.c_double
    lib.mpmref_get_time.argtypes = [C.c_void_p]
    lib.mpmref_add_bc.argtypes = [C.c_void_p, C.c_int, D, C.c_int, C.c_int, C.POINTER(C.c_int)]
    for f in ("mpmref_compute_mu_lam", "mpmref_compute_mass", "mpmref_compute_cov_from_F", "mpmref_compute_bulk",
              "mpmref_compute_R_from_F"):
        getattr(lib, f).argtypes = [C.c_void_p]
    lib.mpmref_svd3.argtypes = [D, D, D, D]
    lib.mpmref_apply_additional_params.argtypes = [C.c_void_p, D]
    lib.mpmref_select_box.argtypes = [C.c_void_p, D, D, C.POINTER(C.c_int)]
    lib.mpmref_select_cylinder.argtypes = [C.c_void_p, D, D, C.c_double, C.c_double, C.POINTER(C.c_int)]
    lib.mpmref_stress_of_F.argtypes = [C.c_void_p, C.c_int]
    lib.mpmref_stress_probe.argtypes = [C.c_void_p, C.c_int, D]
    lib.mpmref_step.argtypes = [C.c_void_p, C.c_int, C.c_double]
    lib.mpmref_num_threads.restype = C.c_int
    lib.mpmref_set_num_threads.argtypes = [C.c_int]
    lib.mpmref_set_active.argtypes = [C.c_void_p, C.c_int]
    lib.mpmref_scatter.argtypes = [C.c_void_p, C.c_double]
    lib.mpmref_finish.argtypes = [C.c_void_p, C.c_double, C.c_int, C.c_int]
    lib.mpmref_planes_get.argtypes = [C.c_void_p, C.c_int, C.c_int, D]
    lib.mpmref_planes_add.argtypes = [C.c_void_p, C.c_int, C.c_int, D]
    lib.mpmref_real_size.restype = C.c_int
    _libs[precision] = lib
    return lib


def _dp(a: np.ndarray):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def friction_alpha(friction_angle_deg: float) -> float:
    """mpm_solver_warp.py:84-86 / 390-393."""
    sin_phi = np.sin(friction_angle_deg / 180.0 * 3.14159265)
    return float(np.sqrt(2.0 / 3.0) * 2.0 * sin_phi / (3.0 - sin_phi))


def svd3(F: np.ndarray, precision: str = "f64"):
    lib = _lib(precision)
    F = np.ascontiguousarray(F, dtype=np.float64).reshape(9)
    U, s, V = np.zeros(9), np.zeros(3), np.zeros(9)
    lib.mpmref_svd3(_dp(F), _dp(U), _dp(s), _dp(V))
    return U.reshape(3, 3), s, V.reshape(3, 3)


class MpmRef:
    """One simulation in the oracle.  precision: 'f32' (the reference's arithmetic) or 'f64'."""

    def __init__(self, n: int, n_grid: int, grid_lim: float, precision: str = "f32"):
        self.lib = _lib(precision)
        self.n, self.n_grid, self.grid_lim, self.precision = n, n_grid, grid_lim, precision
        self.capacity = n
        self.h = C.c_void_p(self.lib.mpmref_create(n, n_grid, float(grid_lim)))
        self.params = dict(g=(0.0, 0.0, 0.0), rpic_damping=0.0, grid_v_damping_scale=1.1, alpha=friction_alpha(25.0),
                           hardening=0.0, xi=0.0, plastic_viscosity=0.0, softening=0.1, update_cov_with_F=0,
                           parallel_p2g=0)
        self._push_params()

    def __del__(self):
        try:
            self.lib.mpmref_destroy(self.h)
        except Exception:
            pass

    def _push_params(self):
        p = self.params
        g = np.asarray(p["g"], dtype=np.float64)
        self.lib.mpmref_set_params(self.h, _dp(g), p["rpic_damping"], p["grid_v_damping_scale"], p["alpha"], p["hardening"],
                                   p["xi"], p["plastic_viscosity"], p["softening"], int(p["update_cov_with_F"]),
                                   int(p["parallel_p2g"]))

    def set_params(self, **kw):
        self.params.update(kw)
        self._push_params()

    def set(self, field: str, data):
        a = np.ascontiguousarray(np.asarray(data, dtype=np.float64).reshape(-1))
        assert a.size == self.n * WIDTH[FIELDS[field]], (field, a.size)
        self.lib.mpmref_set(self.h, FIELDS[field], _dp(a))

    def get(self, field: str) -> np.ndarray:
        w = WIDTH[FIELDS[field]]
        out = np.zeros(self.n * w)
        self.lib.mpmref_get(self.h, FIELDS[field], _dp(out))
        if field in ("F", "F_TRIAL", "C", "STRESS", "R"):
            return out.reshape(self.n, 3, 3)
        return out.reshape(self.n, w) if w > 1 else out

    def grid(self):
        nodes = self.n_grid ** 3
        m, vi, vo = np.zeros(nodes), np.zeros(3 * nodes), np.zeros(3 * nodes)
        self.lib.mpmref_get_grid(self.h, _dp(m), _dp(vi), _dp(vo))
        g = self.n_grid
        return m.reshape(g, g, g), vi.reshape(g, g, g, 3), vo.reshape(g, g, g, 3)

    @property
    def time(self) -> float:
        return self.lib.mpmref_get_time(self.h)

    @time.setter
    def time(self, t: float):
        self.lib.mpmref_set_time(self.h, float(t))

    def add_bc(self, kind: int, point=(0, 0, 0), normal=(0, 0, 0), size=(0, 0, 0), velocity=(0, 0, 0), start_time=0.0,
               end_time=999.0, friction=0.0, surface_type=0, reset=0, h1=(0, 0, 0), h2=(0, 0, 0), hhr=(0, 0),
               rotation_scale=0.0, translation_scale=0.0, mask: Optional[np.ndarray] = None):
        vals = np.array(list(point) + list(normal) + list(size) + list(velocity) + [start_time, end_time, friction] +
                        list(h1) + list(h2) + list(hhr) + [rotation_scale, translation_scale], dtype=np.float64)
        assert vals.size == 25
        mp = None
        if mask is not None:
            mask = np.ascontiguousarray(mask, dtype=np.int32)
            mp = mask.ctypes.data_as(C.POINTER(C.c_int))
        self.lib.mpmref_add_bc(self.h, kind, _dp(vals), int(surface_type), int(reset), mp)

    def compute_mu_lam(self):
        self.lib.mpmref_compute_mu_lam(self.h)

    def compute_mass(self):
        self.lib.mpmref_compute_mass(self.h)

    def compute_cov_from_F(self):
        self.lib.mpmref_compute_cov_from_F(self.h)

    def compute_bulk(self):
        self.lib.mpmref_compute_bulk(self.h)

    def compute_R_from_F(self):
        self.lib.mpmref_compute_R_from_F(self.h)

    def apply_additional_params(self, point, size, E, nu, density, material):
        box = np.array(list(point) + list(size) + [E, nu, density, material], dtype=np.float64)
        self.lib.mpmref_apply_additional_params(self.h, _dp(box))

    def select_box(self, point, size) -> np.ndarray:
        mask = np.zeros(self.n, dtype=np.int32)
        self.lib.mpmref_select_box(self.h, _dp(np.asarray(point, dtype=np.float64)), _dp(np.asarray(size, dtype=np.float64)),
                                   mask.ctypes.data_as(C.POINTER(C.c_int)))
        return mask

    def select_cylinder(self, point, normal, half_height, radius) -> np.ndarray:
        mask = np.zeros(self.n, dtype=np.int32)
        self.lib.mpmref_select_cylinder(self.h, _dp(np.asarray(point, dtype=np.float64)), _dp(np.asarray(normal, dtype=np.float64)),
                                        float(half_height), float(radius), mask.ctypes.data_as(C.POINTER(C.c_int)))
        return mask

    def stress_of(self, p: int):
        self.lib.mpmref_stress_of_F(self.h, p)

    def stress_probe(self, flip: int = 0) -> np.ndarray:
        """`stress_of` for every particle, with the branch decisions whose bits are set in `flip` inverted (bit 0: the
        plastic branch of a return map; bit 1: sand's cone-tip projection / the damage map's mu = lam = 0). Returns each
        particle's two decision margins (relative distance from the boundary, > 0 = taken; inf = not reached)."""
        out = np.zeros(2 * self.n)
        self.lib.mpmref_stress_probe(self.h, int(flip), _dp(out))
        return out.reshape(self.n, 2)

    def step(self, n_substeps: int, dt: float):
        self.lib.mpmref_step(self.h, int(n_substeps), float(dt))

    # ---- split substep (test double of pixie_mpm_substep_scatter / _finish for the slab-decomposition tests)
    def set_active(self, n_active: int):
        assert 0 <= n_active <= self.capacity
        self.n = int(n_active)
        self.lib.mpmref_set_active(self.h, self.n)

    def scatter(self, dt: float):
        self.lib.mpmref_scatter(self.h, float(dt))

    def finish(self, dt: float, x_begin: int, x_end: int):
        self.lib.mpmref_finish(self.h, float(dt), int(x_begin), int(x_end))

    def planes_get(self, a: int, b: int) -> np.ndarray:
        out = np.zeros((b - a) * self.n_grid * self.n_grid * 4)
        self.lib.mpmref_planes_get(self.h, int(a), int(b), _dp(out))
        return out

    def planes_add(self, a: int, b: int, data: np.ndarray):
        d = np.ascontiguousarray(data, dtype=np.float64).reshape(-1)
        assert d.size == (b - a) * self.n_grid * self.n_grid * 4
        self.lib.mpmref_planes_add(self.h, int(a), int(b), _dp(d))

    def num_threads(self) -> int:
        return int(self.lib.mpmref_num_threads())

    def set_num_threads(self, n: int):
        """OpenMP threads of the oracle (torchrun exports OMP_NUM_THREADS=1, which would starve a CPU baseline)."""
        self.lib.mpmref_set_num_threads(int(n))


# Synthetic scene of BASELINE config 3: shared with bench.py, lives with the other synthetic-data
# generators (pure numpy, no solver arithmetic).
import sys as _sys
_sys.path.insert(0, os.path.dirname(_HERE))
from pixie_b200.synthetic import synthetic_scene  # noqa: E402,F401
