"""ctypes binding of include/pixie_b200.h.  This is the stub a maintainer of the reference would add
(see INTEGRATION.md); everything else in the package is written against it."""
from __future__ import annotations

import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libpixie_b200.so")
ABI_VERSION = 3


class PixieError(RuntimeError):
    pass


class UNetConfig(C.Structure):
    _fields_ = [
        ("feature_channels", C.c_int), ("cond_dim", C.c_int), ("model_channels", C.c_int),
        ("num_res_blocks", C.c_int), ("n_levels", C.c_int), ("channel_mult", C.c_int * 8),
        ("grid_size", C.c_int), ("out_channels", C.c_int), ("max_batch", C.c_int), ("precision", C.c_int),
    ]


class MpmParams(C.Structure):
    _fields_ = [
        ("n_grid", C.c_int), ("grid_lim", C.c_float), ("gravity", C.c_float * 3),
        ("rpic_damping", C.c_float), ("grid_v_damping_scale", C.c_float), ("alpha", C.c_float),
        ("hardening", C.c_float), ("xi", C.c_float), ("plastic_viscosity", C.c_float),
        ("softening", C.c_float), ("update_cov_with_F", C.c_int),
    ]


class MpmBC(C.Structure):
    _fields_ = [
        ("kind", C.c_int), ("point", C.c_float * 3), ("normal", C.c_float * 3), ("size", C.c_float * 3),
        ("velocity", C.c_float * 3), ("start_time", C.c_float), ("end_time", C.c_float),
        ("friction", C.c_float), ("surface_type", C.c_int), ("reset", C.c_int),
        ("horizontal_axis_1", C.c_float * 3), ("horizontal_axis_2", C.c_float * 3),
        ("half_height_and_radius", C.c_float * 2), ("rotation_scale", C.c_float),
        ("translation_scale", C.c_float), ("mask_dev", C.c_void_p),
    ]


# enum pixie_mpm_field
FIELDS = dict(X=0, V=1, F=2, F_TRIAL=3, C=4, STRESS=5, R=6, COV=7, INIT_COV=8, VOL=9, MASS=10, DENSITY=11,
              E=12, NU=13, MU=14, LAM=15, BULK=16, YIELD=17, MATERIAL=18, SELECTION=19)
# enum pixie_mpm_bc_kind
BC_SURFACE_COLLIDER, BC_CUBOID, BC_BOUNDING_BOX, BC_IMPULSE, BC_VELOCITY_TRANSLATION, BC_VELOCITY_ROTATION = range(6)

# name -> (restype, argtypes); every symbol the header declares
_SIGNATURES = {
    "pixie_last_error": (C.c_char_p, []),
    "pixie_abi_version": (C.c_int, []),
    "pixie_device_ok": (C.c_int, []),
    "pixie_unet_create": (C.c_int, [C.POINTER(UNetConfig), C.POINTER(C.c_void_p)]),
    "pixie_unet_set_tensor": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.POINTER(C.c_int64), C.c_int]),
    "pixie_unet_finalize": (C.c_int, [C.c_void_p]),
    "pixie_unet_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "pixie_unet_forward_ncdhw": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "pixie_unet_forward_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "pixie_unet_profile": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_int), C.POINTER(C.c_double), C.c_int]),
    "pixie_pack_predictions": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_void_p]),
    "pixie_unet_launch_count": (C.c_int, [C.c_void_p]),
    "pixie_unet_check": (C.c_int, [C.c_void_p]),
    "pixie_unet_flops": (C.c_double, [C.c_void_p]),
    "pixie_unet_debug_fetch": (C.c_int64, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int64]),
    "pixie_unet_debug_names": (C.c_int64, [C.c_void_p, C.c_char_p, C.c_int64]),
    "pixie_unet_destroy": (None, [C.c_void_p]),
    "pixie_mpm_create": (C.c_int, [C.c_int, C.c_int, C.c_float, C.POINTER(C.c_void_p)]),
    "pixie_mpm_bind": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p]),
    "pixie_mpm_set_params": (C.c_int, [C.c_void_p, C.POINTER(MpmParams)]),
    "pixie_mpm_add_bc": (C.c_int, [C.c_void_p, C.POINTER(MpmBC)]),
    "pixie_mpm_clear_bcs": (C.c_int, [C.c_void_p]),
    "pixie_mpm_set_time": (C.c_int, [C.c_void_p, C.c_double]),
    "pixie_mpm_get_time": (C.c_int, [C.c_void_p, C.POINTER(C.c_double)]),
    "pixie_mpm_step": (C.c_int, [C.c_void_p, C.c_int, C.c_double, C.c_void_p]),
    "pixie_mpm_compute_mu_lam": (C.c_int, [C.c_void_p, C.c_void_p]),
    "pixie_mpm_compute_bulk": (C.c_int, [C.c_void_p, C.c_void_p]),
    "pixie_mpm_compute_mass": (C.c_int, [C.c_void_p, C.c_void_p]),
    "pixie_mpm_compute_cov_from_F": (C.c_int, [C.c_void_p, C.c_void_p]),
    "pixie_mpm_compute_R_from_F": (C.c_int, [C.c_void_p, C.c_void_p]),
    "pixie_mpm_apply_additional_params": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "pixie_mpm_select_box": (C.c_int, [C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_void_p, C.c_void_p]),
    "pixie_mpm_select_cylinder": (C.c_int, [C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_float, C.c_float, C.c_void_p, C.c_void_p]),
    "pixie_mpm_sync": (C.c_int, [C.c_void_p, C.c_void_p]),
    "pixie_field_extract": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double),
                                      C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int), C.c_void_p]),
    "pixie_knn_assign": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                   C.c_int, C.c_double, C.c_int, C.POINTER(C.c_float), C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int), C.c_void_p]),
    "pixie_dbscan": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_double, C.c_int, C.c_void_p, C.c_void_p, C.POINTER(C.c_int),
                               C.POINTER(C.c_int), C.c_void_p]),
    "pixie_cluster_stats": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "pixie_particle_volume":(C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_void_p, C.c_void_p]),
    "pixie_frame_transform": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_float, C.c_float, C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_int,
                                        C.c_void_p, C.c_void_p, C.c_void_p]),
    "pixie_gaussian_ply_records": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "pixie_gaussian_checkpoint_decode": (C.c_int, [C.c_void_p, C.c_longlong, C.c_int, C.POINTER(C.c_int), C.c_int, C.c_int, C.c_float, C.c_void_p,
                                                   C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_longlong), C.c_void_p]),
    "pixie_gaussian_checkpoint_decode_scale_rot": (C.c_int, [C.c_void_p, C.c_longlong, C.c_int, C.POINTER(C.c_int), C.c_int, C.c_void_p,
                                                             C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "pixie_image_metrics": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_float), C.c_void_p, C.c_void_p]),
    "pixie_material_metrics": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int64, C.POINTER(C.c_double),
                                         C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "pixie_fill_density": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p]),
    "pixie_fill_grids": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_float, C.POINTER(C.c_float), C.c_float, C.c_float, C.c_int, C.c_int,
                                   C.c_int, C.c_ulonglong, C.c_void_p, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_void_p]),
    "pixie_nearest_gaussian": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "pixie_part_similarity": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_float, C.c_void_p,
                                        C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "pixie_knn_label_vote": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "pixie_nearest_vertex": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "pixie_gs_renderer_create": (C.c_int, [C.POINTER(C.c_void_p)]),
    "pixie_gs_render": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                  C.c_void_p, C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_float,
                                  C.c_float, C.c_int, C.c_int, C.POINTER(C.c_float), C.c_void_p, C.c_void_p, C.POINTER(C.c_int),
                                  C.POINTER(C.c_float), C.c_void_p]),
    "pixie_gs_renderer_destroy": (None, [C.c_void_p]),
    "pixie_mpm_set_active_count": (C.c_int, [C.c_void_p, C.c_int]),
    "pixie_mpm_grid_ptrs": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p)]),
    "pixie_mpm_launch_count": (C.c_longlong, [C.c_void_p]),
    "pixie_mpm_exchange_buffer": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t)]),
    "pixie_mpm_slab_attach": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "pixie_mpm_slab_phase": (C.c_int, [C.c_void_p, C.c_int, C.c_double, C.c_void_p]),
    "pixie_mpm_slab_error": (C.c_int, [C.c_void_p, C.POINTER(C.c_int)]),
    "pixie_mpm_slab_excursion": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "pixie_ipc_export": (C.c_int, [C.c_void_p, C.c_char_p]),
    "pixie_ipc_open": (C.c_int, [C.c_char_p, C.POINTER(C.c_void_p)]),
    "pixie_ipc_close": (C.c_int, [C.c_void_p]),
    "pixie_mpm_destroy": (None, [C.c_void_p]),
}

_lib = None


def load():
    """Load libpixie_b200.so and bind every symbol of the header. Raises if the library is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise PixieError(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "or `make -C pixie_b200/csrc`. pixie_b200 has no CPU/PyTorch fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in _SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError here = header/library mismatch
        fn.restype = res
        fn.argtypes = args
    if lib.pixie_abi_version() != ABI_VERSION:
        raise PixieError("libpixie_b200.so ABI version mismatch")
    _lib = lib
    return lib


def last_error() -> PixieError:
    """The library's message for the failure the last call on this thread reported."""
    return PixieError(load().pixie_last_error().decode("utf-8", "replace"))


def check(rc: int):
    if rc != 0:
        raise last_error()


def require_cuda(op: str, *tensors):
    if not all(t.is_cuda for t in tensors):
        raise PixieError(f"{op} requires CUDA tensors; there is no CPU fallback")


def ptr(t):
    """A tensor's device pointer as the library borrows it; None (a null pointer) for an absent array."""
    return None if t is None else C.c_void_p(t.data_ptr())


def stream(dev) -> C.c_void_p:
    """The current stream of `dev`, which every device operation takes as its last argument."""
    return C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def call(name: str, dev, *args):
    """Run the stateless device operation `name` on `dev`'s current stream: tensors are passed as borrowed pointers, every
    other argument as given, and a non-zero return raises the library's message. Callers check the device themselves."""
    with torch.cuda.device(dev):
        check(getattr(load(), name)(*(ptr(a) if isinstance(a, torch.Tensor) else a for a in args), stream(dev)))


def require_device():
    lib = load()
    if not lib.pixie_device_ok():
        raise PixieError("pixie_b200 needs an sm_90 (H100) CUDA device; there is no CPU fallback")
    return lib
