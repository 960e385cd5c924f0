"""CPU-only checks of the boundary: the C-ABI library loads and exports every symbol the header
declares; host-side mirrors of the reference interface behave like the reference without a GPU."""
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_symbols():
    txt = open(os.path.join(ROOT, "include", "pixie_b200.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(pixie_[a-z0-9_]+)\s*\(", txt)))


def test_library_exports_every_header_symbol(built_lib):
    from pixie_b200 import _lib
    syms = _header_symbols()
    assert len(syms) >= 30
    for s in syms:
        assert hasattr(built_lib, s), f"{s} declared in include/pixie_b200.h but not exported"
        assert s in _lib._SIGNATURES, f"{s} has no ctypes signature in pixie_b200/_lib.py"
    assert built_lib.pixie_abi_version() == _lib.ABI_VERSION


def test_no_cpu_fallback(built_lib):
    """Without an sm_90 device every compute entry point must fail loudly."""
    from pixie_b200 import _lib
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    assert built_lib.pixie_device_ok() == 0
    with pytest.raises(_lib.PixieError):
        _lib.require_device()
    import ctypes as C
    h = C.c_void_p()
    cfg = _lib.UNetConfig()
    assert built_lib.pixie_unet_create(C.byref(cfg), C.byref(h)) != 0
    assert b"no CPU fallback" in built_lib.pixie_last_error()
    assert built_lib.pixie_mpm_create(10, 8, 1.0, C.byref(h)) != 0
    from pixie_b200.mpm_solver_warp import MPM_Simulator_WARP
    with pytest.raises(_lib.PixieError):
        MPM_Simulator_WARP(10)


def test_product_package_never_imports_the_oracle():
    for dirpath, _, files in os.walk(os.path.join(ROOT, "pixie_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert "oracle" not in src.replace("no oracle", ""), f"{f} references oracle/"


def test_unet_shim_state_dict_contract():
    """Key names / shapes are the reference's (SURVEY appendix A); strict loading errors like torch."""
    from oracle import unet_ref as O
    from pixie_b200.unet import RegressionUNet, SegmentationUNet, _expected_keys
    ref = O.SegmentationUNet(768, 32, 64, 3, (1, 1, 2, 4), (), 64, 8)
    assert {k: tuple(v.shape) for k, v in ref.state_dict().items()} == _expected_keys(768, 32, 64, 3, (1, 1, 2, 4), 64, 8)
    net = RegressionUNet(64, 32, 64, 1, (1, 2), (), 8, 3)
    small = O.RegressionUNet(64, 32, 64, 1, (1, 2), (), 8, 3)
    sd = O.seeded_state_dict(small, 0)
    missing, unexpected = net.load_state_dict({("module." + k): v for k, v in sd.items()}, strict=False)
    assert not missing and not unexpected
    bad = dict(sd)
    bad.pop("unet.out.2.bias")
    fresh = RegressionUNet(64, 32, 64, 1, (1, 2), (), 8, 3)
    with pytest.raises(RuntimeError):
        fresh.load_state_dict(bad, strict=True)
    m, u = fresh.load_state_dict({**bad, "extra.key": torch.zeros(1)}, strict=False)
    assert m == ["unet.out.2.bias"] and u == ["extra.key"]
    with pytest.raises(RuntimeError):
        fresh.load_state_dict({"unet.out.2.bias": torch.zeros(5)}, strict=False)        # size mismatch
    with pytest.raises(NotImplementedError):
        SegmentationUNet(64, 32, 64, 1, (1, 2), (2,), 8, 8)


def test_material_name_quirk():
    """get_material_name maps NAME -> id (mpm_solver_warp.py:29-39), unknown -> -1."""
    from pixie_b200.mpm_solver_warp import get_material_id, get_material_name
    assert get_material_name("jelly") == 0 and get_material_name("rigid") == 6 and get_material_name("sand") == 2
    assert get_material_name("fluid") == -1 and get_material_name(3) == -1
    assert get_material_id("snow") == 5
