"""Failures of the stateless device operations behind the C ABI: input that cannot be indexed is refused before the device
is touched, and a CUDA error is reported with CUDA's description and does not make the next, valid call fail."""
import ctypes as C

import numpy as np
import pytest
import torch


def test_field_extract_refuses_grids_beyond_int32(built_lib):
    """D^3 voxels are indexed in int32, so D = 1291 is refused by its limit rather than by the device check."""
    p = C.c_void_p(1)                                   # never dereferenced: validation comes first
    ranges, lo, hi = (C.c_double * 6)(), (C.c_double * 3)(), (C.c_double * 3)()
    count = C.c_int(0)
    rc = built_lib.pixie_field_extract(p, 8, p, 1291, ranges, lo, hi, p, p, p, p, p, p, C.byref(count), None)
    assert rc != 0
    msg = built_lib.pixie_last_error()
    assert b"1290" in msg and b"no CPU fallback" not in msg


@pytest.mark.gpu
def test_refused_scratch_is_reported_and_not_blamed_on_the_next_call(built_lib, cuda_dev):
    from pixie_b200.frame_export import get_particle_volume
    stream = C.c_void_p(torch.cuda.current_stream(cuda_dev).cuda_stream)
    # a 100000^3 grid asks for ~4e15 bytes of scratch: the allocator refuses it before anything is launched
    assert built_lib.pixie_particle_volume(None, 0, 100000, 1.0, None, stream) != 0
    msg = built_lib.pixie_last_error().decode()
    assert msg.startswith("particle_volume:") and "out of memory" in msg, msg

    n_grid, dx = 32, 2.0 / 32
    pos = torch.from_numpy(np.random.default_rng(3).uniform(-0.1, 2.1, size=(5000, 3)).astype(np.float32))
    got = get_particle_volume(pos.to(cuda_dev), n_grid, dx).cpu()
    dxf = torch.tensor(dx, dtype=torch.float32)
    cell = torch.clamp(torch.floor(pos / dxf).long(), 0, n_grid - 1)
    flat = (cell[:, 0] * n_grid + cell[:, 1]) * n_grid + cell[:, 2]
    count = torch.bincount(flat, minlength=n_grid ** 3)
    torch.testing.assert_close(got, dxf * dxf * dxf / count[flat].float(), rtol=1e-6, atol=0)
