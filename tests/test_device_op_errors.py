"""Failures behind the C ABI, of the stateless device operations and of the MPM, U-Net and rasterizer handles: input that
cannot be indexed is refused before the device is touched, every failure leaves its own message, and a CUDA error is
reported with CUDA's description and does not make the next, valid call fail. A refused allocation leaves a handle as it
was."""
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


def _mpm_pair(cuda_dev, n=2000, ng=32):
    """The solver and the fp32 oracle on smoke()'s 2000-particle scene."""
    from oracle import mpm_ref
    from pixie_b200.mpm_solver_warp import MPM_Simulator_WARP
    sc = mpm_ref.synthetic_scene(n, ng, seed=0)
    s = MPM_Simulator_WARP(10, device=cuda_dev)
    s.load_initial_data_from_torch(torch.from_numpy(sc["x"]).to(cuda_dev), torch.from_numpy(sc["vol"]).to(cuda_dev), None,
                                   n_grid=ng, grid_lim=2.0)
    s.set_parameters_dict({"material": "jelly", "g": [0.0, 0.0, -9.8], "density": 1000.0, "E": 1e5, "nu": 0.3})
    s.mpm_model.E = torch.from_numpy(sc["E"]).to(cuda_dev)
    s.mpm_model.nu = torch.from_numpy(sc["nu"]).to(cuda_dev)
    s.reset_densities_and_update_masses(torch.from_numpy(sc["density"]).to(cuda_dev))
    s.import_particle_v_from_torch(torch.from_numpy(sc["v"]).to(cuda_dev))
    s.finalize_mu_lam()
    s.add_bounding_box()
    o = mpm_ref.MpmRef(n, ng, 2.0, "f32")
    for k, f in (("x", "X"), ("v", "V"), ("vol", "VOL"), ("density", "DENSITY"), ("E", "E"), ("nu", "NU"), ("material", "MATERIAL")):
        o.set(f, sc[k])
    o.compute_mass(); o.compute_mu_lam(); o.set_params(g=(0, 0, -9.8)); o.add_bc(mpm_ref.BC_BBOX)
    return s, o


def _step_and_compare(s, o, n):
    s.p2g2p_n(n, 1e-4)
    o.step(n, 1e-4)
    assert np.abs(s.export_particle_x_to_torch().cpu().numpy() - o.get("X")).max() < 1e-5
    assert np.abs(s.export_particle_v_to_torch().cpu().numpy() - o.get("V")).max() < 1e-3


@pytest.mark.gpu
def test_refused_mpm_create_is_reported_and_not_blamed_on_the_next_call(built_lib, cuda_dev):
    h = C.c_void_p()
    # a 100000^3 grid asks for ~1.6e16 bytes: the allocator refuses it before anything is launched
    assert built_lib.pixie_mpm_create(10, 100000, 1.0, C.byref(h)) != 0
    msg = built_lib.pixie_last_error().decode()
    assert msg.startswith("mpm_create:") and "out of memory" in msg, msg
    assert torch.ones(1000, device=cuda_dev).sum().item() == 1000.0     # torch's launch check finds no stale error
    s, o = _mpm_pair(cuda_dev)
    _step_and_compare(s, o, 20)


@pytest.mark.gpu
def test_refused_regrid_keeps_the_previous_grid(built_lib, cuda_dev):
    from pixie_b200 import _lib
    s, o = _mpm_pair(cuda_dev)
    _step_and_compare(s, o, 10)
    p = _lib.MpmParams()
    p.n_grid, p.grid_lim = 100000, 2.0                  # ~1.6e16 bytes of grid
    s._fence()
    assert built_lib.pixie_mpm_set_params(s._handle, C.byref(p)) != 0
    msg = built_lib.pixie_last_error().decode()
    assert msg.startswith("mpm_set_params:") and "out of memory" in msg, msg
    _step_and_compare(s, o, 20)                        # the refused call changed neither the grid nor the parameters
    s._destroy()
    torch.cuda.synchronize(cuda_dev)


@pytest.mark.gpu
def test_refused_unet_finalize_is_reported_and_not_blamed_on_the_next_call(built_lib, cuda_dev):
    from oracle import unet_ref as O
    from pixie_b200 import _lib
    from pixie_b200.unet import RegressionUNet
    # 8000 x 64^3 x 128 channels of activations need ~1 TB, while every batch x voxel count stays below 2^31
    big = RegressionUNet(feature_channels=128, grid_size=64, out_channels=3, max_batch=8000, precision="fp16",
                         **O.DEFAULT_CFG).to(cuda_dev)
    big.load_state_dict(O.RegressionUNet(feature_channels=128, grid_size=64, out_channels=3, **O.DEFAULT_CFG).state_dict())
    with pytest.raises(_lib.PixieError) as err:
        big._ensure_built()
    assert str(err.value).startswith("unet_finalize:") and "out of memory" in str(err.value), err.value

    C_, G = 128, 16
    _, reg = O.build_pair(C_, G, seed=0)
    x = O.synthetic_features(1, C_, G, seed=1)
    with torch.no_grad():
        y_ref = reg(x)
    net = RegressionUNet(feature_channels=C_, grid_size=G, out_channels=3, max_batch=1, precision="fp16e5", **O.DEFAULT_CFG).to(cuda_dev)
    net.load_state_dict(reg.state_dict())
    y = net(x.to(cuda_dev)).cpu()
    net.check()
    assert (y - y_ref).abs().max().item() < 1e-3


@pytest.mark.gpu
def test_each_failure_leaves_its_own_message(built_lib, cuda_dev):
    from oracle import unet_ref as O
    from pixie_b200 import _lib
    from pixie_b200.unet import RegressionUNet
    p = C.c_void_p(1)                                   # never dereferenced: every call below is refused first
    msgs = []

    def refused(rc):
        assert rc != 0
        msgs.append(built_lib.pixie_last_error().decode())

    m = C.c_void_p()
    _lib.check(built_lib.pixie_mpm_create(100, 16, 1.0, C.byref(m)))
    try:
        refused(built_lib.pixie_mpm_step(m, 1, 1e-4, None))                  # nothing bound
        refused(built_lib.pixie_mpm_slab_phase(m, 0, 1e-4, None))            # not a slab
        bc = _lib.MpmBC()
        bc.kind = _lib.BC_BOUNDING_BOX
        for _ in range(256):
            _lib.check(built_lib.pixie_mpm_add_bc(m, C.byref(bc)))
        refused(built_lib.pixie_mpm_add_bc(m, C.byref(bc)))                  # the 257th
    finally:
        built_lib.pixie_mpm_destroy(m)

    cfg = _lib.UNetConfig(feature_channels=128, cond_dim=32, model_channels=64, num_res_blocks=3, n_levels=4, grid_size=16,
                          out_channels=3, max_batch=1, precision=0)
    cfg.channel_mult[:4] = (1, 1, 2, 4)
    u = C.c_void_p()
    _lib.check(built_lib.pixie_unet_create(C.byref(cfg), C.byref(u)))
    try:
        refused(built_lib.pixie_unet_forward(u, p, 1, p, None))             # before finalize
    finally:
        built_lib.pixie_unet_destroy(u)
    _, reg = O.build_pair(128, 16, seed=0)
    net = RegressionUNet(feature_channels=128, grid_size=16, out_channels=3, max_batch=1, **O.DEFAULT_CFG).to(cuda_dev)
    net.load_state_dict(reg.state_dict())
    net._ensure_built()
    refused(built_lib.pixie_unet_forward(net._handle, p, 2, p, None))       # batch > max_batch

    assert all(msgs), msgs
    assert all(a != b for a, b in zip(msgs, msgs[1:])), msgs
    assert "too many boundary conditions" in msgs[2] and "finalize" in msgs[3] and "max_batch" in msgs[4], msgs
