"""Two (or more) slabs of BASELINE configs[4] inside ONE process on one GPU, driven through the phase API: every flag a kernel
waits for is already raised, so per-kernel times (profiler launch list) show the work of each slab-mode kernel without NVLink or
waiting. usage: profile_slab_local.py [world] [substeps]"""
import contextlib, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from pixie_b200 import _lib
from pixie_b200.mpm_slab import FusedSlabBackend, LocalSlabCluster, SlabRank, balanced_slab_bounds
from pixie_b200.mpm_solver_warp import MPM_Simulator_WARP
from pixie_b200.synthetic import synthetic_scene

world = int(sys.argv[1]) if len(sys.argv) > 1 else 2
nsub = int(sys.argv[2]) if len(sys.argv) > 2 else 4
n, G, lim, dt, slack = 1_000_000, 256, 2.0, 2e-5, 2
dev = "cuda:0"
sc = synthetic_scene(n, G, seed=0, materials=(0,))
base = (sc["x"][:, 0].astype(np.float32) * np.float32(G / lim) - np.float32(0.5)).astype(np.int32)
bounds = balanced_slab_bounds(base, G, world, 2 + 2 * slack)
lib = _lib.require_device()
ranks = []
for rank in range(world):
    x0, x1 = bounds[rank]
    lo = -10 ** 9 if rank == 0 else x0
    hi = 10 ** 9 if rank == world - 1 else x1
    idx = np.where((base >= lo) & (base < hi))[0]
    m, cap = len(idx), len(idx) + 4096
    with contextlib.redirect_stdout(sys.stderr):
        s = MPM_Simulator_WARP(cap, n_grid=G, grid_lim=lim, device=dev)
        for fid, key in (("X", "x"), ("V", "v"), ("VOL", "vol"), ("DENSITY", "density"), ("E", "E"), ("NU", "nu")):
            t = s._t[fid]
            t.view(cap, t.numel() // cap)[:m] = torch.as_tensor(np.asarray(sc[key])[idx].reshape(m, -1), dtype=torch.float32, device=dev)
        s._t["MATERIAL"].view(cap, 1)[:m] = torch.as_tensor(np.asarray(sc["material"])[idx].reshape(m, 1), dtype=torch.int32, device=dev)
        ft = s._t["F_TRIAL"]; ft.zero_(); ft[:, 0, 0] = 1; ft[:, 1, 1] = 1; ft[:, 2, 2] = 1
        s.mpm_model.gravitational_accelaration = (0.0, 0.0, -9.8)
        s.mpm_model.grid_v_damping_scale = 0.9999
        s._push_params()
        _lib.check(lib.pixie_mpm_compute_mass(s._handle, s._stream()))
        _lib.check(lib.pixie_mpm_compute_mu_lam(s._handle, s._stream()))
        s.add_bounding_box()
        s.set_velocity_on_cuboid(point=[1.0, 1.0, 0.62], size=[0.51, 0.51, 0.04], velocity=[0, 0, 0])
    ranks.append(SlabRank(FusedSlabBackend(s, m), rank, world, slack=slack, migrate_every=1000, ids=torch.from_numpy(idx.astype(np.int64)),
                          bounds=bounds[rank]))
cl = LocalSlabCluster(ranks)
for _ in range(nsub):
    cl.substep(dt)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(20):
    cl.substep(dt)
e1.record()
torch.cuda.synchronize()
for r in ranks:
    r.check_device_error()
print(f"world {world}: {e0.elapsed_time(e1) / 20 * 1e3:.1f} us per substep for ALL slabs on one GPU (phase API, direct launches)")
