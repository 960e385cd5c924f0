"""One warm-up + one measured scene (both networks, then a short MPM rollout) for profiler captures."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bench

class A: pass
a = A(); a.grid, a.channels, a.particles, a.mpm_grid = 64, 512, 100_000, 64
prec = sys.argv[1] if len(sys.argv) > 1 else "fp16x3"
nsub = int(sys.argv[2]) if len(sys.argv) > 2 else 50
from pixie_b200.inference import MaterialFieldPredictor
sd_seg, sd_reg = bench.make_state_dicts(a.channels, a.grid)
pred = MaterialFieldPredictor(feature_channels=a.channels, grid_size=a.grid, device="cuda:0", max_batch=1, precision=prec, **bench.UNET_CFG)
pred.load_state_dicts(sd_seg, sd_reg)
feat = bench.make_features(a.grid, a.channels, 1).cuda()
solver = bench.setup_solver(bench.make_mpm_scene(a.particles, a.mpm_grid, 0), a.mpm_grid, "cuda:0")
for _ in range(2):
    pred.predict(feat)
    solver.p2g2p_n(nsub, 1e-4)
torch.cuda.synchronize()
print("done")
