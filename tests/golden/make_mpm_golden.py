"""Generates tests/golden/mpm_golden.npz by EXECUTING THE REFERENCE'S OWN MPM SOURCE
($PIXIE_REFERENCE/third_party/PhysGaussian/mpm_solver_warp/{mpm_solver_warp,mpm_utils,warp_utils}.py) on the
float32 `warp` stand-in of tests/golden/_fake_warp.py.  PIXIE_REFERENCE names a checkout of the reference:

    python tests/golden/make_mpm_golden.py

The fixture pins oracle/mpm_ref.c (tests/test_mpm_golden.py, CPU) and the CUDA path (same file, `-m gpu`) to what
the reference's kernels compute: every return map (incl. the yield-stress mutation), every stress model, p2g, grid
update with each BC closure, g2p (+update_cov), the selection kernels, apply_additional_params, compute_cov_from_F,
compute_R_from_F, and 20-substep rollouts per material.  Nothing of the reference is copied: it is imported.
"""
import json
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
REF = os.path.join(os.environ["PIXIE_REFERENCE"], "third_party", "PhysGaussian", "mpm_solver_warp")

import _fake_warp as wp  # noqa: E402

wp.install()
for missing in ("h5py", "plyfile"):               # imported by engine_utils.py for file I/O only
    if missing not in sys.modules:
        m = types.ModuleType(missing)
        m.PlyData = m.PlyElement = m.File = None
        sys.modules[missing] = m
sys.path.insert(0, REF)
import mpm_solver_warp as REFMOD  # noqa: E402  (the reference)

import mpm_scenarios as S  # noqa: E402


class ReferenceBackend:
    device = "cpu"

    def tensor(self, a):
        return torch.from_numpy(np.ascontiguousarray(a))

    def to_numpy(self, t):
        return t.detach().numpy()

    def set_state(self, s, name, arr):
        dtype = {"particle_F_trial": wp.mat33, "particle_cov": float}[name]
        setattr(s.mpm_state, name, wp.from_numpy(arr, dtype=dtype))

    def get_state(self, s, names):
        return {k: np.array(getattr(s.mpm_state, k).numpy(), copy=True) for k in names}

    def get_model(self, s, names):
        return {k: np.array(getattr(s.mpm_model, k).numpy(), copy=True) for k in names}

    def get_masks(self, s):
        return [np.array(p.mask.numpy(), copy=True) for p in list(s.impulse_params) + list(s.particle_velocity_modifier_params)]

    def get_grid(self, s):
        return {"grid_m": s.mpm_state.grid_m.numpy().copy(), "grid_v_in": s.mpm_state.grid_v_in.numpy().copy(),
                "grid_v_out": s.mpm_state.grid_v_out.numpy().copy()}


def main():
    blob, meta = {}, {}
    be = ReferenceBackend()
    for sc in S.scenarios():
        d = S.inputs(sc)
        out = S.replay(REFMOD.MPM_Simulator_WARP, sc, be, data=d)
        name = sc["name"]
        for k, v in d.items():
            blob[f"{name}/in/{k}"] = v
        for k, v in out["setup"].items():
            blob[f"{name}/setup/{k}"] = v
        for i, m in enumerate(out["masks"]):
            blob[f"{name}/mask/{i}"] = m.astype(np.int32)
        for cp in S.CHECKPOINTS:
            for k, v in out[cp].items():
                blob[f"{name}/step{cp}/{k}"] = v
        for k, v in out["export"].items():
            blob[f"{name}/export/{k}"] = v
        meta[name] = {"n": sc["n"], "materials": sorted(set(int(v) for v in out["setup"]["particle_material"]))}
        x1, x20 = out[S.CHECKPOINTS[0]]["particle_x"], out[S.CHECKPOINTS[-1]]["particle_x"]
        print(f"{name:12s} materials {meta[name]['materials']}  max|dx| over the rollout {np.abs(x20 - d['x']).max():.3e}  "
              f"finite {np.isfinite(x20).all()}  yield changed {np.abs(out[S.CHECKPOINTS[-1]]['yield_stress'] - 3e3).max() > 0}",
              flush=True)
    blob["meta"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    np.savez_compressed(os.path.join(HERE, "mpm_golden.npz"), **blob)
    print("wrote", os.path.join(HERE, "mpm_golden.npz"), len(blob), "arrays")


if __name__ == "__main__":
    main()
