"""MPM parity against vectors produced by the REFERENCE'S OWN SOURCE.

tests/golden/mpm_golden.npz was written by tests/golden/make_mpm_golden.py, which imports
third_party/PhysGaussian/mpm_solver_warp/{mpm_solver_warp,mpm_utils,warp_utils}.py and executes those
kernels on a float32 `warp` stand-in (tests/golden/_fake_warp.py).  Here the same scenarios (tests/golden/mpm_scenarios.py)
are replayed on
  * oracle/mpm_ref.c (fp32 build) behind the reference's call surface           -> CPU tests (pins the oracle),
  * pixie_b200's MPM_Simulator_WARP, i.e. the CUDA kernels through the C ABI    -> `-m gpu` tests,
and compared field by field: selection masks / material ids exactly, floating-point fields relative to the field's
largest magnitude (float32 arithmetic in a different operation order: a few 1e-7 after one substep, amplified by the
plastic return maps over 20 substeps).  Tolerances are in TOL below.
"""
import json
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, HERE)

import mpm_scenarios as S  # noqa: E402

GOLD = np.load(os.path.join(HERE, "golden", "mpm_golden.npz"))
META = json.loads(bytes(GOLD["meta"]).decode())
NAMES = [sc["name"] for sc in S.scenarios()]

# relative to max|reference field|; positions additionally absolute (domain size 2)
TOL = {"setup": 1e-6, "step1": 5e-6, "step20": 5e-5, "export": 2e-5}
TOL_X_ABS = {"step1": 1e-7, "step20": 1e-6}


def _inputs(name):
    pre = name + "/in/"
    return {k[len(pre):]: GOLD[k] for k in GOLD.files if k.startswith(pre)}


def _check(name, out, skip=()):
    for i, m in enumerate(out["masks"]):
        assert (np.asarray(m) == GOLD[f"{name}/mask/{i}"]).all(), f"{name}: selection mask {i}"
    assert (np.asarray(out["setup"]["particle_material"]).astype(np.int64) == GOLD[f"{name}/setup/particle_material"]).all()
    worst = {}
    # every back end reports the grid velocities of the first substep; they are compared where the reference put mass
    # (the CUDA grid sweep covers only the particles' node box and leaves the nodes outside it alone)
    assert "grid_v_out" in out[1], f"{name}: the back end reported no grid velocities"
    touched = GOLD[f"{name}/step1/grid_m"] > 0
    assert touched.sum() > 100
    for grp, rec in (("setup", out["setup"]), ("step1", out[1]), ("step20", out[20]), ("export", out["export"])):
        for k, v in rec.items():
            if k in skip:
                continue
            ref = GOLD[f"{name}/{grp}/{k}"].astype(np.float64)
            v = np.asarray(v, dtype=np.float64).reshape(ref.shape)
            if k == "grid_v_out":
                ref, v = ref[touched], v[touched]
            assert np.isfinite(v).all(), f"{name}/{grp}/{k} not finite"
            err = np.abs(v - ref).max()
            rel = err / max(np.abs(ref).max(), 1e-30)
            worst[f"{grp}/{k}"] = rel
            assert rel <= TOL[grp], f"{name}/{grp}/{k}: rel {rel:.2e} (abs {err:.2e}) > {TOL[grp]:.0e}"
            if k == "particle_x" and grp in TOL_X_ABS:
                assert err <= TOL_X_ABS[grp], f"{name}/{grp}/particle_x abs {err:.2e}"
    return worst


def test_fixture_covers_every_material_and_quirk():
    mats = set()
    for name in NAMES:
        mats |= set(META[name]["materials"])
    assert mats == {0, 1, 2, 3, 4, 5, 6}
    # plasticity really happened (yield-stress mutation of the von Mises maps, mpm_utils.py:127-131, 165-171)
    for name in ("metal", "snow", "mixed"):
        assert np.abs(GOLD[f"{name}/step20/yield_stress"] - 3e3).max() > 1.0
    # the "cut" collider's 0.3-scaling branch and the non-sticky overwrite-to-zero quirk (:809-840) were exercised
    vo = GOLD["paths/step1/grid_v_out"]
    cut = vo[:, :6, 4, :]                       # y < 0.78 (nodes 0..5 of 6.24), z = 0.5
    assert np.abs(cut[..., 1]).max() == 0.0 and np.abs(cut[..., [0, 2]]).max() > 0.0
    # moving cuboid + rotation modifier + bounding box changed something
    assert np.abs(GOLD["paths/step20/particle_x"] - GOLD["paths/in/x"]).max() > 1e-2


@pytest.mark.parametrize("name", NAMES)
def test_oracle_matches_reference_source(name):
    from mpm_backends import OracleBackend, OracleSolver
    sc = next(s for s in S.scenarios() if s["name"] == name)
    out = S.replay(OracleSolver, sc, OracleBackend(), data=_inputs(name))
    _check(name, out)


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_cuda_matches_reference_source(built_lib, cuda_dev, name):
    from mpm_backends import CudaBackend
    from pixie_b200.mpm_solver_warp import MPM_Simulator_WARP
    sc = next(s for s in S.scenarios() if s["name"] == name)
    out = S.replay(MPM_Simulator_WARP, sc, CudaBackend(), data=_inputs(name))
    worst = _check(name, out)
    print(name, {k: f"{v:.1e}" for k, v in sorted(worst.items(), key=lambda kv: -kv[1])[:5]})
