#!/usr/bin/env python
"""bench.py — headline benchmark of the pixie_b200 hot path on an H100 (see DESIGN.md).

    python bench.py --gpus 1 --steps K --warmup W              # our arm (CUDA, through the C ABI)
    python bench.py ... --dump-outputs DIR                     # also write the last timed step's outputs as DIR/<name>.npy
    python bench.py --impl reference --steps K --warmup W      # reference arm: the CPU path on host cores
    torchrun --nproc-per-node N ... bench.py --gpus N ...      # one rank per GPU, scenes sharded, weak scaling

One "step" = one scene of BASELINE.json configs[1] + configs[2]:
    material field   : SegmentationUNet + RegressionUNet forward on a 64^3 x 512 fp16 voxel grid
    physics rollout  : 1000 MPM substeps of 100k particles on a 64^3 grid
The two halves are timed in two separate regions of exactly K steps each (barrier + synchronize on both
sides, CUDA events on the launching stream, max over ranks); `value` is the U-Net voxels/s, the MPM
particle-steps/s is reported under "mpm"; `ms_per_step` is the sum of both per-step times.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

UNET_CFG = dict(cond_dim=32, model_channels=64, num_res_blocks=3, channel_mult=(1, 1, 2, 4), attention_resolutions=())


def host_cores():
    """Physical cores of the box: what the CPU arms use, set explicitly (torchrun exports OMP_NUM_THREADS=1, and
    torch.get_num_threads() would then report 1)."""
    try:
        import psutil
        n = psutil.cpu_count(logical=False)
    except Exception:
        n = None
    if not n:
        n = max(1, (os.cpu_count() or 2) // 2)
    try:
        n = min(n, len(os.sched_getaffinity(0)))
    except Exception:
        pass
    return int(n)


def peaks():
    """Data-sheet peaks of the H100 SXM at 700 W (dense fp16 tensor rate, HBM3 bandwidth): ceilings, not measured rates."""
    return dict(hbm=3350.0, tensor=989.0, src="H100 SXM data sheet (700 W)")


class ClockSampler:
    """nvidia-smi clocks / throttle reasons during the timed region."""

    def __init__(self, index: int):
        self.index, self.rows, self.proc = index, [], None

    def start(self):
        q = "clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.index), f"--query-gpu={q}", "--format=csv,noheader,nounits", "-lms", "100"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            threading.Thread(target=self._read, daemon=True).start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([c.strip() for c in line.split(",")])

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.15)
        self.proc.terminate()
        sm, mx, reasons = [], [], set()
        for r in self.rows:
            try:
                sm.append(float(r[0])); mx.append(float(r[1]))
                for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), r[3:7]):
                    if v.lower().startswith("active"):
                        reasons.add(name)
            except Exception:
                pass
        load = [s for s in sm if s > 0.6 * max(sm)] if sm else []
        return {"sm_mhz": float(np.median(load)) if load else None, "sm_max_mhz": max(mx) if mx else None,
                "reasons": sorted(reasons), "samples": len(sm)}


# ------------------------------------------------------------------------------------------------ workloads
def make_state_dicts(C, G):
    """Seeded parameters for the two networks (reference key names / shapes)."""
    from pixie_b200.synthetic import seeded_state_dict
    from pixie_b200.unet import _expected_keys
    mk = lambda out, seed: seeded_state_dict(_expected_keys(C, UNET_CFG["cond_dim"], UNET_CFG["model_channels"],
                                                            UNET_CFG["num_res_blocks"], UNET_CFG["channel_mult"], G, out), seed)
    return mk(8, 0), mk(3, 1)


def make_unet_oracle(C, G):
    """CPU baseline / reference arm only: the restated reference modules with the same parameters."""
    from oracle import unet_ref as O
    cfg = dict(UNET_CFG)
    seg = O.SegmentationUNet(feature_channels=C, grid_size=G, num_classes=8, **cfg).eval()
    reg = O.RegressionUNet(feature_channels=C, grid_size=G, out_channels=3, **cfg).eval()
    sd_seg, sd_reg = make_state_dicts(C, G)
    seg.load_state_dict(sd_seg); reg.load_state_dict(sd_reg)
    return seg, reg


def make_features(G, C, seed):
    from pixie_b200.synthetic import synthetic_features_ndhwc
    return synthetic_features_ndhwc(1, C, G, seed=seed)                            # on-disk layout, fp16 NDHWC


def make_mpm_scene(n, ng, seed, materials=(0,)):
    from pixie_b200.synthetic import synthetic_scene
    return synthetic_scene(n, ng, seed=seed, materials=materials)


def setup_solver(sc, ng, dev):
    from pixie_b200.mpm_solver_warp import MPM_Simulator_WARP
    s = MPM_Simulator_WARP(10, device=dev)
    t = lambda a: torch.from_numpy(a).to(dev)
    s.load_initial_data_from_torch(t(sc["x"]), t(sc["vol"]), None, n_grid=ng, grid_lim=2.0, device=dev)
    s.set_parameters_dict({"material": "jelly", "g": [0.0, 0.0, -9.8], "density": 1000.0, "E": 1e5, "nu": 0.3, "yield_stress": 2e3,
                           "friction_angle": 30.0, "grid_v_damping_scale": 0.9999, "rpic_damping": 0.0}, device=dev)
    s.mpm_model.E = t(sc["E"]); s.mpm_model.nu = t(sc["nu"])
    s.mpm_state.particle_material = t(sc["material"])
    s.reset_densities_and_update_masses(t(sc["density"]))
    s.import_particle_v_from_torch(t(sc["v"]))
    s.finalize_mu_lam()
    s.add_bounding_box()
    s.set_velocity_on_cuboid(point=[1.0, 1.0, 0.62], size=[0.51, 0.51, 0.04], velocity=[0, 0, 0])   # "stationary" cluster pin
    s.add_impulse_on_particles(force=[0.05, 0.0, -0.02], dt=1e-4, point=[1.0, 1.0, 1.2], size=[0.2, 0.2, 0.1], num_dt=20)
    return s


def setup_oracle_mpm(sc, ng, parallel=1, precision="f32"):
    from oracle import mpm_ref as R
    n = sc["x"].shape[0]
    o = R.MpmRef(n, ng, 2.0, precision)
    for k, f in (("x", "X"), ("v", "V"), ("vol", "VOL"), ("density", "DENSITY"), ("E", "E"), ("nu", "NU"), ("material", "MATERIAL")):
        o.set(f, sc[k])
    o.set("YIELD", np.full(n, 2e3))
    o.compute_mass(); o.compute_mu_lam()
    o.set_params(g=(0, 0, -9.8), grid_v_damping_scale=0.9999, parallel_p2g=parallel, alpha=R.friction_alpha(30.0))
    o.add_bc(R.BC_BBOX)
    o.add_bc(R.BC_CUBOID, point=[1.0, 1.0, 0.62], size=[0.51, 0.51, 0.04])
    mask = (np.abs(sc["x"] - np.float32([1.0, 1.0, 1.2])) < np.float32([0.2, 0.2, 0.1])).all(1).astype(np.int32)
    o.add_bc(R.BC_IMPULSE, velocity=[0.05, 0.0, -0.02], start_time=0.0, end_time=20e-4, mask=mask)
    return o


def run_mpm_slab_block(args, rank, world, dev, pk):
    """BASELINE.json configs[4]: ONE 1M-particle scene on a 256^3 grid, strong scaling over the ranks. N = 1 runs the
    undivided scene; N > 1 shards it into x-slabs with (nearly) equal particle counts: the overlap sums are exchanged on
    the device (the grid sweep adds the neighbours' partial sums straight from their memory over NVLink after one flag handshake), particle migration every
    `migrate_every` substeps goes through NCCL send/recv. Returns the dict reported under "mpm_slab" (rank 0) or None."""
    import contextlib
    import torch.distributed as dist
    from pixie_b200 import _lib
    from pixie_b200.mpm_slab import DistSlabDriver, FusedSlabBackend, SlabRank, balanced_slab_bounds
    from pixie_b200.mpm_solver_warp import MPM_Simulator_WARP
    from pixie_b200.synthetic import synthetic_scene
    # dt: the scene's stiffest particles (E = 10^6.5, rho = 200) have a wave speed of 126 m/s; with dx = 2/256 the explicit update
    # needs c dt / dx < 1, i.e. dt < 6e-5 (the 64^3 scene of configs[2] runs at 1e-4 with dx = 2/64)
    n, G, lim, dt = args.slab_particles, args.slab_grid, 2.0, 2e-5
    slack, migrate_every, lazy = args.slab_slack, args.slab_migrate_every, args.slab_lazy_trigger
    sc = synthetic_scene(n, G, seed=0, materials=(0,))              # identical on every rank (seeded)
    base = (sc["x"][:, 0].astype(np.float32) * np.float32(G / lim) - np.float32(0.5)).astype(np.int32)
    bounds = balanced_slab_bounds(base, G, world, 2 + 2 * slack) if world > 1 else [(0, G)]
    x0, x1 = bounds[rank]
    lo = -10 ** 9 if rank == 0 else x0
    hi = 10 ** 9 if rank == world - 1 else x1
    idx = np.where((base >= lo) & (base < hi))[0]
    cap = n if world == 1 else max(len(idx) + 4096, int(1.25 * n / world) + 4096)
    m = len(idx)
    with contextlib.redirect_stdout(sys.stderr):
        s = MPM_Simulator_WARP(cap, n_grid=G, grid_lim=lim, device=dev)

        def put(fid, arr, dtype=torch.float32):
            t = s._t[fid]
            t.view(cap, t.numel() // cap)[:m] = torch.as_tensor(np.asarray(arr)[idx].reshape(m, -1), dtype=dtype, device=dev)

        for fid, key in (("X", "x"), ("V", "v"), ("VOL", "vol"), ("DENSITY", "density"), ("E", "E"), ("NU", "nu")):
            put(fid, sc[key])
        put("MATERIAL", sc["material"], torch.int32)
        ft = s._t["F_TRIAL"]; ft.zero_(); ft[:, 0, 0] = 1; ft[:, 1, 1] = 1; ft[:, 2, 2] = 1
        s.mpm_model.gravitational_accelaration = (0.0, 0.0, -9.8)
        s.mpm_model.grid_v_damping_scale = 0.9999
        s._push_params()
        lib = _lib.require_device()
        _lib.check(lib.pixie_mpm_compute_mass(s._handle, s._stream()))
        _lib.check(lib.pixie_mpm_compute_mu_lam(s._handle, s._stream()))
        s.add_bounding_box()
        s.set_velocity_on_cuboid(point=[1.0, 1.0, 0.62], size=[0.51, 0.51, 0.04], velocity=[0, 0, 0])
    if world > 1:
        r = SlabRank(FusedSlabBackend(s, m), rank, world, slack=slack, migrate_every=migrate_every,
                     ids=torch.from_numpy(idx.astype(np.int64)), bounds=bounds[rank], lazy_trigger=lazy if lazy > 0 else None)
        drv = DistSlabDriver(r)
        run = lambda k: drv.run(k, dt)
        active = lambda: r.b.active
    else:
        run = lambda k: s.p2g2p_n(k, dt)
        active = lambda: m
    sub = args.slab_substeps
    run(migrate_every * 2)                                            # warm-up: graphs instantiated, first migration done
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    checks0, migr0 = (r.checks, r.migrations) if world > 1 else (0, 0)
    e0.record(); run(sub); e1.record()
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    t = torch.tensor([e0.elapsed_time(e1)], device=dev, dtype=torch.float64)
    cnt = torch.tensor([float(active())], device=dev, dtype=torch.float64)
    checks, migrations = (r.checks - checks0, r.migrations - migr0) if world > 1 else (0, 0)
    mx = cnt.clone()
    if world > 1:
        derr = torch.tensor([float(r.b.error())], device=dev, dtype=torch.float64)
        dist.all_reduce(derr, op=dist.ReduceOp.MAX)
        if derr.item() != 0:             # same value on every rank: all of them leave together
            raise RuntimeError(f"slab exchange reported device error {int(derr.item())} (1: neighbour timeout, 2: drift beyond slack)")
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        dist.all_reduce(cnt, op=dist.ReduceOp.SUM)
        dist.all_reduce(mx, op=dist.ReduceOp.MAX)
    xs = s.mpm_state.particle_x.numpy()[: active()]
    fin = torch.tensor([float(np.isfinite(xs).all() and xs.min() > 0.3 and xs.max() < 1.7)], device=dev, dtype=torch.float64)
    if world > 1:
        dist.all_reduce(fin, op=dist.ReduceOp.MIN)
    # ---- the decomposed run against the undivided one (same scene, same number of substeps, rank 0's GPU): the device-side
    #      exchange must reproduce it up to the summation order of the fp32 atomics
    vs_single = None
    if world > 1 and not args.skip_slab_parity:
        total_sub = migrate_every * 2 + sub
        x_all = drv.gather("X")                                       # rank 0: [n, 3] ordered by global particle id
        if rank == 0:
            with contextlib.redirect_stdout(sys.stderr):
                w = MPM_Simulator_WARP(n, n_grid=G, grid_lim=lim, device=dev)
                for fid, key in (("X", "x"), ("V", "v"), ("VOL", "vol"), ("DENSITY", "density"), ("E", "E"), ("NU", "nu")):
                    tt = w._t[fid]
                    tt.view(n, tt.numel() // n)[:] = torch.as_tensor(np.asarray(sc[key]).reshape(n, -1), dtype=torch.float32, device=dev)
                w._t["MATERIAL"].view(n, 1)[:] = torch.as_tensor(np.asarray(sc["material"]).reshape(n, 1), dtype=torch.int32, device=dev)
                ft = w._t["F_TRIAL"]; ft.zero_(); ft[:, 0, 0] = 1; ft[:, 1, 1] = 1; ft[:, 2, 2] = 1
                w.mpm_model.gravitational_accelaration = (0.0, 0.0, -9.8)
                w.mpm_model.grid_v_damping_scale = 0.9999
                w._push_params()
                _lib.check(lib.pixie_mpm_compute_mass(w._handle, w._stream()))
                _lib.check(lib.pixie_mpm_compute_mu_lam(w._handle, w._stream()))
                w.add_bounding_box()
                w.set_velocity_on_cuboid(point=[1.0, 1.0, 0.62], size=[0.51, 0.51, 0.04], velocity=[0, 0, 0])
                w.p2g2p_n(total_sub, dt)
            xw = w.mpm_state.particle_x.numpy().reshape(n, 3).astype(np.float64)
            moved = float(np.abs(xw - np.asarray(sc["x"], dtype=np.float64).reshape(n, 3)).max())
            dmax = float(np.abs(x_all.numpy().reshape(n, 3) - xw).max())
            vs_single = {"max_abs_dx": dmax, "substeps": total_sub, "max_displacement_of_the_run": moved, "tolerance": 1e-4,
                         "ok": bool(dmax < 1e-4)}
            del w
    if rank != 0:
        return None
    ms = float(t.item())
    algo = 212.0 * n + 56.0 * G ** 3                                  # SURVEY.md 8d: 1.15 GB per substep at 1M / 256^3
    ach = algo * sub / (ms * 1e-3) * 1e-9
    # node box of the particles (yz extent) x shared planes x 16 B: what one grid sweep reads from ONE neighbour per substep
    ext = [int(np.floor(sc["x"][:, a].max() * G / lim - 0.5)) + 3 - int(np.floor(sc["x"][:, a].min() * G / lim - 0.5)) + 4 for a in (1, 2)]
    return {"metric": "mpm_particle_steps_per_s", "value": n * sub / (ms * 1e-3), "unit": "particle-steps/s", "us_per_substep": ms / sub * 1e3,
            "scaling": "strong", "substeps": sub, "particles": n, "grid": G, "particles_after": int(cnt.item()),
            "state_finite_and_in_bounds": bool(fin.item() > 0), "vs_single_domain_run": vs_single, "dt": dt, "max_particles_per_rank": int(mx.item()), "slab_bounds": bounds, "slack_planes": slack, "migrate_every": migrate_every,
            "lazy_trigger_planes": lazy, "migration_checks_in_timed_region": checks, "migrations_in_timed_region": migrations,
            "exchange": ("none (undivided scene)" if world == 1 else
                         "device-side: the grid sweep reads the neighbours' partial sums over NVLink (cudaIpc-mapped grids, one flag handshake per substep); "
                         "migration over NCCL send/recv"),
            "halo_bytes_per_substep_per_neighbour": 0 if world == 1 else (2 + 2 * slack) * ext[0] * ext[1] * 16,
            "roofline": {"bound": "hbm", "achieved": ach, "peak": pk["hbm"] * world, "unit": "GB/s", "frac": ach / (pk["hbm"] * world),
                         "note": "algorithmic bytes 212*Np + 56*Ng per substep of the whole scene / (N x measured HBM peak)"}}


# ------------------------------------------------------------------------------------------------ reference arm
def run_reference(args, emit):
    """The reference's own CPU implementation of the path on the host cores: the restated PyTorch modules
    (oracle/unet_ref.py, bit-identical to the reference's — tests/test_oracle_unet.py) and the C
    restatement of its Warp kernels (oracle/mpm_ref.c; warp-lang is not installable here)."""
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    G, C, n, ng = args.grid, args.channels, args.particles, args.mpm_grid
    cores = host_cores()
    torch.set_num_threads(cores)
    seg, reg = make_unet_oracle(C, G)
    x = make_features(G, C, 1).float().permute(0, 4, 1, 2, 3).contiguous()       # fp32 NCDHW, my_data.py:221
    sc = make_mpm_scene(n, ng, 0)
    o = setup_oracle_mpm(sc, ng)
    o.set_num_threads(cores)
    sample_sub = args.ref_substeps
    t_un, t_mp = [], []
    for it in range(args.warmup + args.steps):
        t0 = time.perf_counter()
        with torch.no_grad():
            seg(x); reg(x)
        t1 = time.perf_counter()
        o.step(sample_sub, 1e-4)
        t2 = time.perf_counter()
        if it >= args.warmup:
            t_un.append(t1 - t0); t_mp.append(t2 - t1)
    vps = G ** 3 * len(t_un) / sum(t_un)
    pps = n * sample_sub * len(t_mp) / sum(t_mp)
    sample = f"U-Net: full seg+reg forward at {G}^3x{C} per step; MPM: {sample_sub} of {args.substeps} substeps of the {n}-particle scene per step"
    measured_ms = 1e3 * (sum(t_un) + sum(t_mp)) / len(t_un)
    line = {
        "impl": "reference", "metric": "unet_voxels_per_s", "value": vps, "unit": "voxels/s", "n_gpus": args.gpus,
        "steps": args.steps, "warmup": args.warmup,
        # measured wall time of one step of THIS run (full U-Net forward pair + the bounded MPM sample)
        "ms_per_step": measured_ms,
        # not measured: the same step with all `substeps` MPM substeps, extrapolated from the sample's rate
        "ms_per_step_full_workload_extrapolated": 1e3 * (sum(t_un) + sum(t_mp) * args.substeps / sample_sub) / len(t_un),
        "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": workload_config(args), "precision": "f32 (CPU)",
        "mpm": {"metric": "mpm_particle_steps_per_s", "value": pps, "unit": "particle-steps/s"},
        "cpu_baseline": {"value": vps, "unit": "voxels/s", "cores": cores, "kind": "port", "sample": sample,
                         "mpm_value": pps, "mpm_unit": "particle-steps/s", "mpm_threads": o.num_threads(),
                         "torch_threads": torch.get_num_threads()},
        "e2e": {"value": vps, "unit": "voxels/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
    }
    emit(json.dumps(line))


def workload_config(args):
    """Identical for both arms (the arithmetic precision of an arm is reported under the top-level "precision" key)."""
    return {"workload": f"configs[1]+configs[2]: U-Net seg+reg forward on one {args.grid}^3x{args.channels} fp16 voxel grid, then "
                        f"{args.substeps} MPM substeps of {args.particles} particles on a {args.mpm_grid}^3 grid; 1 scene per GPU per step",
            "parallelism": f"scene-dp{args.gpus}",
            "l2": "U-Net input grid (268 MB) and activations exceed the 50 MB L2; the MPM working set (36 MB/substep) fits in it, "
                  "a 256 MB buffer is written between timed steps"}


# ------------------------------------------------------------------------------------------------ our arm
def run_ours(args, emit):
    import torch.distributed as dist
    from pixie_b200 import _lib
    from pixie_b200.inference import MaterialFieldPredictor

    rank, world = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    _lib.load()
    torch.cuda.set_device(local)
    dev = f"cuda:{local}"
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device(dev))
    G, C, n, ng, SUB = args.grid, args.channels, args.particles, args.mpm_grid, args.substeps
    pk = peaks()

    # ---- build: identical seeded weights on every rank (weights replicated, scenes sharded)
    sd_seg, sd_reg = make_state_dicts(C, G)
    pred = MaterialFieldPredictor(feature_channels=C, grid_size=G, device=dev, max_batch=1, precision=args.precision, **UNET_CFG)
    pred.load_state_dicts(sd_seg, sd_reg)
    feat_host = make_features(G, C, 1 + rank).pin_memory()
    feat_dev = feat_host.to(dev)
    sc = make_mpm_scene(n, ng, rank)
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.float32, device=dev)        # 256 MB > L2

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def timed(fn, steps, warmup, prep=None):
        """K steps of fn(), each preceded by an (untimed, event-excluded) L2 flush + prep; returns the
        max-over-ranks sum of per-step device times in ms."""
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
        for _ in range(warmup):
            if prep: prep()
            fn()
        barrier()
        for i in range(steps):
            if prep: prep()
            flush.fill_(1.0)
            ev[i][0].record(); fn(); ev[i][1].record()
        barrier()
        ms = sum(a.elapsed_time(b) for a, b in ev)
        t = torch.tensor([ms], device=dev, dtype=torch.float64)
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()

    # ---- region 1: material field (both networks), inputs resident in HBM
    out_holder = {}
    def unet_step():
        out_holder["seg"], out_holder["cont"] = pred.predict(feat_dev)
    ms_unet = timed(unet_step, args.steps, args.warmup)
    pred.seg_network.check(); pred.cont_network.check()
    dumps = {}                      # --dump-outputs: what the timed paths returned in their last step
    if args.dump_outputs and rank == 0:
        dumps["unet_seg_logits"] = out_holder["seg"].float().cpu().numpy()
        dumps["unet_cont"] = out_holder["cont"].float().cpu().numpy()

    # ---- region 2: MPM rollout, state resident; every step restarts from the same initial scene
    solver = setup_solver(sc, ng, dev)
    x0, v0 = solver.export_particle_x_to_torch().clone(), solver.export_particle_v_to_torch().clone()
    def mpm_prep():
        solver.export_particle_x_to_torch().copy_(x0); solver.export_particle_v_to_torch().copy_(v0)
        solver._t["C"].zero_(); ft = solver._t["F_TRIAL"]; ft.zero_(); ft[:, 0, 0] = 1; ft[:, 1, 1] = 1; ft[:, 2, 2] = 1
        solver.time = 0.0
    def mpm_step():
        solver.p2g2p_n(SUB, 1e-4)
    launches0 = solver.launch_count()
    ms_mpm = timed(mpm_step, args.steps, args.warmup, prep=mpm_prep)
    mpm_launches_per_rollout = (solver.launch_count() - launches0) / (args.steps + args.warmup)
    x_after_rollout = solver.export_particle_x_to_torch().clone()                   # state after SUB substeps from the initial scene
    if args.dump_outputs and rank == 0:
        dumps["mpm_x"] = x_after_rollout.float().cpu().numpy()
        dumps["mpm_v"] = solver.export_particle_v_to_torch().float().cpu().numpy()
    clocks = sampler.stop() if rank == 0 else None

    # ---- optional variants of SURVEY 8d config 3: the SVD-based plastic materials (one rollout each, after a warm-up)
    variants = {}
    if rank == 0 and not args.skip_variants:
        for name, mat in (("sand", 2), ("metal", 1)):
            sv = setup_solver(make_mpm_scene(n, ng, rank, materials=(mat,)), ng, dev)
            sv.p2g2p_n(100, 1e-4)
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(); sv.p2g2p_n(SUB, 1e-4); b.record(); torch.cuda.synchronize()
            xs = sv.export_particle_x_to_torch()
            variants[name] = {"us_per_substep": a.elapsed_time(b) / SUB * 1e3, "particle_steps_per_s": n * SUB / (a.elapsed_time(b) * 1e-3),
                              "finite": bool(torch.isfinite(xs).all().item())}
            del sv

    # ---- e2e: host buffers in, host results out, through the public API (per step: H2D grid, both nets,
    #      pack, D2H field; H2D particles, rollout, D2H positions)
    packed_host = torch.empty((1, 11, G, G, G), dtype=torch.float32).pin_memory()
    host_scene = {k: torch.from_numpy(v).pin_memory() for k, v in sc.items() if k != "material"}
    x_out_host = torch.empty((n, 3), dtype=torch.float32).pin_memory()
    def e2e_unet():
        pred.predict_packed_host(feat_host, packed_host)
    def e2e_mpm():
        solver.export_particle_x_to_torch().copy_(host_scene["x"], non_blocking=True)
        solver.export_particle_v_to_torch().copy_(host_scene["v"], non_blocking=True)
        solver._t["E"].copy_(host_scene["E"], non_blocking=True); solver._t["NU"].copy_(host_scene["nu"], non_blocking=True)
        solver._t["DENSITY"].copy_(host_scene["density"], non_blocking=True); solver._t["VOL"].copy_(host_scene["vol"], non_blocking=True)
        solver.reset_densities_and_update_masses(solver._t["DENSITY"]); solver.finalize_mu_lam()
        solver.p2g2p_n(SUB, 1e-4)
        x_out_host.copy_(solver.export_particle_x_to_torch(), non_blocking=True)
        torch.cuda.current_stream().synchronize()
    # K scenes through the pipelined host API: scene i+1's H2D overlaps scene i's networks; every scene's H2D and D2H is inside the
    # timed region, which is bracketed like the others (barrier + synchronize, CUDA events, max over ranks). The 268 MB input
    # grid is larger than L2, so there is no flush between the scenes of one pipelined run.
    def e2e_unet_pipelined(k):
        pred.predict_packed_host_stream([feat_host] * k, [packed_host] * k)
    for _ in range(max(1, args.warmup // 2)):
        e2e_unet_pipelined(2)
    # two repetitions of the K-scene run, the better one is reported (both are in the JSON): a single host-side hiccup — one
    # 225 ms scene was seen once on a 2-GPU box, three re-runs on another box were within 1 % of each other — would otherwise
    # decide the end-to-end figure
    e2e_samples = []
    for _ in range(2):
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); e2e_unet_pipelined(args.steps); e1.record()
        barrier()
        tt = torch.tensor([e0.elapsed_time(e1)], device=dev, dtype=torch.float64)
        if world > 1:
            dist.all_reduce(tt, op=dist.ReduceOp.MAX)
        e2e_samples.append(float(tt.item()))
    ms_e2e_unet = min(e2e_samples)
    ms_e2e_unet_serial = timed(e2e_unet, args.steps, args.warmup)
    ms_e2e_mpm = timed(e2e_mpm, args.steps, args.warmup, prep=mpm_prep)
    h2d = feat_host.numel() * 2 + sum(t.numel() * 4 for t in host_scene.values())
    d2h = packed_host.numel() * 4 + x_out_host.numel() * 4

    # ---- live per-kernel numbers (rank 0): conv kernel share and achieved TFLOP/s; MPM substep bytes
    roof, roof_mpm, breakdown, n_launch = None, None, None, None
    if rank == 0:
        prof = pred.seg_network.profile(feat_dev) + pred.cont_network.profile(feat_dev)
        by = {}
        for kind, ms, fl in prof:
            a = by.setdefault(kind, [0, 0.0, 0.0]); a[0] += 1; a[1] += ms; a[2] += fl
        conv_ms, conv_fl = by["conv"][1], by["conv"][2]
        ach = conv_fl / (conv_ms * 1e-3) * 1e-12
        roof = {"kernel": "conv3d_igemm_kernel (wgmma implicit GEMM), all convolutions of seg+reg", "bound": "tensor",
                "achieved": ach, "peak": pk["tensor"], "unit": "TFLOP/s", "frac": ach / pk["tensor"],
                "peak_source": pk["src"] + ", dense fp16",
                "note": "achieved = algorithmic FLOPs (2*MACs of the reference graph) / sum of conv launch times from CUDA events; "
                        + {"fp16x3": "fp16x3 executes 3 fp16 tensor-core passes per algorithmic FLOP (ceiling 1/3)",
                           "fp16e5": "fp16e5 executes one fp16 pass + one E5M2 pass at twice the rate = 2 pass-equivalents per algorithmic FLOP (ceiling 1/2)",
                           "fp16": "1 tensor-core pass (does not meet the 1e-3 tolerance)"}[args.precision]}
        breakdown = {k: {"launches": v[0], "ms": round(v[1], 4)} for k, v in by.items()}
        per_sub_bytes = 212.0 * n + 56.0 * ng ** 3
        sub_s = ms_mpm * 1e-3 / (args.steps * SUB)
        roof_mpm = {"kernel": "mpm substep: mpm_fused_kernel (g2p + stress + p2g) + mpm_gridbox_kernel", "bound": "hbm", "achieved": per_sub_bytes / sub_s * 1e-9,
                    "peak": pk["hbm"], "unit": "GB/s", "frac": per_sub_bytes / sub_s * 1e-9 / pk["hbm"], "peak_source": pk["src"],
                    "algorithmic_bytes_per_substep": per_sub_bytes, "us_per_substep": sub_s * 1e6}
        # counted, not estimated: the U-Net executors and the MPM handle count the kernels they enqueue (graph replays count their nodes)
        n_launch = int(round(args.steps * (pred.seg_network.launch_count() + pred.cont_network.launch_count() + mpm_launches_per_rollout)))

    # ---- parity of the benchmarked mode and CPU baseline (rank 0, N=1 only: bounded sample)
    cpu, parity = None, None
    if rank == 0 and world == 1 and not args.skip_cpu:
        cores = host_cores()
        torch.set_num_threads(cores)
        seg_o, reg_o = make_unet_oracle(C, G)
        x32 = feat_host.float().permute(0, 4, 1, 2, 3).contiguous()
        t0 = time.perf_counter()
        with torch.no_grad():
            ys, yr = seg_o(x32), reg_o(x32)
        t_cpu_unet = time.perf_counter() - t0
        parity = {"unet_max_abs_err_cont": float((out_holder["cont"].cpu() - yr).abs().max()),
                  "unet_max_abs_err_seg_logits": float((out_holder["seg"].cpu() - ys).abs().max()),
                  "tolerance": 2e-2 if args.precision == "fp16" else 1e-3}
        # MPM: the full rollout in the oracle, fp32 (= the CPU baseline sample, and the noise floor) and fp64 (drift reference):
        # north-star "particle-position drift < 1e-4 vs the reference over 1000 steps" on the benchmarked scene itself
        cpu_sub = SUB if not args.skip_drift else args.ref_substeps
        o = setup_oracle_mpm(sc, ng)
        o.set_num_threads(cores)
        t0 = time.perf_counter(); o.step(cpu_sub, 1e-4); t_cpu_mpm = time.perf_counter() - t0
        if not args.skip_drift:
            o64 = setup_oracle_mpm(sc, ng, precision="f64")
            o64.step(SUB, 1e-4)
            xg = x_after_rollout.cpu().numpy().astype(np.float64)
            parity.update({"mpm_substeps": SUB, "mpm_drift_vs_fp64_oracle": float(np.abs(xg - o64.get("X")).max()),
                           "mpm_fp32_oracle_vs_fp64_oracle": float(np.abs(o.get("X") - o64.get("X")).max()),
                           "mpm_drift_vs_fp32_oracle": float(np.abs(xg - o.get("X")).max()), "mpm_drift_tolerance": 1e-4})
        cpu = {"value": G ** 3 / t_cpu_unet, "unit": "voxels/s", "cores": cores, "kind": "port",
               "sample": f"one seg+reg forward at {G}^3x{C} (oracle/unet_ref.py, fp32 torch CPU, {cores} threads); "
                         f"MPM: {cpu_sub} substeps of the {n}-particle scene (oracle/mpm_ref.c fp32, OpenMP {o.num_threads()} threads)",
               "mpm_value": n * cpu_sub / t_cpu_mpm, "mpm_unit": "particle-steps/s"}

    # ---- configs[4]: one big scene, slab-decomposed over the ranks (strong scaling; N = 1 is the undivided scene)
    slab = None
    if not args.skip_slab:
        del solver
        torch.cuda.empty_cache()
        try:
            slab = run_mpm_slab_block(args, rank, world, dev, pk)
        except Exception as e:           # reported, not fatal: the headline line must still be printed
            slab = {"error": f"{type(e).__name__}: {e}"}
            print(f"[bench] mpm_slab block failed on rank {rank}: {slab['error']}", file=sys.stderr)

    if world > 1:
        dist.barrier()
        dist.destroy_process_group()
    if rank != 0:
        return
    if args.dump_outputs:
        os.makedirs(args.dump_outputs, exist_ok=True)
        for name, a in dumps.items():
            np.save(os.path.join(args.dump_outputs, name + ".npy"), np.ascontiguousarray(a, dtype=np.float32))
    K = args.steps
    vps = world * G ** 3 * K / (ms_unet * 1e-3)
    pps = world * n * SUB * K / (ms_mpm * 1e-3)
    line = {
        "metric": "unet_voxels_per_s", "value": vps, "unit": "voxels/s", "n_gpus": world, "steps": K, "warmup": args.warmup,
        "ms_per_step": (ms_unet + ms_mpm) / K, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": args.precision + " (U-Net, fp32 accumulate) + f32 (MPM)", "data": "synthetic",
        "config": workload_config(args), "precision": args.precision,
        "unet_ms_per_scene": ms_unet / K, "mpm_ms_per_rollout": ms_mpm / K,
        "unet_streams": 1 if os.environ.get("PIXIE_UNET_STREAMS", "2") == "1" else 2,
        "unet_streams_note": "the two networks of a scene run concurrently on two streams (CUDA-graph replays); unet_kernel_breakdown_ms and roofline use "
                             "per-launch CUDA events of each network run ALONE, so their sum may exceed unet_ms_per_scene",
        "mpm": {"metric": "mpm_particle_steps_per_s", "value": pps, "unit": "particle-steps/s", "us_per_substep": ms_mpm / K / SUB * 1e3,
                "variants": variants},
        "mpm_slab": slab,
        "roofline": roof, "roofline_mpm": roof_mpm, "unet_kernel_breakdown_ms": breakdown,
        "cpu_baseline": cpu, "parity": parity,
        "e2e": {"value": world * G ** 3 * K / (ms_e2e_unet * 1e-3), "unit": "voxels/s", "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": d2h,
                "mpm_value": world * n * SUB * K / (ms_e2e_mpm * 1e-3), "mpm_unit": "particle-steps/s",
                "ms_per_step": (ms_e2e_unet + ms_e2e_mpm) / K,
                "api": "MaterialFieldPredictor.predict_packed_host_stream (H2D of scene i+1 overlaps the networks of scene i) + MPM_Simulator_WARP.p2g2p_n",
                "unpipelined_value": world * G ** 3 * K / (ms_e2e_unet_serial * 1e-3),
                "unet_ms_samples": [m / K for m in e2e_samples], "unet_ms_reported": "min of the two K-scene repetitions"},
        "gpu_launches": n_launch, "clocks": clocks,
    }
    emit(json.dumps(line))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--precision", default="fp16e5", choices=["fp16e5", "fp16x3", "fp16"],
                    help="fp16e5 (default: one fp16 pass + one E5M2 pass = 2 pass-equivalents) and fp16x3 (3 fp16 passes) meet the "
                         "1e-3 material-field tolerance; fp16 is the single-pass mode (4.5e-3)")
    ap.add_argument("--grid", type=int, default=64)
    ap.add_argument("--channels", type=int, default=512)
    ap.add_argument("--particles", type=int, default=100_000)
    ap.add_argument("--mpm-grid", type=int, default=64)
    ap.add_argument("--substeps", type=int, default=1000)
    ap.add_argument("--ref-substeps", type=int, default=20, help="MPM substeps per step in the CPU sample")
    ap.add_argument("--skip-cpu", action="store_true")
    ap.add_argument("--skip-drift", action="store_true", help="CPU MPM sample of --ref-substeps instead of the full rollout + fp64 drift check")
    ap.add_argument("--skip-variants", action="store_true", help="skip the sand / metal MPM timing variants")
    ap.add_argument("--skip-slab", action="store_true", help="skip the configs[4] block (one 1M-particle / 256^3 scene over all ranks)")
    ap.add_argument("--slab-particles", type=int, default=1_000_000)
    ap.add_argument("--slab-grid", type=int, default=256)
    ap.add_argument("--slab-substeps", type=int, default=200)
    ap.add_argument("--skip-slab-parity", action="store_true", help="skip the decomposed-vs-undivided trajectory check at N > 1")
    ap.add_argument("--slab-slack", type=int, default=2, help="planes a particle may drift out of its slab between two migrations")
    ap.add_argument("--slab-migrate-every", type=int, default=25, help="substeps between two migration check points")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write the last step's outputs (U-Net seg logits and material field, MPM positions "
                         "and velocities after the rollout) to DIR/<name>.npy as float32; inputs are seeded, so runs with the same "
                         "arguments can be compared output for output")
    ap.add_argument("--slab-lazy-trigger", type=int, default=2,
                    help="migrate only once a particle is this many planes outside its slab (0: migrate at every check point)")
    args = ap.parse_args()
    if args.warmup < 3 and args.impl == "ours":
        args.warmup = 3
    # the shims mirror the reference's progress prints; keep stdout for the ONE JSON line
    import contextlib
    real_stdout = sys.stdout
    out = {}
    def emit(line):
        out["line"] = line
    with contextlib.redirect_stdout(sys.stderr):
        if args.impl == "reference":
            run_reference(args, emit)
        else:
            run_ours(args, emit)
    if "line" in out:
        real_stdout.write(out["line"] + "\n")
        real_stdout.flush()


if __name__ == "__main__":
    main()
