"""Per-frame 3DGS PLY export (pixie_b200.frame_export, csrc/gs_ply.cu):
  kernel     CUDA-event median of gaussian_ply_records at N = 100k and 1M Gaussians, K = 16 SH coefficients, with the
             bytes it must move (pos, cov, shs, opacity in; 248 B records out) over that time, against the H100 SXM
             data-sheet 3.35 TB/s
  rollout    per-frame wall time of one scene-driver rollout (N Gaussians, --substeps per frame) with save_ply off and on,
             alternating, from the first frame to the last file closed
  cpu_ref    for context, the CPU time of the reference's step at the same N: batched torch.linalg.eigh, the descending
             sort and handedness fix, scipy Rotation.from_matrix, and save_ply's per-vertex tuple packing
Prints the card's name and power limit and one JSON line.

    python scripts/profile_ply_export.py [--repeats 20] [--rollout-n 100000] [--frames 8] [--substeps 100]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch
from scipy.spatial.transform import Rotation

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pixie_b200 import frame_export as FE  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def gaussians(n, K, seed):
    rng = np.random.default_rng(seed)
    ev = 10.0 ** rng.uniform(-6, -3, size=(n, 3))
    Q = Rotation.random(n, random_state=seed).as_matrix()
    m = Q @ (ev[:, :, None] * np.eye(3)) @ Q.transpose(0, 2, 1)
    cov = np.stack([m[:, 0, 0], m[:, 0, 1], m[:, 0, 2], m[:, 1, 1], m[:, 1, 2], m[:, 2, 2]], axis=1).astype(np.float32)
    return (rng.uniform(-1, 1, (n, 3)).astype(np.float32), cov, (rng.standard_normal((n, K, 3)) * 0.4).astype(np.float32),
            rng.uniform(0, 1, n).astype(np.float32))


def timed(fn, repeats):
    fn()
    ms = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms))


def kernel(n, repeats):
    K = 16
    pos, cov, shs, opacity = [torch.from_numpy(a).cuda() for a in gaussians(n, K, 1)]
    ms = timed(lambda: FE.gaussian_ply_records(pos, cov, shs, opacity), repeats)
    nbytes = n * 4 * ((3 + 6 + 3 * K + 1) + (14 + 3 * K))
    return {"n": n, "K": K, "ms": ms, "bytes": nbytes, "GB_per_s": nbytes / ms / 1e6, "share_of_3.35TB_per_s": nbytes / (ms * 1e-3) / HBM_BYTES_PER_S}


def cpu_reference(n):
    """The reference's CPU step, restated: eigh, sort, clamp, handedness, scipy from_matrix, per-vertex tuples."""
    pos, cov, shs, opacity = gaussians(n, 16, 2)
    c = torch.from_numpy(cov)
    t0 = time.perf_counter()
    S = c[:, [0, 1, 2, 1, 3, 4, 2, 4, 5]].view(-1, 3, 3)
    evals, evecs = torch.linalg.eigh(S)
    idx = torch.argsort(evals, dim=1, descending=True)
    evals, evecs = evals.gather(1, idx), evecs.gather(2, idx.unsqueeze(1).expand(-1, 3, -1))
    log_s = torch.log(torch.sqrt(torch.clamp(evals, min=1e-12)))
    neg = torch.det(evecs) < 0
    evecs[neg, :, 2] *= -1
    t1 = time.perf_counter()
    q = Rotation.from_matrix(evecs.numpy()).as_quat()[:, [3, 0, 1, 2]]
    t2 = time.perf_counter()
    names = FE.gaussian_ply_attributes(16)
    attrs = np.concatenate([pos, np.zeros_like(pos), shs[:, 0], shs[:, 1:].transpose(0, 2, 1).reshape(n, -1), opacity[:, None],
                            log_s.numpy(), q], axis=1)
    el = np.empty(n, dtype=[(a, "f4") for a in names])
    el[:] = list(map(tuple, attrs))
    t3 = time.perf_counter()
    return {"n": n, "eigh_s": t1 - t0, "from_matrix_s": t2 - t1, "tuple_packing_s": t3 - t2, "total_s": t3 - t0,
            "threads": torch.get_num_threads()}


def rollout(n, frames, substeps, repeats):
    from oracle import unet_ref as O
    from pixie_b200 import material_transfer as MT
    from pixie_b200 import scene_driver as SD
    dev = "cuda:0"
    C, G = 64, 16
    seg, reg = O.build_pair(C, G, seed=3)
    drv = SD.SceneBatchDriver(feature_channels=C, grid_size=G, device=dev, seg_state_dict=seg.state_dict(), cont_state_dict=reg.state_dict(),
                              **O.DEFAULT_CFG)
    rng = np.random.default_rng(4)
    pred = np.zeros((11, G, G, G), np.float32)
    pred[:3] = rng.uniform(-0.2, 0.2, size=(3, G, G, G))
    pred[3 + rng.integers(0, 8, size=(G, G, G)), np.arange(G)[:, None, None], np.arange(G)[None, :, None], np.arange(G)[None, None, :]] = 1.0
    ranges = dict(density_min=2.95, density_max=3.05, E_min=4.4, E_max=4.6, nu_min=0.29, nu_max=0.31)
    cloud = MT.extract_material_points(torch.from_numpy(pred).to(dev), torch.ones((G, G, G)).to(dev), [-0.5] * 3, [0.5] * 3, ranges)
    pos, cov, shs, opacity = gaussians(n, 16, 5)
    pos = pos * 0.4
    sc = dict(name="obj", grid=None, mask=None, min_bounds=[-0.5] * 3, max_bounds=[0.5] * 3, particles=torch.from_numpy(pos),
              cov=torch.from_numpy(cov), opacity=torch.from_numpy(opacity), shs=torch.from_numpy(shs),
              material_params={"n_grid": 64, "grid_lim": 2.0, "material": "jelly", "g": [0.0, 0.0, -9.8], "density": 1000.0, "E": 1e5, "nu": 0.3},
              bc_params=[{"type": "bounding_box"}], time_params={"substep_dt": 1e-4, "frame_dt": substeps * 1e-4, "frame_num": frames},
              nn_distance_threshold=0.2)
    out = {"n": n, "frames": frames, "substeps_per_frame": substeps, "off_ms_per_frame": [], "on_ms_per_frame": []}
    with tempfile.TemporaryDirectory() as d:
        for r in range(repeats + 1):                     # the first pair warms up
            for save in (False, True):
                t = {}

                def on_frame(f, p, c):
                    if f == 0:
                        torch.cuda.synchronize()
                        t[0] = time.perf_counter()
                drv.run_physics_simulation(SD.Scene(**sc, save_ply=save), cloud, on_frame=on_frame, ply_dir=d if save else None)
                torch.cuda.synchronize()
                if r:
                    out["on_ms_per_frame" if save else "off_ms_per_frame"].append((time.perf_counter() - t[0]) * 1e3 / frames)
        out["ply_file_bytes"] = os.path.getsize(os.path.join(d, "frame_00000.ply"))
    for k in ("off_ms_per_frame", "on_ms_per_frame"):
        out[k + "_median"] = float(np.median(out[k]))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--rollout-n", type=int, default=100_000)
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--substeps", type=int, default=100)
    ap.add_argument("--rollout-repeats", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("profile_ply_export.py needs a CUDA device")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    out = {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": smi.stdout.strip()}
    print(f"card: {out['gpu']}  (name, power limit: {out['nvidia_smi']})", file=sys.stderr)
    out["kernel"] = [kernel(n, args.repeats) for n in (100_000, 1_000_000)]
    for k in out["kernel"]:
        print(f"records kernel N={k['n']}: {k['ms']:.3f} ms, {k['GB_per_s']:.0f} GB/s ({100 * k['share_of_3.35TB_per_s']:.0f} % of 3.35 TB/s)",
              file=sys.stderr)
    out["rollout"] = rollout(args.rollout_n, args.frames, args.substeps, args.rollout_repeats)
    r = out["rollout"]
    print(f"rollout N={r['n']}, {r['substeps_per_frame']} substeps/frame: {r['off_ms_per_frame_median']:.2f} ms/frame without save_ply, "
          f"{r['on_ms_per_frame_median']:.2f} with", file=sys.stderr)
    out["cpu_ref"] = [cpu_reference(n) for n in (100_000, 1_000_000)]
    for c in out["cpu_ref"]:
        print(f"reference CPU step N={c['n']}: eigh {c['eigh_s']:.3f} s, from_matrix {c['from_matrix_s']:.3f} s, "
              f"tuple packing {c['tuple_packing_s']:.3f} s ({c['threads']} threads)", file=sys.stderr)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
