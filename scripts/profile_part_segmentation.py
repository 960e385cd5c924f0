"""VLM part segmentation (pixie_b200.segmentation) on the device:
  similarity  pixie_part_similarity at 64^3 x 768, P = 8 and 64, at 5 %, 30 % and 100 % occupancy: the call (CUDA-event
              median over --iters calls, host work included) and the similarity kernel alone (its mean device time under
              torch.profiler, a separate run). Bytes: the occupied rows' fp16 features, the mask, and the similarities,
              probabilities, labels and scores written; over the kernel time, against the H100 SXM data-sheet 3.35 TB/s
  torch       for context, run_clip's own expressions on the same device from the same device grid: the masked gather,
              the fp32 copy, the normalisation, the matmul and the softmax, then argmax and gather (CUDA-event median)
  vote        pixie_knn_label_vote at k = 200 on N ~ 20k, 100k and 262k voxels of a solid lattice block and of a
              one-voxel-thick spherical lattice shell (CUDA-event median of the call, and the vote kernel alone as above)
  cli         `python -m pixie_b200.segmentation` end to end (main(), host clock) on a 64^3 x 768 grid at 10 % occupancy,
              P = 8, with and without --use_spatial_smoothing, against the reference's path restated on the same machine
              (np.load, torch fp32 run_clip on the device, the per-voxel scikit-learn KDTree + scipy mode loop, the cKDTree
              colour lookup and the numpy writer of oracle/segmentation_ref.py)
Prints the card's name and power limit and one JSON line; writes it to --out when given.

    python scripts/profile_part_segmentation.py [--iters 20] [--out file.json]
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import segmentation_ref as O  # noqa: E402
from pixie_b200 import segmentation as S  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
DEV = "cuda:0"


def median_ms(fn, iters):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def kernel_ms(fn, name, reps=10):
    """Mean device time per call of the kernels whose name contains `name`, under torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    return sum(e.device_time for e in prof.events() if e.device_type.name == "CUDA" and name in e.name) / reps / 1e3


def grid(D, C, P, occ, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    feats = torch.randn((D, D, D, C), generator=g, device=DEV).half()
    mask = torch.rand((D, D, D), generator=g, device=DEV) < occ
    q = torch.randn((P, C), generator=g, device=DEV)
    return feats, mask, q


def torch_run_clip(feats, mask, q, T=0.1):
    f = feats.reshape(-1, feats.shape[-1])[mask.reshape(-1)].to(torch.float32)
    f /= f.norm(dim=-1, keepdim=True)
    qq = q.float()
    qq /= qq.norm(dim=-1, keepdim=True)
    probs = torch.softmax((f @ qq.T) / T, dim=1)
    labels = torch.argmax(probs, dim=1)
    return probs, torch.gather(probs, 1, labels[:, None])[:, 0]


def profile_similarity(iters):
    out = []
    D, C = 64, 768
    for P in (8, 64):
        for occ in (0.05, 0.30, 1.0):
            feats, mask, q = grid(D, C, P, occ, seed=int(occ * 100) + P)
            n = int(mask.sum())
            uq = S.normalize_queries(q, DEV)
            call = lambda: S.part_similarity(feats, uq, 0.1, mask=mask, n_occupied=n)      # noqa: E731
            ms = median_ms(call, iters)
            kms = kernel_ms(call, "similarity_kernel")
            bytes_ = n * C * 2 + D ** 3 + n * (2 * P * 4 + 12)
            ms_t = median_ms(lambda: torch_run_clip(feats, mask, q), iters)
            out.append({"P": P, "occupancy": occ, "n": n, "call_ms": round(ms, 4), "kernel_ms": round(kms, 4), "bytes": bytes_,
                        "tb_per_s": round(bytes_ / kms / 1e9, 3), "share_of_3.35TB/s": round(bytes_ / (kms * 1e-3) / HBM_BYTES_PER_S, 3),
                        "torch_run_clip_call_ms": round(ms_t, 4)})
            print(json.dumps(out[-1]), flush=True)
            del feats, mask
    return out


def lattice_points(kind, n_target):
    if kind == "solid":
        D = int(round(n_target ** (1 / 3)))
        m = np.ones((D, D, D), bool)
    else:
        R = np.sqrt(n_target / (4 * np.pi))
        D = int(2 * R + 4)
        a = (np.arange(D) - (D - 1) / 2) ** 2
        m = np.abs(np.sqrt(a[:, None, None] + a[None, :, None] + a[None, None, :]) - R) < 0.5
    axes = [torch.linspace(-1.0, 1.0, D) for _ in range(3)]
    g = torch.stack(torch.meshgrid(*axes, indexing="ij"), -1)
    return g[torch.from_numpy(m)].to(DEV)


def profile_vote(iters):
    out = []
    rng = np.random.default_rng(0)
    for kind in ("solid", "shell"):
        for n_target in (20_000, 100_000, 262_144):
            pts = lattice_points(kind, n_target)
            labels = torch.from_numpy(rng.integers(0, 8, len(pts))).to(DEV)
            call = lambda: S.knn_label_vote(pts, labels, 200)          # noqa: E731
            ms = median_ms(call, max(3, iters // 4))
            kms = kernel_ms(call, "knn_vote_kernel", 3)
            out.append({"kind": kind, "n": len(pts), "k": 200, "call_ms": round(ms, 3), "vote_kernel_ms": round(kms, 3)})
            print(json.dumps(out[-1]), flush=True)
    return out


def write_case(d, D, C, P, occ, seed):
    rng = np.random.default_rng(seed)
    os.makedirs(d, exist_ok=True)
    table = rng.normal(0, 1, (P, C)).astype(np.float32)
    mask = rng.uniform(size=(D, D, D)) < occ
    part = rng.integers(0, P, (D, D, D))
    feats = np.empty((D, D, D, C), np.float16)
    for x in range(D):
        feats[x] = (2.0 * table[part[x]] + rng.standard_normal((D, D, C), dtype=np.float32)).astype(np.float16)
    lo, hi = np.array([-0.5] * 3, np.float32), np.array([0.5] * 3, np.float32)
    np.savez(os.path.join(d, "clip_features.npz"), min_bounds=lo, max_bounds=hi, grid_shape=np.array([D] * 3))
    np.save(os.path.join(d, "clip_features_features.npy"), feats)
    np.save(os.path.join(d, "clip_features_mask.npy"), mask.astype(np.float32))
    axes = [torch.linspace(-0.5, 0.5, D).numpy() for _ in range(3)]
    idx = np.argwhere(mask)
    verts = np.stack([axes[a][idx[:, a]] for a in range(3)], 1).astype(np.float64)
    cols = rng.integers(0, 256, (len(verts), 3)).astype(np.uint8)
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import make_segmentation_golden as G
    with open(os.path.join(d, "occupancy.ply"), "wb") as f:
        f.write(G.ply_bytes(verts, cols))
    props = {f"part {i}": {"density": 100.0 + i, "E": 1e5 * (i + 1), "nu": 0.3, "material_id": i % 7} for i in range(P)}
    json.dump(props, open(os.path.join(d, "materials.json"), "w"))
    np.save(os.path.join(d, "q.npy"), table)
    return table, verts, np.column_stack([cols, np.full(len(cols), 255, np.uint8)]), props, mask


def reference_cli(d, table, verts, cols, props, mask, smooth):
    """The reference's __main__ path restated on this machine (its own expressions and libraries)."""
    from scipy.stats import mode
    from sklearn.neighbors import KDTree
    feats = np.load(os.path.join(d, "clip_features_features.npy"))
    D = mask.shape[0]
    axes = [torch.linspace(-0.5, 0.5, D, device=DEV) for _ in range(3)]
    coords = torch.stack(torch.meshgrid(*axes, indexing="ij"), -1)[torch.from_numpy(mask).to(DEV)]
    f = torch.from_numpy(feats).to(DEV).reshape(-1, feats.shape[-1])[torch.from_numpy(mask.reshape(-1)).to(DEV)]
    f = f.to(torch.float32)
    f /= f.norm(dim=-1, keepdim=True)
    q = torch.from_numpy(table).to(DEV).float()
    q /= q.norm(dim=-1, keepdim=True)
    probs = torch.softmax((f @ q.T) / 0.1, dim=1)
    labels = torch.argmax(probs, dim=1)
    if smooth:
        c = coords.cpu().numpy()
        lab = labels.cpu().numpy()
        tree = KDTree(c)
        new = lab.copy()
        for i, p in enumerate(c):
            _, ind = tree.query(p.reshape(1, -1), k=200)
            new[i] = mode(lab[ind[0]], keepdims=False).mode
        labels = torch.tensor(new, device=DEV)
    od = os.path.join(d, "ref_out")
    np.save(os.path.join(d, "ref_labels.npy"), labels.cpu().numpy())
    O.save_files(coords.cpu().numpy(), labels.cpu().numpy(), od, verts, cols, list(props), props, mask.shape, mask)


def profile_cli():
    out = []
    with tempfile.TemporaryDirectory() as d:
        table, verts, cols, props, mask = write_case(d, 64, 768, 8, 0.10, seed=1)
        for smooth in (False, True):
            argv = ["--grid_feature_path", os.path.join(d, "clip_features.npz"), "--occupancy_path", os.path.join(d, "occupancy.ply"),
                    "--output_dir", os.path.join(d, "out"), "--material_dict_path", os.path.join(d, "materials.json"),
                    "--query_embeddings", os.path.join(d, "q.npy"), "--overwrite", "true", "--use_spatial_smoothing", str(smooth)]
            S.main(argv)                                     # warm-up: module loads
            ts = []
            for _ in range(3):
                torch.cuda.synchronize()
                t = time.perf_counter()
                S.main(argv)
                torch.cuda.synchronize()
                ts.append((time.perf_counter() - t) * 1e3)
            try:
                reference_cli(d, table, verts, cols, props, mask, False)      # warm-up
                torch.cuda.synchronize()
                t = time.perf_counter()
                reference_cli(d, table, verts, cols, props, mask, smooth)
                torch.cuda.synchronize()
                ref_ms = round((time.perf_counter() - t) * 1e3, 1)
            except ImportError as e:
                ref_ms = f"not measured ({e})"
            out.append({"n": int(mask.sum()), "smoothing": smooth, "cli_ms": round(float(np.median(ts)), 1), "reference_path_ms": ref_ms})
            print(json.dumps(out[-1]), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    ap.add_argument("--skip_cli", action="store_true")
    a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"[card] {q}", flush=True)
    res = {"card": q, "similarity": profile_similarity(a.iters), "vote": profile_vote(a.iters)}
    if not a.skip_cli:
        res["cli"] = profile_cli()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
