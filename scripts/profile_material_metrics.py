"""Evaluation-metric pass (pixie_b200.network_files.material_metrics, csrc/material_metrics.cu) at 64^3, N = 1 and 4:
  kernel   pixie_material_metrics alone (both kernels, CUDA events over --iters launches), with the bytes it must move
           (raw grid 16 B, mask 4 B, 8 logits 32 B, 3 predictions 12 B in, 16 B of gt out, per voxel) over its time,
           against the H100 SXM data-sheet 3.35 TB/s
  ref      for context, the reference's path restated on the same batch: numpy normalisation of each material_grid
           (MaterialVoxelDataset.__getitem__), the H2D copy, and process_batch's compute_accuracy / masked_mean torch
           expressions on the device (host clock around a synchronised call)
  ours     material_metrics + batch_metrics end to end from the device inputs (host clock around a synchronised call)
Prints the card's name and power limit and one JSON line; writes it to --out when given.

    python scripts/profile_material_metrics.py [--iters 200] [--out file.json]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import network_files_ref as O  # noqa: E402
from pixie_b200 import _lib  # noqa: E402
from pixie_b200 import network_files as NF  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
RANGES = {"density_min": 1.7031893730163574, "density_max": 3.871432304382324, "E_min": 3.0183002948760986, "E_max": 10.881680488586426,
          "nu_min": 0.21027633547782898, "nu_max": 0.4492689371109009}


def inputs(n, D, seed):
    rng = np.random.default_rng(seed)
    mat = np.zeros((n, D, D, D, 4), np.float32)
    mat[..., 0] = 10.0 ** rng.uniform(1.0, 4.5, mat.shape[:-1])
    mat[..., 1] = 10.0 ** rng.uniform(2.5, 11.5, mat.shape[:-1])
    mat[..., 2] = rng.uniform(0.15, 0.5, mat.shape[:-1])
    mat[..., 3] = rng.integers(0, 8, mat.shape[:-1])
    mask = (mat[..., 3] != 7).astype(np.float32)
    logits = rng.standard_normal((n, 8, D, D, D), dtype=np.float32)
    cont = rng.uniform(-1, 1, (n, 3, D, D, D)).astype(np.float32)
    return mat, mask, logits, cont


def reference_path(mat_h, mask_h, seg, cont, dev):
    gts = np.stack([O.normalize_gt(m, RANGES) for m in mat_h])
    gt = torch.from_numpy(gts).to(dev)
    mat_id = gt[:, 3].long()
    mask = torch.from_numpy(mask_h).to(dev)
    pred = seg.argmax(1)
    m = mask.bool()
    acc = ((pred == mat_id) & m).sum().float() / m.sum().float()
    fg = mask.unsqueeze(1)
    diff_sq = (cont - gt[:, :3]) ** 2
    num = (diff_sq * fg).sum((2, 3, 4))
    mse = num / (fg.sum((2, 3, 4)).clamp(min=1) + 1e-8)
    out = [acc.item(), mse.mean().item()]
    for i in range(len(mat_h)):
        out.append(mse[i].tolist())
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    lib = _lib.require_device()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"[gpu] {q}")
    D = 64
    res = {"gpu": q, "D": D}
    for n in (1, 4):
        mat_h, mask_h, seg_h, cont_h = inputs(n, D, n)
        mat, mask, seg, cont = (torch.from_numpy(a).to(dev) for a in (mat_h, mask_h, seg_h, cont_h))
        gt = torch.empty((n, 4, D, D, D), dtype=torch.float32, device=dev)
        counts = torch.empty((n, 2), dtype=torch.int64, device=dev)
        sums = torch.empty((n, 4), dtype=torch.float64, device=dev)
        rng = (C.c_double * 6)(*[RANGES[k] for k in ("density_min", "density_max", "E_min", "E_max", "nu_min", "nu_max")])
        st = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        p = lambda t: C.c_void_p(t.data_ptr())                                          # noqa: E731
        call = lambda: _lib.check(lib.pixie_material_metrics(p(mat), 4, p(mask), p(seg), 8, p(cont), n, D ** 3, rng, 7, p(gt), p(counts), p(sums), st))  # noqa: E731
        for _ in range(20):
            call()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.iters):
            call()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.iters
        nbytes = n * D ** 3 * (16 + 4 + 32 + 12 + 16)

        def timed(fn, reps=10):
            fn()
            torch.cuda.synchronize()
            ts = []
            for _ in range(reps):
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                ts.append(time.perf_counter() - t0)
            return float(np.median(ts)) * 1e3

        ours = timed(lambda: NF.batch_metrics(*NF.material_metrics(mat, mask, seg, cont, RANGES, 7)[1:]))
        ref = timed(lambda: reference_path(mat_h, mask_h, seg, cont, dev))
        res[f"n{n}"] = {"kernel_ms": ms, "bytes": nbytes, "GBps": nbytes / ms / 1e6, "hbm_share": nbytes / (ms * 1e-3) / HBM_BYTES_PER_S,
                        "ours_ms": ours, "ref_ms": ref}
        print(f"[N={n}] kernel {ms:.4f} ms, {nbytes / 1e6:.1f} MB, {nbytes / ms / 1e6:.0f} GB/s "
              f"({100 * nbytes / (ms * 1e-3) / HBM_BYTES_PER_S:.0f}% of 3.35 TB/s); end to end {ours:.2f} ms vs reference path {ref:.2f} ms")
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f)


if __name__ == "__main__":
    main()
