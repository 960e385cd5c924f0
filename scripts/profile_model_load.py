"""Trained-checkpoint decode (pixie_b200.scene_files, csrc/gs_load.cu) on K = 16 checkpoints of 300k / 1M / 3M Gaussians:
  read        file -> pinned host buffer (host clock; the page cache is warm after the first repeat)
  h2d         the one pinned H2D copy of the vertex table (CUDA events)
  kernel      pixie_gaussian_checkpoint_decode without and with the 0.02 opacity filter (CUDA events; the filtered call
              includes its count pass, scan and one host sync), with the bytes it must move (the 248 B rows in; pos, shs,
              opacity, cov out) over the unfiltered time, against the H100 SXM data-sheet 3.35 TB/s
  load        load_gaussians end to end (file to filtered device tensors; host clock around a synchronised call)
  ref         for context, the reference's path restated on the same file: numpy column extraction as load_ply does
              it (float64 staging), torch.tensor(..., device="cuda") per array, then sigmoid / exp / build_rotation /
              L L^T and the mask on the device (host clock around a synchronised call)
Medians over --repeats. Prints the card's name and power limit and one JSON line; writes it to --out when given.

    python scripts/profile_model_load.py [--repeats 10] [--sizes 300000,1000000,3000000] [--out file.json]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import gaussian_model_ref as GM  # noqa: E402
from pixie_b200 import _lib  # noqa: E402
from pixie_b200 import scene_files as SF  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
K = 16


def write_checkpoint(path, n, seed):
    names = ["x", "y", "z", "nx", "ny", "nz", "f_dc_0", "f_dc_1", "f_dc_2"] + [f"f_rest_{i}" for i in range(3 * K - 3)] + \
            ["opacity", "scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3"]
    rng = np.random.default_rng(seed)
    a = rng.standard_normal((n, len(names)), dtype=np.float32)
    a[:, names.index("opacity")] = rng.normal(-1.0, 2.5, n)
    a[:, names.index("scale_0"):names.index("scale_2") + 1] = rng.uniform(-7, -3, (n, 3))
    head = "ply\nformat binary_little_endian 1.0\n" + f"element vertex {n}\n" + "".join(f"property float {nm}\n" for nm in names) + "end_header\n"
    with open(path, "wb") as f:
        f.write(head.encode())
        f.write(a.tobytes())


def reference_path(path, dev):
    """load_ply's column extraction + the reference's torch activations, get_covariance and the :405 mask."""
    rows = SF.read_ply(path).read()
    xyz = np.stack((np.asarray(rows["x"]), np.asarray(rows["y"]), np.asarray(rows["z"])), axis=1)
    opac = np.asarray(rows["opacity"])[..., np.newaxis]
    dc = np.zeros((len(rows), 3, 1))
    for c in range(3):
        dc[:, c, 0] = rows[f"f_dc_{c}"]
    rest = np.zeros((len(rows), 3 * K - 3))
    for i in range(3 * K - 3):
        rest[:, i] = rows[f"f_rest_{i}"]
    scale = np.zeros((len(rows), 3))
    for i in range(3):
        scale[:, i] = rows[f"scale_{i}"]
    rot = np.zeros((len(rows), 4))
    for i in range(4):
        rot[:, i] = rows[f"rot_{i}"]
    raw = {"xyz": xyz, "f_dc": dc[:, :, 0], "f_rest": rest, "opacity": opac[:, 0], "scale": scale, "rot": rot}
    out = GM.torch_reference(raw, dev)
    mask = out["opacity"][:, 0] > 0.02
    return {k: v[mask] for k, v in out.items() if k != "L"}


def median_ms(xs):
    return float(np.median(xs))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--sizes", default="300000,1000000,3000000")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    lib = _lib.require_device()
    stream = torch.cuda.current_stream(dev)
    results = {}
    with tempfile.TemporaryDirectory() as d:
        for n in [int(s) for s in args.sizes.split(",")]:
            path = os.path.join(d, f"ckpt_{n}.ply")
            write_checkpoint(path, n, n)
            el = SF.read_ply(path)
            cols = SF._checkpoint_columns(el, K)
            stride = el.dtype.itemsize
            host = torch.empty(n * stride, dtype=torch.uint8, pin_memory=True)
            table = torch.empty(n * stride, dtype=torch.uint8, device=dev)
            outs = [torch.empty((n, w), dtype=torch.float32, device=dev) for w in (3, 3 * K, 1, 6)]
            m = C.c_longlong(0)

            def decode(threshold):
                _lib.check(lib.pixie_gaussian_checkpoint_decode(C.c_void_p(table.data_ptr()), n, stride, (C.c_int * len(cols))(*cols), K,
                                                                int(threshold is not None), 0.0 if threshold is None else float(np.float32(threshold)),
                                                                *[C.c_void_p(o.data_ptr()) for o in outs], C.byref(m), C.c_void_p(stream.cuda_stream)))

            t_read, t_h2d, t_k, t_kf, t_load, t_ref = [], [], [], [], [], []
            for rep in range(args.repeats + 1):
                t0 = time.perf_counter()
                with open(path, "rb") as f:
                    f.seek(el.data_offset)
                    f.readinto(memoryview(host.numpy()))
                t_read.append((time.perf_counter() - t0) * 1e3)
                e = [torch.cuda.Event(enable_timing=True) for _ in range(6)]
                e[0].record()
                table.copy_(host, non_blocking=True)
                e[1].record()
                e[2].record()
                decode(None)
                e[3].record()
                e[4].record()
                decode(0.02)
                e[5].record()
                torch.cuda.synchronize()
                t_h2d.append(e[0].elapsed_time(e[1]))
                t_k.append(e[2].elapsed_time(e[3]))
                t_kf.append(e[4].elapsed_time(e[5]))
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                g = SF.decode_checkpoint_ply(path, 3, 0.02, dev)
                torch.cuda.synchronize()
                t_load.append((time.perf_counter() - t0) * 1e3)
                t0 = time.perf_counter()
                r = reference_path(path, dev)
                torch.cuda.synchronize()
                t_ref.append((time.perf_counter() - t0) * 1e3)
                if rep == 0:
                    assert torch.equal(g["pos"], r["pos"]) and torch.equal(g["shs"], r["shs"]) and torch.equal(g["opacity"], r["opacity"])
                    t_read, t_h2d, t_k, t_kf, t_load, t_ref = [], [], [], [], [], []          # first pass is warm-up
            moved = n * stride + n * 4 * (3 + 3 * K + 1 + 6)
            results[n] = {"read_ms": median_ms(t_read), "h2d_ms": median_ms(t_h2d), "kernel_ms": median_ms(t_k),
                          "kernel_filtered_ms": median_ms(t_kf), "load_gaussians_ms": median_ms(t_load), "reference_path_ms": median_ms(t_ref),
                          "kernel_bytes": moved, "kernel_TBps": moved / (median_ms(t_k) * 1e-3) / 1e12,
                          "kernel_share_of_3.35TBps": moved / (median_ms(t_k) * 1e-3) / HBM_BYTES_PER_S, "kept": int(m.value)}
            print(f"N={n}: {json.dumps(results[n])}", file=sys.stderr)
            del host, table, outs
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    out = {"gpu": torch.cuda.get_device_name(dev), "nvidia_smi": smi.stdout.strip(), "K": K, "repeats": args.repeats, "sizes": results}
    print(f"card: {out['gpu']}  (name, power limit: {out['nvidia_smi']})", file=sys.stderr)
    print(json.dumps(out))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
