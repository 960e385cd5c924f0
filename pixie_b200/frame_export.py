"""Either side of the MPM substep loop, on the device (SURVEY.md 8f-2).

    get_particle_volume(pos, grid_n, grid_dx, unifrom=False)      PG/particle_filling/filling.py:273-288 (Taichi in the reference)
    render_frame_transform(pos, cov, z_shift_value, scale_origin, original_mean_pos, rotation_matrices)
                                                                   PG/gs_simulation.py:591-600 + utils/transformation_utils.py
    cov3D_to_log_scales_and_quats(cov3D)                           PG/gs_simulation.py:253-288
    export_gaussians_to_ply(ply_out_dir, mpm_solver, ...)          PG/gs_simulation.py:290-322 + gaussian_model.py:177-208
    gaussian_ply_header(n, K), gaussian_ply_records(pos, cov, shs, opacity), PlyFrameWriter
                                                                   the PLY file those write, and its asynchronous writer
Same argument meaning as the reference (including its `unifrom` spelling). No CPU fallback.
"""
from __future__ import annotations

import concurrent.futures
import ctypes as C
import os
from typing import Optional, Sequence, Tuple

import torch

from . import _lib


def get_particle_volume(pos: torch.Tensor, grid_n: int, grid_dx: float, unifrom: bool = False) -> torch.Tensor:
    """vol[p] = grid_dx^3 / (number of particles in p's cell); with `unifrom` the mean volume for every particle (:282-285)."""
    _lib.require_device()
    if not pos.is_cuda:
        raise _lib.PixieError("get_particle_volume requires a CUDA tensor; there is no CPU fallback")
    p = pos.detach().reshape(-1, 3).to(torch.float32).contiguous()
    n = p.shape[0]
    vol = torch.empty(n, dtype=torch.float32, device=p.device)
    _lib.call("pixie_particle_volume", p.device, p, n, int(grid_n), float(grid_dx), vol)
    if unifrom:
        return torch.mean(vol).repeat(n)
    return vol


def render_frame_transform(pos: torch.Tensor, cov: Optional[torch.Tensor], z_shift_value: float, scale_origin, original_mean_pos,
                           rotation_matrices: Sequence[torch.Tensor]) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """(pos_render, cov3D_render) of gs_simulation.py:594-598: simulation frame -> the Gaussians' original frame."""
    _lib.require_device()
    _lib.require_cuda("render_frame_transform", pos)
    dev = pos.device
    p = pos.detach().reshape(-1, 3).to(torch.float32).contiguous()
    n = p.shape[0]
    c = None if cov is None else cov.detach().reshape(-1, 6).to(dev, torch.float32).contiguous()
    if c is not None and c.shape[0] != n:
        raise ValueError("pos and cov disagree on the particle count")
    scale = float(scale_origin.item() if torch.is_tensor(scale_origin) else scale_origin)
    mean = [float(v) for v in (original_mean_pos.detach().cpu().tolist() if torch.is_tensor(original_mean_pos) else original_mean_pos)]
    rots = [r.detach().to("cpu", torch.float32).reshape(9).tolist() for r in rotation_matrices]
    if len(rots) > 8:
        raise ValueError("at most 8 rotation matrices")
    flat = (C.c_float * max(1, 9 * len(rots)))(*[v for r in rots for v in r])
    po = torch.empty_like(p)
    co = None if c is None else torch.empty_like(c)
    _lib.call("pixie_frame_transform", dev, p, c, n, float(z_shift_value), scale, (C.c_float * 3)(*mean), flat, len(rots), po, co)
    return po, co


PLY_SH_COEFFS = (1, 4, 9, 16)


def gaussian_ply_attributes(K: int):
    """GaussianModel.construct_list_of_attributes (gaussian_model.py:177-189) for K SH coefficients per colour channel."""
    return (["x", "y", "z", "nx", "ny", "nz"] + [f"f_dc_{i}" for i in range(3)] + [f"f_rest_{i}" for i in range(3 * (K - 1))]
            + ["opacity"] + [f"scale_{i}" for i in range(3)] + [f"rot_{i}" for i in range(4)])


def gaussian_ply_header(n: int, K: int) -> bytes:
    """The header plyfile writes for save_ply's structured array of n vertices with K SH coefficients: `ply`, the binary
    little-endian format line, `element vertex n`, one `property float <name>` per attribute, `end_header`, each line
    ended by a newline. The n rows of 14 + 3K little-endian float32 follow it."""
    if K not in PLY_SH_COEFFS:
        raise ValueError(f"K must be one of {PLY_SH_COEFFS}, got {K}")
    lines = ["ply", "format binary_little_endian 1.0", f"element vertex {int(n)}"]
    lines += [f"property float {a}" for a in gaussian_ply_attributes(K)] + ["end_header"]
    return ("\n".join(lines) + "\n").encode("ascii")


def gaussian_ply_records(pos: torch.Tensor, cov: torch.Tensor, shs: torch.Tensor, opacity: torch.Tensor) -> torch.Tensor:
    """The (N, 14 + 3K) float32 PLY vertex rows of N Gaussians, on their device: pos (N, 3), cov (N, 6) upper triangle,
    shs (N, K, 3) with K in {1, 4, 9, 16}, opacity N values. Columns in gaussian_ply_attributes(K) order: pos, zero
    normals, shs[:, 0], shs[:, 1:] transposed to (3, K - 1) and flattened, opacity, the log scales and the (w, x, y, z)
    quaternion of cov3D_to_log_scales_and_quats. A covariance with a NaN or +-Inf entry gives NaN log scales and a NaN
    quaternion in its row; its other columns are copied as they are. One kernel, stream-ordered on the current stream."""
    _lib.require_device()
    _lib.require_cuda("gaussian_ply_records", pos)
    dev = pos.device
    p = pos.detach().reshape(-1, 3).to(torch.float32).contiguous()
    n = p.shape[0]
    c = cov.detach().reshape(-1, 6).to(dev, torch.float32).contiguous()
    s = shs.detach().to(dev, torch.float32).contiguous()
    o = opacity.detach().reshape(-1).to(dev, torch.float32).contiguous()
    if s.dim() != 3 or s.shape[2] != 3 or s.shape[1] not in PLY_SH_COEFFS:
        raise ValueError(f"shs must be (N, K, 3) with K in {PLY_SH_COEFFS}, got {tuple(s.shape)}")
    if c.shape[0] != n or s.shape[0] != n or o.shape[0] != n:
        raise ValueError(f"pos, cov, shs and opacity disagree on the Gaussian count ({n}, {c.shape[0]}, {s.shape[0]}, {o.shape[0]})")
    K = s.shape[1]
    rec = torch.empty((n, 14 + 3 * K), dtype=torch.float32, device=dev)
    _lib.call("pixie_gaussian_ply_records", dev, p, c, s, K, o, n, rec)
    return rec


def cov3D_to_log_scales_and_quats(cov3D: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """gs_simulation.py:253-288 on the device: (log_scales (N, 3), quats_wxyz (N, 4)) of (N, 6) upper-triangular
    covariances. The eigenvalues in descending order give log sqrt(max(lambda, 1e-12)) (a negative eigenvalue from
    rounding gives log 1e-6); the eigenvectors, as columns of R with the third negated when det R < 0, give the
    quaternion by scipy's Rotation.from_matrix, with scipy's sign (w is not forced >= 0). Both are float32: the
    reference returns float64 quaternions, but the PLY stores float32. The eigen-decomposition is a cyclic Jacobi in
    fp64; eigenvectors of equal eigenvalues are any orthonormal basis of their space, as with eigh."""
    if not cov3D.is_cuda:
        raise _lib.PixieError("cov3D_to_log_scales_and_quats requires a CUDA tensor; there is no CPU fallback")
    c = cov3D.detach().reshape(-1, 6)
    n, dev = c.shape[0], c.device
    rec = gaussian_ply_records(torch.zeros((n, 3), device=dev), c, torch.zeros((n, 1, 3), device=dev), torch.zeros(n, device=dev))
    return rec[:, 10:13].contiguous(), rec[:, 13:17].contiguous()


def _write_ply(path: str, header: bytes, rows) -> None:
    with open(path, "wb") as f:
        f.write(header)
        f.write(rows.numpy())                    # raw bytes, no copy; an empty frame writes the header alone


def export_gaussians_to_ply(ply_out_dir, mpm_solver, active_sh_degree, gs_num, scale_origin, rotation_matrices, opacity_render,
                            shs_render, frame, preprocessing_params, original_mean_pos, to_original_coord=True) -> str:
    """gs_simulation.py:290-322: writes the first gs_num particles of the solver as the 3DGS PLY
    `<ply_out_dir>/frame_{frame:05d}.ply` (returned) and returns once the file is closed. Kept as the reference has it:
      - `opacity` holds opacity_render as given; the reference passes post-sigmoid opacities (get_opacity), not logits;
      - with to_original_coord=False, the positions are the raw solver positions while the scales and rotations still
        come from the world-frame covariances apply_inverse_cov_rotations(cov / scale_origin^2, rotation_matrices);
      - only the first gs_num particles (and gs_num rows of opacity_render / shs_render) are written, K = shs_render's
        coefficient count whatever active_sh_degree is (save_ply does not read it).
    preprocessing_params needs "z_shift_value"."""
    x = mpm_solver.export_particle_x_to_torch()[:gs_num]
    cov_raw = mpm_solver.export_particle_cov_to_torch().view(-1, 6)[:gs_num]
    pr, cov_world = render_frame_transform(x, cov_raw, preprocessing_params["z_shift_value"], scale_origin, original_mean_pos,
                                           rotation_matrices)
    rec = gaussian_ply_records(pr if to_original_coord else x, cov_world, shs_render[:gs_num], opacity_render[:gs_num])
    os.makedirs(ply_out_dir, exist_ok=True)
    path = os.path.join(ply_out_dir, f"frame_{frame:05d}.ply")
    _write_ply(path, gaussian_ply_header(rec.shape[0], (rec.shape[1] - 14) // 3), rec.cpu())
    return path


class PlyFrameWriter:
    """Writes one 3DGS PLY per frame without holding up the device. submit() launches the record kernel on the current
    stream and returns: a side stream, ordered after the kernel by an event, copies the records into one of two pinned
    host buffers, and one background thread writes header + records to `<directory>/frame_{frame:05d}.ply`. So the
    current stream goes on with the next frame's work while the copy and the write run. At most two frames are in
    flight: submit() waits for the write that last used its buffer. A failed write is raised at the next submit() or at
    close(); close() returns when every submitted file is written and closed. Existing files are overwritten."""

    def __init__(self, directory: str, device=None):
        self.directory = directory
        os.makedirs(directory, exist_ok=True)
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self._copy_stream = torch.cuda.Stream(self.device)
        self._host = [None, None]
        self._pending = [None, None]
        self._slot = 0
        self._pool = concurrent.futures.ThreadPoolExecutor(max_workers=1, thread_name_prefix="ply-writer")

    @staticmethod
    def _write(path, header, rows, done, records):
        done.synchronize()                       # the copy has landed; `records` may be released from here on
        del records
        _write_ply(path, header, rows)

    def _take(self, slot):
        f, self._pending[slot] = self._pending[slot], None
        if f is not None:
            f.result()

    def submit(self, frame: int, pos: torch.Tensor, cov: torch.Tensor, shs: torch.Tensor, opacity: torch.Tensor) -> str:
        """Queue frame `frame`: gaussian_ply_records(pos, cov, shs, opacity) written to frame_{frame:05d}.ply."""
        for s in (0, 1):                         # an earlier write that failed
            if self._pending[s] is not None and self._pending[s].done():
                self._take(s)
        slot = self._slot
        self._slot ^= 1
        self._take(slot)
        with torch.cuda.device(self.device):
            records = gaussian_ply_records(pos, cov, shs, opacity)
            n, w = records.shape
            if self._host[slot] is None or self._host[slot].numel() < records.numel():
                self._host[slot] = torch.empty(max(1, records.numel()), dtype=torch.float32, pin_memory=True)
            rows = self._host[slot][:records.numel()].view(n, w)
            ready = torch.cuda.Event()
            ready.record()
            self._copy_stream.wait_event(ready)
            with torch.cuda.stream(self._copy_stream):
                rows.copy_(records, non_blocking=True)
                done = torch.cuda.Event()
                done.record(self._copy_stream)
        path = os.path.join(self.directory, f"frame_{frame:05d}.ply")
        self._pending[slot] = self._pool.submit(self._write, path, gaussian_ply_header(n, (w - 14) // 3), rows, done, records)
        return path

    def close(self) -> None:
        """Wait for every queued file; raise the first write error."""
        try:
            self._take(self._slot ^ 1)           # the older frame first
            self._take(self._slot)
        finally:
            for s in (0, 1):
                if self._pending[s] is not None:
                    self._pending[s].exception()
                    self._pending[s] = None
            self._pool.shutdown(wait=True)

    def __enter__(self):
        return self

    def __exit__(self, exc_type, exc, tb):
        if exc_type is None:
            self.close()
        else:
            try:
                self.close()
            except Exception:
                pass                             # the exception already propagating is the one to report
        return False
