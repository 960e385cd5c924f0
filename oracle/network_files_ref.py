"""fp64 / numpy oracle of csrc/material_metrics.cu: the ground-truth normalisation as MaterialVoxelDataset.__getitem__
writes it in numpy float32 (my_data.py:178-219), torch.argmax's rules and the per-sample counts and sums, accumulated in
fp64. network_files.batch_metrics turns the counts and sums into the reference's float32 metrics."""
from __future__ import annotations

import numpy as np


def normalize_gt(mat: np.ndarray, ranges) -> np.ndarray:
    """(D, D, D, C_mat) raw material grid -> (4, D, D, D) float32, the `mat_grid` save_predictions stores."""
    mat = mat.astype(np.float32)
    r = ranges

    def scale(x, lo, hi):
        x = np.clip(x, lo, hi)
        return 2.0 * (x - lo) / (hi - lo) - 1.0

    with np.errstate(divide="ignore", invalid="ignore"):
        d = scale(np.log10(mat[..., 0] + 1e-6), r["density_min"], r["density_max"])
        e = scale(np.log10(mat[..., 1] + 1e-6), r["E_min"], r["E_max"])
    nu = scale(mat[..., 2], r["nu_min"], r["nu_max"])
    ids = mat[..., -1].astype(np.int64).astype(np.float32)
    return np.stack([d, e, nu, ids]).astype(np.float32)


def argmax_torch(logits: np.ndarray) -> np.ndarray:
    """torch.argmax over axis 0: the first maximal index, and the first NaN when there is one."""
    nan = np.isnan(logits)
    idx = np.argmax(np.where(nan, -np.inf, logits), axis=0)
    any_nan = nan.any(axis=0)
    return np.where(any_nan, np.argmax(nan, axis=0), idx)


def sample_counts_sums(gt: np.ndarray, mask, logits: np.ndarray, cont: np.ndarray, background_id: int = 7):
    """One sample: (total, correct), (sum (cont_c - gt_c)^2 * mask for c < 3 in fp64 of the float32 products, sum mask)."""
    target = gt[3].astype(np.int64)
    m = (target != background_id).astype(np.float32) if mask is None else mask.astype(np.float32)
    on = m != 0
    pred = argmax_torch(logits)
    total, correct = int(on.sum()), int(((pred == target) & on).sum())
    with np.errstate(invalid="ignore", over="ignore"):
        d = (cont.astype(np.float32) - gt[:3]).astype(np.float32)
        terms = ((d * d).astype(np.float32) * m).astype(np.float32)
    sums = [float(np.sum(terms[c].astype(np.float64))) for c in range(3)] + [float(np.sum(m.astype(np.float64)))]
    return (total, correct), sums
