"""Generates tests/golden/gaussian_ply_edges_golden.npz by EXECUTING THE REFERENCE'S OWN cov3D_to_log_scales_and_quats
(PhysGaussian's gs_simulation.py:253-288), pulled out with `ast` and run on CPU torch in float32 as in
make_gaussian_ply_golden.py (whose extraction helpers this reuses):

    PIXIE_REFERENCE=<checkout> python tests/golden/make_gaussian_ply_edges_golden.py

The reference's float32 eigh gives eigenvectors good to ~1e-7 lambda_max only, so this fixture pins what rounding
cannot move: quaternion signs of exact rotations and what happens to non-finite covariances. Cases:
  diag/*       diagonal covariances with three distinct variances in all 6 orderings, each with the off-diagonals +0,
               one of them -0.0 (each of the three in turn) and all three -0.0 (30 rows, one batch): the eigenvectors
               are a signed permutation, so the quaternion is exact
  nonfinite/*  one NaN, +Inf or -Inf in each of the six entries of a finite rotated covariance (18 rows), each row run
               on its own; `outcome` is "nan" when the reference returns (NaN log scales or quaternion), "eigh" or
               "from_matrix" when that step raises (outputs NaN then) and `error` the exception's class name
  versions     torch, numpy and scipy versions the outcomes were recorded with (they decide raise versus NaN)
A rerun reproduces the file byte for byte (fixed member time stamps).
"""
import io
import itertools
import os
import sys
import zipfile

import numpy as np
import scipy
import torch
from scipy.spatial.transform import Rotation

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_gaussian_ply_golden as G  # noqa: E402

VARIANCES = (3e-3, 4e-4, 1e-5)
NEG_ZERO_AT = ((), (1,), (2,), (4,), (1, 2, 4))                     # upper-triangle slots set to -0.0
BASE = np.array([4e-4, 1e-5, -2e-5, 3e-4, 5e-6, 1e-4], np.float32)   # SPD, every off-diagonal non-zero
NONFINITE = (np.nan, np.inf, -np.inf)


class _StagedRotation:
    """scipy's Rotation whose from_matrix notes that it was reached, to tell its errors from eigh's."""
    reached = False

    @classmethod
    def from_matrix(cls, R):
        cls.reached = True
        return Rotation.from_matrix(R)


def diagonal_rows():
    rows = []
    for perm in itertools.permutations(VARIANCES):
        for neg in NEG_ZERO_AT:
            u = np.zeros(6, np.float32)
            u[[0, 3, 5]] = perm
            u[list(neg)] = -0.0
            rows.append(u)
    return np.stack(rows)


def nonfinite_rows():
    rows = []
    for j in range(6):
        for v in NONFINITE:
            u = BASE.copy()
            u[j] = v
            rows.append(u)
    return np.stack(rows)


def save_npz(path, blob):
    """np.savez_compressed with a fixed time stamp on every member, so that a rerun reproduces the file byte for byte."""
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as z:
        for k, v in blob.items():
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(v), allow_pickle=False)
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, buf.getvalue())


def main():
    ns = G.namespace()
    ns["scipy_R"] = _StagedRotation
    f = ns["cov3D_to_log_scales_and_quats"]
    out = {}

    cov = diagonal_rows()
    ls, q = f(torch.from_numpy(cov.copy()))
    out["diag/cov"], out["diag/log_scales"], out["diag/quats"] = cov, ls.numpy(), q.numpy()

    cov = nonfinite_rows()
    ls_all, q_all = np.full((len(cov), 3), np.nan, np.float32), np.full((len(cov), 4), np.nan, np.float64)
    outcome, error = [], []
    for i, u in enumerate(cov):
        _StagedRotation.reached = False
        try:
            ls, q = f(torch.from_numpy(u[None].copy()))
        except Exception as e:                                          # eigh or from_matrix rejected the matrix
            outcome.append("from_matrix" if _StagedRotation.reached else "eigh")
            error.append(type(e).__name__)
            continue
        ls_all[i], q_all[i] = ls.numpy()[0], q.numpy()[0]
        outcome.append("nan" if np.isnan(ls_all[i]).any() or np.isnan(q_all[i]).any() else "finite")
        error.append("")
    out.update({"nonfinite/cov": cov, "nonfinite/log_scales": ls_all, "nonfinite/quats": q_all,
                "nonfinite/outcome": np.array(outcome), "nonfinite/error": np.array(error),
                "versions": np.array([f"torch {torch.__version__}", f"numpy {np.__version__}", f"scipy {scipy.__version__}"])})
    path = os.path.join(HERE, "gaussian_ply_edges_golden.npz")
    save_npz(path, out)
    print(f"wrote {path}: {len(out)} arrays; non-finite outcomes {dict(zip(*np.unique(outcome, return_counts=True)))}")


if __name__ == "__main__":
    main()
