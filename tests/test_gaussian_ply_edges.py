"""The 3DGS PLY export at its edges: flat Gaussians (disks and needles down to 1e-14 variance ratios), every magnitude,
exact rotations, non-finite covariances, bit-exact copies and PlyFrameWriter's frame sequences. CPU: the fp64 oracle
against tests/golden/gaussian_ply_edges_golden.npz (the reference's own function, make_gaussian_ply_edges_golden.py)
and under power-of-two scaling; GPU: the record kernel against the oracle and the fixture.

Bounds against the fp64 oracle (oracle/gaussian_ply_ref.py: numpy eigh of the float32 matrix as given), per component:
  log scales   |ls - ls_ref| <= 2 ulp32(ls_ref) + LS_C 2^-52 lambda_max / lambda_ref where lambda_ref >= 2^-30 lambda_max
               and lambda_ref is clear of the clamp by the eigenvalue error LAM_C 2^-52 lambda_max; both eigen-solvers
               are backward stable in fp64, so an eigenvalue moves by a small multiple of 2^-52 lambda_max
  clamp        lambda_ref below 1e-12 by that margin: ls is float32(log(1e-6)) bit for bit
  directions   eigenvector i whose gap to both neighbours is >= 2^-20 lambda_max: sin(angle to the oracle's) <= ANGLE_TOL
               (fp64 error 2^-52 lambda_max / gap <= 2^-32; the rest is the float32 quaternion)
Scaling the covariance by 2^k (no underflow) scales every Jacobi step, the sort and Markley's decision exactly, so the
quaternion must be bit-identical and the log scales shift by k/2 ln 2 to float32 rounding. Non-finite convention: a row
with a NaN or +-Inf covariance entry gets NaN log scales and quaternion; everything else is as if it were finite.
"""
import os
import sys

import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import gaussian_ply_ref as R  # noqa: E402
from test_gaussian_ply import _dev, check_against_oracle, degenerate_covs, random_inputs, read_ply  # noqa: E402

F32, U32 = np.float32, np.uint32
CLAMP32 = F32(np.log(np.sqrt(1e-12)))
EPS64 = 2.0 ** -52
LS_C = 0.0              # measured 0 on one H100 80GB HBM3 (700 W): the largest log-scale error was 0.51 ulp32
LAM_C = 64.0            # the band around the clamp where neither the clamp nor the log-scale bound is asserted
ANGLE_TOL = 3.4e-7      # 4x the 8.5e-8 measured on one H100 (flat cases); float32 quaternions round at ~6e-8
LS_FLOOR, GAP_FLOOR = 2.0 ** -30, 2.0 ** -20
RATIOS = [10.0 ** -e for e in range(2, 15, 2)]
GAPS = [10.0 ** -e for e in range(3, 10)]
KS = list(range(-40, 41, 2))
FLT_MIN = float(np.finfo(F32).tiny)
# -0.0, the smallest subnormals of both signs, the largest subnormal, quiet and signalling NaNs with payloads, +-Inf
SPECIAL_BITS = np.array([0x80000000, 0x00000001, 0x80000001, 0x007FFFFF, 0x7FC00001, 0xFFC12345, 0x7F800001, 0xFFBFFFFF,
                         0x7F800000, 0xFF800000], U32)


@pytest.fixture(scope="module")
def edges():
    return dict(np.load(os.path.join(ROOT, "tests", "golden", "gaussian_ply_edges_golden.npz")))


def upper(m):
    return np.stack([m[..., 0, 0], m[..., 0, 1], m[..., 0, 2], m[..., 1, 1], m[..., 1, 2], m[..., 2, 2]], axis=-1)


def from_eigs(lam, Q):
    """float32 upper triangles of Q diag(lam) Q^T, formed in fp64."""
    return upper(Q @ (np.asarray(lam, np.float64)[:, :, None] * np.eye(3)) @ Q.transpose(0, 2, 1)).astype(F32)


PERMS = [(0, 1, 2), (0, 2, 1), (1, 0, 2), (1, 2, 0), (2, 0, 1), (2, 1, 0)]


def axis_aligned(lam):
    """Diagonal covariances of the rows of lam in all 6 orderings."""
    lam = np.asarray(lam, np.float64)
    out = np.zeros((len(lam) * 6, 6), F32)
    for i, p in enumerate(PERMS):
        out[i::6][:, [0, 3, 5]] = lam[:, list(p)]
    return out


def flat_covs(seed, n_rot=40):
    """Disks (lambda0 ~ lambda1 >> lambda2) and needles (lambda0 >> lambda1 ~ lambda2) at every ratio in RATIOS, rotated
    and axis-aligned, and near-degenerate pairs at relative gaps GAPS, at scales 1e-6 .. 1e-2."""
    rng = np.random.default_rng(seed)
    rows = []
    for r in RATIOS:
        s = 10.0 ** rng.uniform(-6, -2, size=(n_rot, 1))
        u = rng.uniform(0, 0.3, size=(n_rot, 1))
        disk, needle = s * np.hstack([np.ones_like(u), 1 - u, np.full_like(u, r)]), s * np.hstack([np.ones_like(u), r * (1 + u), np.full_like(u, r)])
        for lam in (disk, needle):
            rows += [from_eigs(lam, Rotation.random(n_rot, random_state=rng).as_matrix()), axis_aligned(lam[:2])]
    for g in GAPS:
        s = 10.0 ** rng.uniform(-6, -2, size=(10, 1))
        for lam in (s * [1, 1 - g, 0.1], s * [1, 0.3, 0.3 * (1 - g)], s * [1, 1 - g, 1e-6], s * [1, 1e-6 * (1 + g), 1e-6]):
            rows += [from_eigs(lam, Rotation.random(10, random_state=rng).as_matrix()), axis_aligned(lam[:1])]
    return np.concatenate(rows)


def extreme_covs(seed):
    """Background-sized variances 1e2 .. 1e6, covariances near FLT_MAX, and eigenvalues at 1e-12 (1 +- 2^-20)."""
    rng = np.random.default_rng(seed)
    big = 10.0 ** rng.uniform(2, 6, size=(60, 3))
    big[:20, 2] = big[:20, 0] * 1e-6                                      # flat background splats too
    huge = rng.uniform(1e37, 3e38, size=(30, 1)) * np.hstack([np.ones((30, 1)), 10.0 ** rng.uniform(-8, 0, size=(30, 2))])
    near = 1e-12 * np.array([[4.0, 1 + 2.0 ** -20, 1 - 2.0 ** -20], [1 + 2.0 ** -20, 1 - 2.0 ** -20, 0.5],
                             [2.0, 1.0, 1 - 2.0 ** -20]])
    rot = Rotation.random(90 + 12, random_state=rng).as_matrix()
    return np.concatenate([from_eigs(big, rot[:60]), from_eigs(huge, rot[60:90]), from_eigs(np.repeat(near, 4, axis=0), rot[90:]),
                           axis_aligned(big[:4]), axis_aligned(huge[:4] / 2), axis_aligned(near)])


def near_half_turns():
    """Rotations by pi - delta about the axes and three oblique axes, of distinct variances: w ~ 0, so Markley's x, y or
    z branch builds the quaternion."""
    axes = np.array([[1, 0, 0], [0, 1, 0], [0, 0, 1], [1, 1, 0], [1, 1, 1], [1, -2, 0.5]], np.float64)
    axes /= np.linalg.norm(axes, axis=1, keepdims=True)
    rv = np.array([a * (np.pi - d) for a in axes for d in (0.0, 1e-7, 1e-5, 1e-3, 1e-1)])
    Q = Rotation.from_rotvec(rv).as_matrix()
    return from_eigs(np.tile([3e-3, 4e-4, 1e-5], (len(Q), 1)), Q)


def tied_covs():
    """Equal eigenvalues, whose eigenvectors are any basis of their space: held by the rebuild only."""
    Q = Rotation.random(4, random_state=11).as_matrix()
    lam = np.array([[5e-4, 5e-4, 2e-6], [5e-4, 2e-6, 2e-6], [3e-4, 3e-4, 3e-4], [1e-2, 1e-2, 1e-14]])
    return np.concatenate([from_eigs(lam, Q), axis_aligned(lam)])


def ulp32(x):
    return np.spacing(np.abs(np.asarray(x, np.float64)).astype(F32)).astype(np.float64)


def check_against_fp64(cov, ls, q):
    """The per-component bounds of the module docstring; returns the measured LS_C, the log-scale error in ulp32, the
    largest direction error and the counts."""
    lam, R_ref = R.eigen_frame(cov)
    ls_ref = np.log(np.sqrt(np.maximum(lam, 1e-12)))
    lam_max = np.abs(lam).max(axis=1, keepdims=True)
    ls32 = np.asarray(ls, F32)
    margin = LAM_C * EPS64 * lam_max
    clamped = lam + margin < 1e-12
    assert np.all(ls32[clamped].view(U32) == CLAMP32.view(U32)), "a clamped scale is not float32(log 1e-6)"
    checked = (lam >= LS_FLOOR * lam_max) & (lam - margin > 1e-12)
    scaled = EPS64 * lam_max / np.where(checked, lam, 1.0)
    excess = np.abs(ls32.astype(np.float64) - ls_ref) - 2 * ulp32(ls_ref)
    c = max(0.0, float(np.max(np.where(checked, excess / scaled, 0.0))))
    ulps = float(np.max(np.where(checked, np.abs(ls32 - ls_ref) / ulp32(ls_ref), 0.0)))
    assert np.all(excess[checked] <= LS_C * scaled[checked]), f"log scale error {c:.3g} x 2^-52 lambda_max / lambda"
    gap = np.minimum(np.abs(lam - np.roll(lam, 1, axis=1)), np.abs(lam - np.roll(lam, -1, axis=1)))
    sharp = gap >= GAP_FLOOR * lam_max
    qd = np.asarray(q, np.float64)
    Rq = R.matrix_from_quat_wxyz(qd / np.linalg.norm(qd, axis=1, keepdims=True))
    sin = np.linalg.norm(np.cross(Rq.transpose(0, 2, 1), R_ref.transpose(0, 2, 1)), axis=2)
    angle = float(sin[sharp].max(initial=0.0))
    assert angle <= ANGLE_TOL, f"eigenvector off by {angle:.3g}"
    return dict(c=c, ulps=ulps, angle=angle, checked=int(checked.sum()), clamped=int(clamped.sum()), sharp=int(sharp.sum()),
                negative=int((lam < 0).sum()))


def scaled_copies(base):
    """base * 2^k for k in KS (float32, exact: rows that would reach the subnormal range are dropped from base)."""
    a = np.abs(base)
    keep = np.all((a == 0) | (a * 2.0 ** KS[0] >= FLT_MIN), axis=1) & np.all(a * 2.0 ** KS[-1] < np.finfo(F32).max, axis=1)
    base = base[keep]
    out = np.stack([base * F32(2.0 ** k) for k in KS])
    assert all(np.array_equal(out[i] / F32(2.0 ** k), base) for i, k in enumerate(KS))
    return base, out


def check_scale_invariance(base, ls, q, exact_ls):
    """ls, q (len(KS), N, .) of base * 2^k: q bit-identical across k; ls shifted by k/2 ln 2 where neither side clamps."""
    i0 = KS.index(0)
    qb = q.view(U32 if q.dtype == F32 else np.uint64)
    assert np.all(qb == qb[i0])
    worst = 0.0
    for i, k in enumerate(KS):
        free = (ls[i] > exact_ls) & (ls[i0] > exact_ls)
        want = ls[i0].astype(np.float64) + k / 2 * np.log(2.0)
        err = np.abs(ls[i].astype(np.float64) - want)
        tol = (0.5 * ulp32(ls[i]) + 0.5 * ulp32(ls[i0])) if ls.dtype == F32 else 1e-14 * (np.abs(want) + 1)
        assert np.all(err[free] <= tol[free] + 1e-12 * np.abs(want[free])), k
        worst = max(worst, float(np.max(np.where(free, err - tol, -np.inf))))
    return worst


# ------------------------------------------------------------------------------------------------------------------ CPU
def test_clamp_is_float32_log_of_1e_6():
    assert CLAMP32.view(U32) == F32(np.log(1e-6)).view(U32)


def test_cases_reach_the_edges():
    """The flat cases include thin eigenvalues that float32 rounding made negative, clamped ones, and every ratio; the
    half-turns take Markley's x, y and z branches."""
    cov = flat_covs(1)
    lam, _ = R.eigen_frame(cov)
    assert (lam[:, 2] < 0).sum() >= 20 and (lam[:, 2] < 1e-12).sum() >= 100
    _, Rr = R.eigen_frame(near_half_turns())
    dec = np.stack([Rr[:, 0, 0], Rr[:, 1, 1], Rr[:, 2, 2], np.trace(Rr, axis1=1, axis2=2)], axis=1)
    assert set(np.argmax(dec, axis=1)) >= {0, 1, 2}
    lam, _ = R.eigen_frame(extreme_covs(2))
    assert np.any(np.abs(lam / 1e-12 - 1 - 2.0 ** -20) < 2.0 ** -22) and np.any(np.abs(lam / 1e-12 - 1 + 2.0 ** -20) < 2.0 ** -22)
    assert np.abs(extreme_covs(2)).max() > 1e38 and np.all(np.isfinite(extreme_covs(2)))


def test_fixture_diagonal_quaternions_match_oracle(edges):
    """Exact rotations: the oracle's quaternion is the reference's bit for bit (float32), -0.0 off-diagonals included."""
    cov = edges["diag/cov"]
    assert np.signbit(cov[:, [1, 2, 4]]).sum() == 6 * 6
    ls, q = R.cov3D_to_log_scales_and_quats(cov)
    _, Rr = R.eigen_frame(cov)
    scipy_q = Rotation.from_matrix(Rr).as_quat()[:, [3, 0, 1, 2]]
    assert np.array_equal(q.astype(F32).view(U32), edges["diag/quats"].astype(F32).view(U32))
    assert np.array_equal(scipy_q.astype(F32).view(U32), edges["diag/quats"].astype(F32).view(U32))
    assert np.all(np.abs(ls - edges["diag/log_scales"]) <= ulp32(edges["diag/log_scales"]))
    assert len({tuple(r) for r in edges["diag/quats"].round(6)}) == 6                # one rotation per ordering


def test_fixture_nonfinite_outcomes(edges):
    """The reference never returns a finite Gaussian for a non-finite covariance: eigh or from_matrix raises, or the
    outputs hold NaN. The product writes NaN for every such row (DESIGN §5)."""
    cov, outcome = edges["nonfinite/cov"], edges["nonfinite/outcome"]
    assert len(cov) == 18 and np.all((~np.isfinite(cov)).sum(axis=1) == 1)
    assert set(outcome) <= {"nan", "eigh", "from_matrix"}
    raised = outcome != "nan"
    assert np.all(np.isnan(edges["nonfinite/log_scales"][raised])) and np.all(edges["nonfinite/error"][raised] != "")
    assert np.all(np.isnan(edges["nonfinite/log_scales"][~raised]).any(axis=1))
    assert [str(v).split()[0] for v in edges["versions"]] == ["torch", "numpy", "scipy"]
    ls, q = R.cov3D_to_log_scales_and_quats(cov)
    assert np.all(np.isnan(ls)) and np.all(np.isnan(q))


def test_oracle_nonfinite_rows_leave_the_rest_alone(edges):
    fin = random_inputs(50, 1, seed=8)[1]
    mixed = fin.copy()
    mixed[::3] = edges["nonfinite/cov"][:len(mixed[::3])]
    ls, q = R.cov3D_to_log_scales_and_quats(mixed)
    ls0, q0 = R.cov3D_to_log_scales_and_quats(fin)
    bad = np.zeros(50, bool)
    bad[::3] = True
    assert np.all(np.isnan(ls[bad])) and np.all(np.isnan(q[bad]))
    assert np.array_equal(ls[~bad], ls0[~bad]) and np.array_equal(q[~bad], q0[~bad])
    rec = R.ply_records(np.zeros((50, 3), F32), mixed, np.zeros((50, 1, 3), F32), np.zeros(50, F32))
    assert np.all(np.isnan(rec[bad, -7:])) and not np.isnan(rec[~bad]).any()


def test_oracle_scale_invariance():
    """The metamorphic check on the oracle: fp64 eigh is invariant under power-of-two scaling too."""
    base = np.concatenate([flat_covs(3, n_rot=8), random_inputs(300, 1, seed=3)[1], degenerate_covs(), near_half_turns()])
    base, covs = scaled_copies(base)
    ls, q = R.cov3D_to_log_scales_and_quats(covs.reshape(-1, 6))
    check_scale_invariance(base, ls.reshape(len(KS), -1, 3), q.reshape(len(KS), -1, 4), np.log(np.sqrt(1e-12)) + 1e-12)


def test_empty_ply_is_the_header_alone(tmp_path):
    from pixie_b200 import frame_export as FE
    p = str(tmp_path / "e.ply")
    FE._write_ply(p, FE.gaussian_ply_header(0, 4), torch.zeros((0, 26)))
    assert open(p, "rb").read() == FE.gaussian_ply_header(0, 4)
    header, _, rows = read_ply(p)
    assert rows.shape == (0, 26)


# ------------------------------------------------------------------------------------------------------------------ GPU
def _scales_quats(cov, dev):
    from pixie_b200.frame_export import cov3D_to_log_scales_and_quats
    ls, q = cov3D_to_log_scales_and_quats(_dev(cov, dev))
    return ls.cpu().numpy(), q.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["flat", "extreme", "half_turns", "ties"])
def test_device_against_fp64_oracle(built_lib, cuda_dev, case):
    cov = {"flat": lambda: flat_covs(1), "extreme": lambda: extreme_covs(2), "half_turns": near_half_turns, "ties": tied_covs}[case]()
    ls, q = _scales_quats(cov, cuda_dev)
    m = check_against_fp64(cov, ls, q)
    print(f"\n[measured] {case}: {m}")
    if case != "extreme":               # its eigenvalue check (a) is in absolute terms, sized for variances 1e-8 .. 1e-2
        check_against_oracle(cov, ls, q)                                    # rebuild, R(q)^T R_ref, from_matrix(R(q)) = q
    if case == "flat":
        assert m["negative"] >= 20 and m["clamped"] >= 100 and m["sharp"] >= 2000


@pytest.mark.gpu
def test_device_scale_invariance(built_lib, cuda_dev):
    base = np.concatenate([flat_covs(4, n_rot=8), random_inputs(500, 1, seed=4)[1], degenerate_covs(), near_half_turns(),
                           tied_covs()])
    base, covs = scaled_copies(base)
    ls, q = _scales_quats(covs.reshape(-1, 6), cuda_dev)
    worst = check_scale_invariance(base, ls.reshape(len(KS), -1, 3), q.reshape(len(KS), -1, 4), CLAMP32)
    print(f"\n[measured] scale invariance: {len(base)} covariances x {len(KS)} k, worst log-scale excess {worst:.3g}")


@pytest.mark.gpu
def test_device_exact_rotations_match_reference(built_lib, cuda_dev, edges):
    """Diagonal covariances (a signed permutation R): the quaternion is the reference's and scipy's of the oracle's R,
    bit for bit and sign included, with and without -0.0 off-diagonals."""
    cov = edges["diag/cov"]
    ls, q = _scales_quats(cov, cuda_dev)
    _, Rr = R.eigen_frame(cov)
    want = Rotation.from_matrix(Rr).as_quat()[:, [3, 0, 1, 2]].astype(F32)
    assert np.array_equal(q.view(U32), want.view(U32)), np.argwhere(q.view(U32) != want.view(U32))
    assert np.array_equal(q.view(U32), edges["diag/quats"].astype(F32).view(U32))
    assert np.all(np.abs(ls - edges["diag/log_scales"]) <= ulp32(edges["diag/log_scales"]))
    cov = axis_aligned(np.array([2e-3, 7e-4, 3e-7]) * 10.0 ** np.arange(-4, 5, 2)[:, None])    # and at other magnitudes
    ls, q = _scales_quats(cov, cuda_dev)
    _, Rr = R.eigen_frame(cov)
    assert np.array_equal(q.view(U32), Rotation.from_matrix(Rr).as_quat()[:, [3, 0, 1, 2]].astype(F32).view(U32))


def _nonfinite_layout(n, seed):
    """Finite inputs and, for every lane of a 128-thread block, one row in that lane made non-finite (NaN, +-Inf or a
    NaN with a payload, in each of the six entries in turn), spread over the blocks including the partial tail block."""
    pos, cov, shs, opacity = random_inputs(n, 16, seed)
    blocks = (n + 127) // 128
    rows = []
    for lane in range(128):
        b = lane % blocks
        if b * 128 + lane >= n:
            b = 0
        rows.append(b * 128 + lane)
    rows += [n - 1, (blocks - 1) * 128]                                      # the tail block's last and first lane
    values = np.array([0x7FC00000, 0x7F800000, 0xFF800000, 0x7FC00123, 0xFF800001], U32).view(F32)
    bad = cov.copy()
    for i, r in enumerate(rows):
        bad[r, i % 6] = values[i % len(values)]
    return pos, cov, bad, shs, opacity, np.array(sorted(set(rows)))


@pytest.mark.gpu
@pytest.mark.parametrize("n", [128, 3 * 128 + 37])
def test_device_nonfinite_rows(built_lib, cuda_dev, n):
    from pixie_b200.frame_export import gaussian_ply_records
    pos, cov, bad, shs, opacity, rows = _nonfinite_layout(n, seed=n)
    args = [_dev(a, cuda_dev) for a in (pos, bad, shs, opacity)]
    got = gaussian_ply_records(*args).cpu().numpy()
    ref = gaussian_ply_records(*[_dev(a, cuda_dev) for a in (pos, cov, shs, opacity)]).cpu().numpy()
    hit = np.zeros(n, bool)
    hit[rows] = True
    assert len(rows) >= min(n, 128) and set(rows % 128) == set(range(min(n, 128)))
    assert np.all(np.isnan(got[hit, -7:]))
    assert np.array_equal(got[hit, :-7].view(U32), ref[hit, :-7].view(U32))   # the copied columns and normals
    assert np.array_equal(got[~hit].view(U32), ref[~hit].view(U32))
    assert not np.isnan(ref).any()
    ls, q = R.cov3D_to_log_scales_and_quats(bad)                              # the oracle agrees on which rows are NaN
    assert np.array_equal(np.isnan(ls).all(axis=1), hit) and np.array_equal(np.isnan(q).all(axis=1), hit)


@pytest.mark.gpu
@pytest.mark.parametrize("K", [1, 4, 9, 16])
@pytest.mark.parametrize("aligned", [True, False])
def test_device_copies_are_bit_exact(built_lib, cuda_dev, K, aligned):
    """xyz, f_dc, f_rest and opacity as uint32: -0.0, subnormals, NaN payloads and +-Inf pass through unchanged."""
    from pixie_b200.frame_export import gaussian_ply_records
    n = 2 * 128 + 77
    pos, cov, shs, opacity = random_inputs(n, K, seed=K)
    sp = SPECIAL_BITS.view(F32)
    for a, step in ((pos, 7), (shs, 5), (opacity, 3)):
        flat = a.reshape(-1)
        flat[::step] = sp[np.arange(len(flat[::step])) % len(sp)]

    def put(a):
        if aligned:
            return _dev(a, cuda_dev)
        buf = torch.zeros(a.size + 1, device=cuda_dev)
        buf[1:] = _dev(a, cuda_dev).reshape(-1)
        return buf[1:].view(a.shape)
    rec = gaussian_ply_records(put(pos), put(cov), put(shs), put(opacity)).cpu().numpy()
    bits = rec.view(U32)
    assert np.array_equal(bits[:, :3], pos.view(U32))
    assert np.all(bits[:, 3:6] == 0)
    assert np.array_equal(bits[:, 6:9], shs[:, 0, :].view(U32))
    assert np.array_equal(bits[:, 9:9 + 3 * (K - 1)], np.ascontiguousarray(shs[:, 1:, :].transpose(0, 2, 1)).reshape(n, -1).view(U32))
    assert np.array_equal(bits[:, 6 + 3 * K], opacity.view(U32))
    assert not np.isnan(rec[:, -7:]).any()


@pytest.mark.gpu
def test_frame_writer_sequences(built_lib, cuda_dev, tmp_path):
    """Frames that shrink after a large one (a reused pinned buffer read through a shorter view), an empty frame, K
    changing between frames, submits under a non-default current stream, and inputs overwritten in place on that stream
    as soon as submit() returns: each file holds the records of the inputs as they were at submit()."""
    from pixie_b200 import frame_export as FE
    plan = [(3000, 16), (700, 16), (0, 4), (1200, 1), (2500, 9), (1, 4), (0, 16), (900, 16)]
    frames = [random_inputs(n, K, seed=20 + f) if n else (np.zeros((0, 3), F32), np.zeros((0, 6), F32), np.zeros((0, K, 3), F32),
                                                          np.zeros(0, F32)) for f, (n, K) in enumerate(plan)]
    want = [FE.gaussian_ply_records(*[_dev(a, cuda_dev) for a in fr]).cpu().numpy() for fr in frames]
    d = tmp_path / "frames"
    side = torch.cuda.Stream(cuda_dev)
    with torch.cuda.stream(side), FE.PlyFrameWriter(str(d), cuda_dev) as w:
        for f, fr in enumerate(frames):
            ins = [_dev(a, cuda_dev) for a in fr]
            w.submit(f, *ins)
            for t in ins:                                                      # the next substeps reuse the buffers
                t.fill_(float("nan"))
    for f, (n, K) in enumerate(plan):
        path = d / f"frame_{f:05d}.ply"
        header = FE.gaussian_ply_header(n, K)
        data = open(path, "rb").read()
        assert data == header + want[f].astype("<f4").tobytes(), f
        _, names, rows = read_ply(str(path))
        assert rows.shape == (n, 14 + 3 * K) and names == R.attribute_names(K)
