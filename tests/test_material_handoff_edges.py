"""Edge cases of the material-field hand-off (U-Net field -> per-particle properties and stationary-cluster BCs).

CPU: the oracles (oracle/material_transfer_ref.py, oracle/frame_export_ref.py, tests/stationary_ref.py) are held to
scikit-learn, numpy and an fp64 restatement of DBSCAN at the same edges, and the class-index rule to the vectors the
reference's own `get_mat_id` / `map_pred_to_ply` wrote into tests/golden/transfer_golden.npz.
GPU (`-m gpu`): csrc/field_transfer.cu and csrc/cluster.cu, through pixie_b200, against those oracles:
  * kNN smoothing at every k in 1..16, plain and weighted, on fields of 1, 255, 256, 257 points and a ragged 64^3 grid,
    with query counts that are not a multiple of the 128-thread block and queries without distance ties;
  * the distance threshold one float32 step either side, and at np.float32(0.1) > 0.1;
  * field extraction of class-index fields, single-channel fields, exact ties, empty and full masks;
  * DBSCAN at eps^2 +- one fp64 ulp, min_samples = 1 and above every neighbourhood, cell keys clamped at 2^21,
    thousands of points in one cell, subsets of 0 and 1 points;
  * particle volume on cell faces and outside the grid, frame transform with 0, 1 and 8 rotations and no points.
Bounds are exact unless a comment states an ulp count and its reason."""
import functools
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import stationary_ref as S  # noqa: E402
from oracle import frame_export_ref as FR  # noqa: E402
from oracle import material_transfer_ref as R  # noqa: E402

G = np.load(os.path.join(HERE, "golden", "transfer_golden.npz"))
RANGES = dict(density_min=1.703, density_max=3.871, E_min=3.018, E_max=10.882, nu_min=0.2103, nu_max=0.4493)
KEYS = ("part_labels", "density", "E", "nu", "material_id", "conf")
FLOATS = ("density", "E", "nu", "conf")


def _f32_ulps(a, b):
    """Distance in float32 ulps between same-signed finite float32 arrays."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    assert np.all(np.signbit(a) == np.signbit(b))
    return np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))


# ================================================================================================== kNN smoothing
def _props(rng, m, n_labels=3):
    """Random per-point properties; few labels, so modes are often tied in count and resolved by neighbour order."""
    return {"density": rng.uniform(200, 3000, m).astype(np.float32), "E": (10 ** rng.uniform(3, 9, m)).astype(np.float32),
            "nu": rng.uniform(0.2, 0.45, m).astype(np.float32), "conf": rng.uniform(0.05, 1, m).astype(np.float32),
            "material_id": rng.integers(0, n_labels, m).astype(np.int32), "part_labels": rng.integers(0, n_labels, m).astype(np.int32)}


@functools.lru_cache(maxsize=None)
def _knn_field(name):
    """Material point clouds whose sizes straddle the kernel's 256-point shared-memory tile."""
    rng = np.random.default_rng({"m1": 11, "m255": 12, "m256": 13, "m257": 14, "grid64": 15}[name])
    if name == "grid64":                                     # voxel centres of a 64^3 grid under a ragged mask
        D = 64
        mask = (rng.uniform(size=(D, D, D)) < 0.3).astype(np.float32)
        mask[0, 0, :7] = 1.0
        axes = [np.linspace(-0.5, 0.5, D) for _ in range(3)]
        pos = np.stack(np.meshgrid(*axes, indexing="ij"), axis=-1)[mask > 0].astype(np.float32)
    else:
        pos = rng.uniform(-0.5, 0.5, size=(int(name[1:]), 3)).astype(np.float32)
    field = {"pos": pos, **_props(rng, len(pos))}
    assert len(pos) % 256 != 0 or name == "m256"
    return field


def _sq_dist(q, pos):
    """fp64 squared distances ((dx^2 + dy^2) + dz^2) of float32 points, as scikit-learn's KD-tree reduces them."""
    d = q.astype(np.float64)[None, :] - pos.astype(np.float64)
    return (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]


def _untied(q, pos, k):
    """True when the k + 1 smallest distances from q are pairwise distinct.

    scikit-learn does not order equal distances by index, so a tie inside the k nearest or at the k-th would leave the
    expected neighbour order (and with it np.mean's summation order and the first-met mode) unpinned. Distances within
    1e-12 relative count as tied too: the device may contract the squared distance into FMAs."""
    j = min(k + 1, len(pos))
    s = np.sort(np.partition(_sq_dist(q, pos), j - 1)[:j])
    return bool(np.all(np.diff(s) > 1e-12 * s[1:]))


def _untied_queries(pos, n, k, rng, spread):
    """n float32 queries scattered around the field's points, drawn by rejection of tied ones."""
    out = []
    while len(out) < n:
        for q in (pos[rng.integers(0, len(pos), 2 * n)] + rng.normal(0, spread, (2 * n, 3))).astype(np.float32):
            if _untied(q, pos, k):
                out.append(q)
                if len(out) == n:
                    break
    return np.array(out, np.float32)


@functools.lru_cache(maxsize=None)
def _knn_case(name, k):
    """(field, queries): 333 queries (the 64^3 field: 389), a few of them beyond the 0.25 threshold."""
    field = _knn_field(name)
    rng = np.random.default_rng(100 * k + len(field["pos"]) % 97)
    n = 389 if name == "grid64" else 333
    q = _untied_queries(field["pos"], n, k, rng, 0.02)
    q[::23] += np.float32(3.0)                               # too far: 15 (17) of 333 (389), under the 10 % the reference asserts
    return field, q


def _run_device(field, q, k, thr, weighted, dev):
    from pixie_b200 import material_transfer as MT
    params = {key: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for key, v in field.items()}
    out = MT.perform_knn_smoothing(torch.from_numpy(q).to(dev), params, k, thr, weighted)
    return [o.cpu().numpy() for o in out]


def _too_far(field, q, thr):
    return np.array([np.sqrt(_sq_dist(x, field["pos"]).min()) > thr for x in q])


def _assert_knn_equal(got, want, weighted, far, exact_defaults):
    for name, g, w in zip(KEYS, got, want):
        assert g.shape == w.shape, name
        if name not in FLOATS:
            assert np.array_equal(g, w), f"{name}: {(g != w).sum()} of {len(w)} differ"
            continue
        near = ~far
        if weighted:
            # the device normalises the weights by a sequential fp64 total and sums w_j * v_j sequentially in fp64; the
            # reference divides by np.sum's pairwise total and calls np.dot. Both round one fp64 value to float32, so
            # they can land on either side of a float32 rounding boundary: one ulp.
            assert _f32_ulps(g[near], w[near]).max(initial=0) <= 1, name
        else:
            assert np.array_equal(g[near], w[near]), f"{name}: {(g[near] != w[near]).sum()} of {near.sum()} differ"
        if exact_defaults:
            assert np.array_equal(g[far], w[far]), name
    # rows beyond the threshold carry the field's mean, which torch reduces on the device in another order than
    # np.mean; _knn_threshold_field uses dyadic values on 256 points so that every order gives the same mean.


@pytest.mark.gpu
@pytest.mark.parametrize("weighted", [False, True], ids=["plain", "weighted"])
@pytest.mark.parametrize("k", list(range(1, 17)))
def test_cuda_knn_every_k_matches_sklearn(built_lib, cuda_dev, k, weighted):
    for name in ("m1", "m255", "m256", "m257", "grid64"):
        field = _knn_field(name)
        if len(field["pos"]) < k:
            continue
        field, q = _knn_case(name, k)
        thr = 0.25
        want = R.perform_knn_smoothing(q, field, k, thr, weighted)
        got = _run_device(field, q, k, thr, weighted, cuda_dev)
        far = _too_far(field, q, thr)
        assert far.sum() == (len(q) + 22) // 23
        assert np.array_equal(got[4][far], np.full(far.sum(), R.STATIONARY_ID)) and np.array_equal(got[0][far], np.zeros(far.sum()))
        _assert_knn_equal(got, want, weighted, far, exact_defaults=False)


def test_oracle_knn_every_k_is_numpy_mean_of_the_sklearn_neighbours():
    """The oracle's plain mean is np.mean over the k nearest in distance order; the device reproduces np.mean's pairwise
    float32 order (numpy_sum_f32: k < 8, multiples of 8, remainders). Hold that order to np.mean itself here."""
    def pairwise_f32(a):
        n = len(a)
        if n < 8:
            r = np.float32(0)
            for x in a:
                r = np.float32(r + x)
            return r
        r = list(a[:8])
        i = 8
        while i < n - n % 8:
            r = [np.float32(r[j] + a[i + j]) for j in range(8)]
            i += 8
        res = np.float32(np.float32(np.float32(r[0] + r[1]) + np.float32(r[2] + r[3])) + np.float32(np.float32(r[4] + r[5]) + np.float32(r[6] + r[7])))
        for x in a[i:]:
            res = np.float32(res + x)
        return res
    rng = np.random.default_rng(7)
    for k in range(1, 17):
        for _ in range(300):
            v = (rng.standard_normal(k) * 10 ** rng.uniform(-3, 8)).astype(np.float32)
            assert np.mean(v) == np.float32(pairwise_f32(v) / np.float32(k)), k
    from sklearn.neighbors import NearestNeighbors
    field, q = _knn_case("m257", 16)
    _, idx = NearestNeighbors(n_neighbors=16).fit(field["pos"]).kneighbors(q)
    order = np.argsort(np.stack([_sq_dist(x, field["pos"]) for x in q]), axis=1, kind="stable")[:, :16]
    assert np.array_equal(idx, order)                        # untied queries: scikit-learn's order is the fp64 distance order


def _knn_threshold_field():
    """256 points: one at the origin, the rest at least 0.6 away. Dyadic property values keep every partial sum exact,
    so the field mean (the default of rows beyond the threshold) is the same whatever the summation order."""
    rng = np.random.default_rng(21)
    pos = rng.uniform(-2, 2, size=(256, 3)).astype(np.float32)
    pos[np.linalg.norm(pos, axis=1) < 0.6] += np.float32(1.5)
    pos[0] = 0.0
    props = {"density": rng.integers(200, 3000, 256).astype(np.float32), "E": rng.integers(1000, 60000, 256).astype(np.float32),
             "nu": (rng.integers(205, 460, 256) / 1024).astype(np.float32), "conf": (rng.integers(1, 256, 256) / 256).astype(np.float32),
             "material_id": rng.integers(0, 6, 256).astype(np.int32), "part_labels": rng.integers(1, 9, 256).astype(np.int32)}
    return {"pos": pos, **props}


def _threshold_queries(thr):
    """Queries on the axes through the origin point, one float32 step either side of `thr` (and at float32(thr))."""
    f = np.float32(thr)
    below = f if float(f) <= thr else np.nextafter(f, np.float32(0))
    steps = sorted({float(below), float(np.nextafter(below, np.float32(1))), float(np.nextafter(below, np.float32(0))), float(f)})
    q = []
    for j, s in enumerate(steps):
        v = np.zeros(3, np.float32)
        v[j % 3] = s if j % 2 == 0 else -s
        q.append(v)
    return np.array(q, np.float32)


def test_oracle_threshold_compares_the_fp64_distance():
    field = _knn_threshold_field()
    thr = 0.1
    edge = _threshold_queries(thr)
    assert all(_untied(x, field["pos"], 5) for x in edge)
    q = np.concatenate([edge, _untied_queries(field["pos"][1:], 60, 4, np.random.default_rng(1), 0.01)])
    out = R.perform_knn_smoothing(q, field, 4, thr, False)
    far = out[4][: len(edge)] == R.STATIONARY_ID
    dist = np.abs(edge).max(axis=1).astype(np.float64)
    assert np.array_equal(far, dist > thr) and far.sum() == 1   # np.float32(0.1) = 0.10000000149 > 0.1: too far for scikit-learn
    assert float(np.float32(0.1)) > 0.1 and np.float32(0.1) in edge


@pytest.mark.gpu
@pytest.mark.parametrize("weighted", [False, True], ids=["plain", "weighted"])
@pytest.mark.parametrize("thr", [0.1, 0.2, 0.125, 0.3, 0.05])
def test_cuda_threshold_one_float32_step_either_side(built_lib, cuda_dev, thr, weighted):
    field = _knn_threshold_field()
    rng = np.random.default_rng(int(thr * 1000))
    edge = _threshold_queries(thr)
    assert all(_untied(x, field["pos"], 5) for x in edge)
    q = np.concatenate([edge, _untied_queries(field["pos"][1:], 77, 5, rng, 0.01)])
    want = R.perform_knn_smoothing(q, field, 5, thr, weighted)
    got = _run_device(field, q, 5, thr, weighted, cuda_dev)
    far = _too_far(field, q, thr)
    assert 1 <= far[: len(edge)].sum() < len(edge)           # the edge queries fall on both sides
    _assert_knn_equal(got, want, weighted, far, exact_defaults=True)


@pytest.mark.gpu
def test_cuda_threshold_counts_float32_point_one_as_too_far(built_lib, cuda_dev, capsys):
    """A query at np.float32(0.1) from the only point within reach is 0.10000000149 away: beyond the 0.1 threshold for
    scikit-learn. Rounding the threshold to float32 would accept it."""
    field = _knn_threshold_field()
    q = np.concatenate([np.array([[np.float32(0.1), 0, 0]], np.float32),
                        _untied_queries(field["pos"][1:], 40, 3, np.random.default_rng(3), 0.01)])
    got = _run_device(field, q, 3, 0.1, False, cuda_dev)
    assert "too far from nearest neighbor: 1," in capsys.readouterr().out
    assert got[4][0] == R.STATIONARY_ID and got[0][0] == 0
    assert got[1][0] == np.mean(field["density"])            # the dyadic field mean is exact


@pytest.mark.gpu
def test_cuda_mirror_labels_weighted_smallest_plain_first(built_lib, cuda_dev):
    """Two labels at mirror-image distances from the query: the weighted votes tie exactly and go to the smaller label;
    the plain counts tie and go to the label met first (the lower field index on equal distances)."""
    pos = np.array([[0.02, 0, 0], [-0.02, 0, 0], [0, 0.5, 0]], np.float32)
    field = {"pos": pos, "density": np.array([1000, 3000, 7], np.float32), "E": np.array([1e5, 3e5, 7], np.float32),
             "nu": np.array([0.25, 0.35, 0.4], np.float32), "conf": np.array([0.5, 1.0, 0.1], np.float32),
             "material_id": np.array([5, 2, 0], np.int32), "part_labels": np.array([7, 3, 0], np.int32)}
    q = np.zeros((1, 3), np.float32)
    for weighted, mat, part in ((True, 2, 3), (False, 5, 7)):
        got = _run_device(field, q, 2, 0.1, weighted, cuda_dev)
        assert got[4][0] == mat and got[0][0] == part, weighted
        assert got[1][0] == np.float32(2000) and got[2][0] == np.float32(2e5) and got[3][0] == np.float32(0.3)
        want = R.perform_knn_smoothing(q, field, 2, 0.1, weighted)
        assert want[4][0] == mat and want[0][0] == part, weighted


def test_knn_k_above_field_size_raises():
    from pixie_b200 import material_transfer as MT
    field = _knn_field("m255")
    small = {key: v[:5] for key, v in field.items()}
    q = np.zeros((7, 3), np.float32)
    with pytest.raises(ValueError):
        R.perform_knn_smoothing(q, small, 6)                 # scikit-learn: n_neighbors > n_samples_fit
    with pytest.raises(ValueError):
        MT.perform_knn_smoothing(torch.from_numpy(q), {key: torch.from_numpy(v) for key, v in small.items()}, 6)


@pytest.mark.gpu
def test_cuda_knn_rejects_k_17_and_k_above_field(built_lib, cuda_dev):
    from pixie_b200 import _lib
    field = _knn_field("m255")
    q = np.zeros((7, 3), np.float32)
    with pytest.raises(_lib.PixieError):
        _run_device(field, q, 17, 0.1, False, cuda_dev)
    with pytest.raises(ValueError):
        _run_device({key: v[:16] for key, v in field.items()}, q, 17, 0.1, False, cuda_dev)
    r = _run_device({key: v[:16] for key, v in field.items()}, q, 16, 10.0, False, cuda_dev)       # k == m is fine
    assert np.all(r[1] == r[1][0])


# ================================================================================================== field extraction
def _index_field(D, seed, fractional=False):
    """(4, D, D, D) prediction whose single class channel holds class indices 0..7 (the label-map format)."""
    rng = np.random.default_rng(seed)
    pred = np.zeros((4, D, D, D), np.float32)
    pred[:3] = rng.uniform(-1.2, 1.2, size=(3, D, D, D))
    pred[3] = rng.integers(0, 8, size=(D, D, D))
    if fractional:                                           # 'i4' storage truncates: 2.75 -> 2, -0.5 -> 0, 7.999 -> 7
        pick = rng.choice(D ** 3, 500, replace=False)
        pred[3].reshape(-1)[pick] = rng.choice(np.array([2.75, -0.5, 7.999, 0.25, 5.5], np.float32), 500)
    mask = (rng.uniform(size=(D, D, D)) < 0.35).astype(np.float32)
    return pred, mask


def test_oracle_class_index_rule_follows_get_mat_id():
    lo, hi = np.array([-0.5, -0.4, -0.3]), np.array([0.5, 0.6, 0.7])
    pred, mask = _index_field(64, 1, fractional=True)
    t = R.vertex_table(pred, mask, lo, hi, RANGES)
    assert np.array_equal(t["material_id"], pred[3][mask > 0].astype(np.int32)) and np.all(t["conf"] == 1.0)
    assert set(np.unique(t["material_id"])) == set(range(8))
    pred16, mask16 = _index_field(16, 2)
    t16 = R.vertex_table(pred16, mask16, lo, hi, RANGES)
    assert np.all(t16["material_id"] == 0) and np.all(t16["part_labels"] == 0) and np.all(t16["conf"] == 1.0)   # argmax of one channel


def test_oracle_class_index_field_matches_reference_golden():
    """tests/golden/transfer_golden.npz 'field_index/*': a (4, 64, 64, 64) label-map prediction run through the
    reference's own map_pred_to_ply, including fractional and negative class values."""
    pred, mask = _golden_index_dense()
    t = R.vertex_table(pred, mask, G["field/min_bounds"], G["field/max_bounds"], RANGES)
    for key, col in (("material_id", "material_id"), ("part_labels", "part_label"), ("conf", "conf")):
        assert np.array_equal(t[key], G[f"field_index/table/{col}"]), key
    pos = np.stack([G[f"field_index/table/{c}"] for c in "xyz"], axis=1)
    assert np.array_equal(t["pos"], pos)
    vals = G["field_index/vals"][:, 3]
    assert np.any(vals != np.round(vals)) and np.any(vals < 0)   # the truncation is exercised


def _golden_index_dense():
    idx, vals = G["field_index/idx"], G["field_index/vals"]
    pred = np.zeros((vals.shape[1], 64, 64, 64), np.float32)
    mask = np.zeros((64, 64, 64), np.float32)
    pred[:, idx[:, 0], idx[:, 1], idx[:, 2]] = vals.T
    mask[idx[:, 0], idx[:, 1], idx[:, 2]] = 1.0
    return pred, mask


def _extract(pred, mask, lo, hi, dev):
    from pixie_b200 import material_transfer as MT
    t = MT.extract_material_points(torch.from_numpy(pred).to(dev), torch.from_numpy(mask).to(dev), lo, hi, RANGES)
    return {key: v.cpu().numpy() for key, v in t.items()}


def _assert_extract(got, want):
    # ids, confidences, positions and the count are exact; the continuous channels (powf) are held by
    # tests/test_transfer_golden.py and tests/test_material_transfer.py
    for key in ("pos", "material_id", "part_labels", "conf"):
        assert got[key].shape == want[key].shape, key
        assert np.array_equal(got[key], want[key]), f"{key}: {(got[key] != want[key]).sum()} differ"


@pytest.mark.gpu
def test_cuda_extract_class_index_fields(built_lib, cuda_dev):
    lo, hi = np.array([-0.5, -0.4, -0.3]), np.array([0.5, 0.6, 0.7])
    for D, seed, frac in ((64, 1, False), (64, 3, True), (16, 2, False)):
        pred, mask = _index_field(D, seed, frac)
        want = R.vertex_table(pred, mask, lo, hi, RANGES)
        got = _extract(pred, mask, lo, hi, cuda_dev)
        _assert_extract(got, want)
        if D == 64:
            assert np.array_equal(got["material_id"], pred[3][mask > 0].astype(np.int32))
        else:
            assert np.all(got["material_id"] == 0)
    pred, mask = _golden_index_dense()
    got = _extract(pred, mask, G["field/min_bounds"], G["field/max_bounds"], cuda_dev)
    assert np.array_equal(got["material_id"], G["field_index/table/material_id"])
    assert np.array_equal(got["part_labels"], G["field_index/table/part_label"])
    assert np.array_equal(got["conf"], G["field_index/table/conf"])


@pytest.mark.gpu
def test_cuda_extract_ties_and_masks(built_lib, cuda_dev):
    rng = np.random.default_rng(4)
    lo, hi = np.array([-0.52, -0.41, -0.33]), np.array([0.49, 0.6, 0.71])
    D = 24
    pred = rng.uniform(-1.2, 1.2, size=(5, D, D, D)).astype(np.float32)
    tie = rng.uniform(size=(D, D, D)) < 0.3
    pred[4][tie] = pred[3][tie]                              # K = 2, exact ties: the first channel wins
    zeros = rng.uniform(size=(D, D, D)) < 0.05
    pred[3][zeros], pred[4][zeros] = np.float32(-0.0), np.float32(0.0)          # -0 == +0 is a tie too
    cases = [("ragged", (rng.uniform(size=(D, D, D)) < 0.4).astype(np.float32)), ("empty", np.zeros((D, D, D), np.float32)),
             ("full", np.ones((D, D, D), np.float32))]
    for name, mask in cases:
        want = R.vertex_table(pred, mask, lo, hi, RANGES)
        got = _extract(pred, mask, lo, hi, cuda_dev)
        _assert_extract(got, want)
        n = int((mask > 0).sum())
        assert len(got["pos"]) == n, name
        if n:
            assert np.any(got["material_id"][tie[mask > 0]] == 0) and np.any(got["material_id"] == 1), name
    full = rng.uniform(-1, 1, size=(11, 64, 64, 64)).astype(np.float32)       # a full 64^3 mask: 262144 points
    mask = np.ones((64, 64, 64), np.float32)
    _assert_extract(_extract(full, mask, lo, hi, cuda_dev), R.vertex_table(full, mask, lo, hi, RANGES))


# ================================================================================================== DBSCAN
def _dbscan_fp64(pts, eps, min_samples):
    """scikit-learn DBSCAN restated: neighbours = fp64 ((dx^2 + dy^2) + dz^2) <= eps^2 with the point itself, core =
    >= min_samples neighbours, clusters = components of core points labelled in order of their first point, border
    points join the first cluster that reaches them in that order (scikit-learn's expansion order)."""
    p = pts.astype(np.float64)
    n = len(p)
    dx, dy, dz = (p[:, None, c] - p[None, :, c] for c in range(3))
    nb = ((dx * dx + dy * dy) + dz * dz) <= eps * eps
    core = nb.sum(1) >= min_samples
    labels = np.full(n, -1)
    lab = 0
    for i in range(n):
        if labels[i] != -1 or not core[i]:
            continue
        stack = [i]
        labels[i] = lab
        while stack:
            j = stack.pop()
            if not core[j]:
                continue
            for t in np.flatnonzero(nb[j] & (labels == -1)):
                labels[t] = lab
                stack.append(t)
        lab += 1
    return labels


def _boundary_pairs(where):
    """(points, eps): 24 isolated pairs whose fp64 squared distance is one ulp below, at, or one ulp above eps^2."""
    rng = np.random.default_rng({"below": 1, "at": 2, "above": 3}[where])
    ulp = 2.0 ** -21                                          # float32 spacing in [4, 8): sums on this lattice below 8 are exact
    for _ in range(1000):
        off = rng.integers(-40000, 40000, 3) * ulp
        d2 = (off[0] * off[0] + off[1] * off[1]) + off[2] * off[2]
        target = {"below": np.nextafter(d2, np.inf), "at": d2, "above": np.nextafter(d2, 0.0)}[where]
        e0 = np.sqrt(target)
        for e in (e0, np.nextafter(e0, 0.0), np.nextafter(e0, 1.0)):
            if e * e == target and 0.015 < e < 0.04:
                base = np.array([[1.5 + x, 1.5 + y, 1.5 + 2 * z] for x in range(4) for y in range(3) for z in range(2)], np.float64)
                pa = base + rng.integers(0, 2 ** 19, base.shape) * ulp
                pts = np.empty((2 * len(base), 3), np.float32)
                pts[0::2], pts[1::2] = pa, pa + off
                assert np.array_equal(pts.astype(np.float64)[1::2] - pts.astype(np.float64)[0::2], np.broadcast_to(off, pa.shape))
                return pts, float(e)
    raise AssertionError("no boundary pair found")


@functools.lru_cache(maxsize=None)
def _dbscan_case(name):
    """(positions, ids or None, eps, min_samples)."""
    rng = np.random.default_rng(sum(map(ord, name)))
    if name in ("below", "at", "above"):
        pts, eps = _boundary_pairs(name)
        return pts, None, eps, 2
    if name.startswith("cloud"):                             # clumps and a sparse background
        c = rng.uniform(0, 1, (12, 3))
        pts = np.concatenate([c[rng.integers(0, 12, 1500)] + rng.normal(0, 0.02, (1500, 3)), rng.uniform(0, 1, (400, 3))]).astype(np.float32)
        ms = {"cloud_ms1": 1, "cloud_ms_huge": 0}[name]
        if ms == 0:                                          # one more than the largest neighbourhood
            d = pts.astype(np.float64)
            ms = max(int((((d[i] - d) ** 2).sum(1) <= 0.03 ** 2).sum()) for i in range(len(d))) + 1
        ids = np.where(rng.uniform(size=len(pts)) < 0.8, S.STATIONARY_ID, 2).astype(np.int32)
        return pts, ids, 0.03, ms
    if name == "clamped":                                    # clusters 2^21 * eps and more apart share clamped cell keys
        centres = np.array([[0, 0, 0], [1e5, 0, 0], [2e5, 0, 0], [1e5, 1e5, 0], [0, 0, 1.5e5], [2e5, 2e5, 2e5]], np.float64)
        assert np.all(centres[1:].max(1) > 2 ** 21 * 0.03)
        pts = np.concatenate([cc + rng.normal(0, 0.025, (150, 3)) for cc in centres]).astype(np.float32)
        ids = np.where(rng.uniform(size=len(pts)) < 0.7, S.STATIONARY_ID, 0).astype(np.int32)
        return pts, ids, 0.03, 5
    if name.startswith("one_cell"):                          # 3000 points inside one eps cell, plus 20 far, isolated points
        pts = np.concatenate([rng.uniform(0, 0.03 / 2, (3000, 3)), 5 + rng.uniform(0, 1, (20, 3))]).astype(np.float32)
        ms = {"one_cell_8": 8, "one_cell_3000": 3000, "one_cell_3001": 3001}[name]
        return pts, None, 0.03, ms
    raise KeyError(name)


DBSCAN_CASES = ["below", "at", "above", "cloud_ms1", "cloud_ms_huge", "clamped", "one_cell_8", "one_cell_3000", "one_cell_3001"]


def _selected(name):
    pts, ids, eps, ms = _dbscan_case(name)
    return (pts if ids is None else pts[ids == S.STATIONARY_ID]), eps, ms


@pytest.mark.parametrize("name", DBSCAN_CASES)
def test_oracle_dbscan_edges_match_fp64_definition(name):
    sel, eps, ms = _selected(name)
    want = _dbscan_fp64(sel, eps, ms)
    got = S.dbscan_labels(sel, eps, ms)
    assert np.array_equal(got, want)
    n_clusters = got.max() + 1
    expect = {"below": 24, "at": 24, "above": 0, "cloud_ms_huge": 0, "one_cell_8": 1, "one_cell_3000": 1, "one_cell_3001": 0}
    if name in expect:
        assert n_clusters == expect[name], n_clusters
    if name == "cloud_ms1":
        assert (got == -1).sum() == 0 and n_clusters > 50
    if name == "clamped":
        assert n_clusters >= 6


def _device_dbscan(pts, ids, eps, ms, dev):
    from pixie_b200 import material_transfer as MT
    sel = None if ids is None else torch.from_numpy(ids).to(dev)
    p = torch.from_numpy(pts).to(dev)
    labels, index, k = MT._dbscan(p, eps, ms, sel, S.STATIONARY_ID)
    sizes, lo, hi = MT._cluster_stats(p, index, labels, k)
    return labels.cpu().numpy(), index.cpu().numpy(), k, sizes, lo, hi


def _assert_stats(sel, labels, k, sizes, lo, hi):
    assert np.array_equal(sizes, np.bincount(labels[labels >= 0], minlength=k).astype(np.int32))
    for c in range(k):
        pc = sel[labels == c]
        assert np.array_equal(lo[c], pc.min(0)) and np.array_equal(hi[c], pc.max(0)), c


@pytest.mark.gpu
@pytest.mark.parametrize("name", DBSCAN_CASES)
def test_cuda_dbscan_edges_match_sklearn(built_lib, cuda_dev, name):
    pts, ids, eps, ms = _dbscan_case(name)
    sel, _, _ = _selected(name)
    want = S.dbscan_labels(sel, eps, ms)
    labels, index, k, sizes, lo, hi = _device_dbscan(pts, ids, eps, ms, cuda_dev)
    assert np.array_equal(index, np.arange(len(pts)) if ids is None else np.flatnonzero(ids == S.STATIONARY_ID))
    assert np.array_equal(labels, want), f"{(labels != want).sum()} labels differ"
    assert k == want.max() + 1
    _assert_stats(sel, labels, k, sizes, lo, hi)


@pytest.mark.gpu
def test_cuda_dbscan_subsets_of_zero_and_one_point(built_lib, cuda_dev):
    rng = np.random.default_rng(5)
    pts = rng.uniform(0, 1, (300, 3)).astype(np.float32)
    none = np.zeros(300, np.int32)
    labels, index, k, sizes, _, _ = _device_dbscan(pts, none, 0.03, 1, cuda_dev)
    assert labels.shape == (0,) and index.shape == (0,) and k == 0 and sizes.shape == (0,)
    one = none.copy()
    one[137] = S.STATIONARY_ID
    for ms, want in ((1, [0]), (2, [-1])):
        assert np.array_equal(S.dbscan_labels(pts[one == S.STATIONARY_ID], 0.03, ms), want)
        labels, index, k, sizes, lo, hi = _device_dbscan(pts, one, 0.03, ms, cuda_dev)
        assert np.array_equal(labels, want) and np.array_equal(index, [137]) and k == max(want) + 1
        _assert_stats(pts[[137]], labels, k, sizes, lo, hi)


# ================================================================================================== volume and frame transform
def _face_positions(n, dx, rng):
    """Positions on cell faces i * dx (as float32 products and as rounded fp64 products), a float32 step either side,
    and positions outside [0, n * dx)."""
    i = rng.integers(0, n + 1, 600)
    faces = np.concatenate([np.float32(i) * np.float32(dx), (i * dx).astype(np.float32)])
    faces = np.concatenate([faces, np.nextafter(faces, np.float32(-1)), np.nextafter(faces, np.float32(10 ** 3))])
    outside = np.array([-5.0, -1e-30, -0.0, np.float32(n * dx), np.nextafter(np.float32(n * dx), np.float32(1e3)), 3 * n * dx, 90.0],
                       np.float32)
    vals = np.concatenate([faces, outside]).astype(np.float32)
    return vals[rng.integers(0, len(vals), (4000, 3))].astype(np.float32)


def test_oracle_volume_clamps_outside_positions():
    pos = np.array([[-5.0, 0.01, 0.01], [0.01, 0.01, 0.01], [1.99, 1.99, 1.99], [7.0, 9.0, 2.0]], np.float32)
    vol = FR.get_particle_volume(pos, 32, 2.0 / 32)
    cell = np.float32(2.0 / 32) ** 3
    assert np.array_equal(vol, [cell / 2, cell / 2, cell / 2, cell / 2])          # clamped into cells (0,0,0) and (31,31,31)


@pytest.mark.gpu
@pytest.mark.parametrize("grid_n", [32, 48, 7])
def test_cuda_particle_volume_on_faces_and_outside(built_lib, cuda_dev, grid_n):
    from pixie_b200.frame_export import get_particle_volume
    dx = 2.0 / grid_n
    pos = _face_positions(grid_n, dx, np.random.default_rng(grid_n))
    idx = np.floor(pos / np.float32(dx))
    assert np.any(idx < 0) and np.any(idx >= grid_n) and np.any(pos == np.float32(dx))
    got = get_particle_volume(torch.from_numpy(pos).to(cuda_dev), grid_n, dx).cpu().numpy()
    assert np.array_equal(got, FR.get_particle_volume(pos, grid_n, dx))
    empty = get_particle_volume(torch.zeros((0, 3), device=cuda_dev), grid_n, dx)
    assert empty.shape == (0,)


def _rotation(rng):
    q = rng.standard_normal(4)
    w, x, y, z = q / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]], np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("n_rot", [0, 1, 8])
@pytest.mark.parametrize("n", [0, 1, 257])
def test_cuda_frame_transform_rotation_counts(built_lib, cuda_dev, n_rot, n):
    from pixie_b200.frame_export import render_frame_transform
    rng = np.random.default_rng(10 * n_rot + n)
    pos = rng.uniform(0.5, 1.5, (n, 3)).astype(np.float32)
    A = rng.standard_normal((n, 3, 3)).astype(np.float32) * 0.05
    cm = A @ A.transpose(0, 2, 1)
    cov = np.stack([cm[:, 0, 0], cm[:, 0, 1], cm[:, 0, 2], cm[:, 1, 1], cm[:, 1, 2], cm[:, 2, 2]], axis=1).astype(np.float32)
    Rs = [_rotation(rng) for _ in range(n_rot)]
    mean, scale, zs = np.array([0.2, -0.1, 0.05], np.float32), float(np.float32(0.43)), float(np.float32(0.07))
    p, c = render_frame_transform(torch.from_numpy(pos).to(cuda_dev), torch.from_numpy(cov).to(cuda_dev), zs, scale, mean.tolist(),
                                  [torch.from_numpy(r) for r in Rs])
    wp, wc = FR.render_frame_transform(pos, cov, zs, scale, mean, Rs)
    assert p.shape == (n, 3) and c.shape == (n, 6)
    if n == 0:
        return
    # float32 on the device against fp64, with mag = the largest coordinate before the rotations (|v|_2 <= sqrt(3) mag):
    # the shift, division and mean are 3 roundings per coordinate (<= 6 ulps of mag in the 2-norm); a rotation keeps the
    # norm and adds a 3-term dot product per coordinate, <= 3u |v|_2 each, <= 9 ulps of mag in the 2-norm.
    mag = np.float32(np.abs(mean).max() + (np.abs(pos.astype(np.float64) - 1.0).max() + zs) / scale)
    assert np.abs(p.cpu().numpy() - wp).max() <= (6 + 9 * n_rot) * np.spacing(mag)
    # cov / scale^2: 2 roundings; a rotation is two 3-term products (M R, then R^T (M R)), each <= 9u |M|_F in the
    # Frobenius norm, which it keeps; |M|_F <= magc = 3 max|entry|.
    magc = np.float32(3 * np.abs(cov).max() / np.float32(scale) ** 2)
    assert np.abs(c.cpu().numpy() - wc).max() <= (2 + 18 * n_rot) * np.spacing(magc)


@pytest.mark.gpu
def test_cuda_frame_transform_rejects_nine_rotations(built_lib, cuda_dev):
    from pixie_b200.frame_export import render_frame_transform
    rng = np.random.default_rng(9)
    with pytest.raises(ValueError):
        render_frame_transform(torch.ones((4, 3), device=cuda_dev), None, 0.0, 1.0, [0.0, 0.0, 0.0],
                               [torch.from_numpy(_rotation(rng)) for _ in range(9)])
