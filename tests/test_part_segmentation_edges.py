"""The VLM part segmentation kernels at their edges (csrc/part_segmentation.cu and the two fp64 searches of csrc/nearest.cu),
against the fp64 oracle of oracle/segmentation_ref.py:
  similarity      every part-count tier (PMAX / V = 8 / 4, 16 / 2, 32 / 2, 64 / 1) at its edges P = 8, 9, 16, 17, 32, 33, 63;
                  C from 1 to 768, with the one-channel last tile of C = 257; every remainder of a block's 8 V voxels; with
                  and without a mask, on the 16 B and the 2 B load paths; query tiles re-staged through shared memory in
                  every tier and at the 200 KB residency edge; duplicate and negated queries; temperatures 0.01 to 10;
                  fp16 extremes; with_probs=False; masks that are not boolean.
  k-NN vote       k on both sides of every candidate-buffer doubling (cap = pow2(2k + 32): 128 | 256 | 512 | 1024 | global)
                  on a jittered cloud and a lattice; coincident, doubled, flat, far-apart and tiny point sets; labels on the
                  sorting path, LLONG_MIN and LLONG_MAX (the sort's padding value) included; float64 input.
  nearest vertex  vertices apart by less than float32 resolution, NaN and Inf vertices (a whole leaf of them), finite vertices
                  past the float32 range, non-finite queries, n = 0, n at the leaf edges and a coplanar set.
Bounds are those of tests/test_part_segmentation.py (DESIGN.md section 5): similarities within sim_bound(C) of the fp64
oracle, labels exact outside the ambiguity band, probabilities within (P + 4) ulp of torch's softmax of the kernel's
similarities; the vote and the nearest vertex exact. On the CPU: the oracles against scikit-learn and cKDTree on the new
point sets, and the wrappers' argument checks."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import segmentation_ref as O  # noqa: E402
from pixie_b200 import segmentation as S  # noqa: E402
from test_part_segmentation import DEV, check_outputs, lattice, make_grid  # noqa: E402

gpu = pytest.mark.gpu
F32, F64 = np.float32, np.float64
LLONG_MIN, LLONG_MAX = int(np.iinfo(np.int64).min), int(np.iinfo(np.int64).max)


# ------------------------------------------------------------------------------------------------ similarity: helpers
def group(P: int) -> int:
    """Occupied voxels per block step of the similarity kernel: 8 warps of V voxels."""
    return 8 * (4 if P <= 8 else 2 if P <= 32 else 1)


def resident(P: int, C: int) -> bool:
    """Whether every 256-channel query tile stays in shared memory (P tiles of 1 KiB each, up to 200 KiB)."""
    return (C + 255) // 256 * P * 1024 <= 200 * 1024


def unit(table):
    return S.normalize_queries(torch.from_numpy(table), DEV)


def unaligned(x: torch.Tensor) -> torch.Tensor:
    """x copied one half past 16 B alignment: the 2 B-load path."""
    buf = torch.empty(x.numel() + 1, dtype=x.dtype, device=x.device)
    off = buf[1:].view(x.shape)
    off.copy_(x)
    return off


def pick(N: int, n: int, seed: int) -> np.ndarray:
    m = np.zeros(N, bool)
    m[np.random.default_rng(seed).permutation(N)[:n]] = True
    return m


def rows_near(table, N, seed, part=None, scale=2.0):
    """(N, C) float16 feature rows scale * table[part] + N(0, 1), part random unless given."""
    rng = np.random.default_rng(seed)
    part = rng.integers(0, len(table), N) if part is None else part
    return (scale * table[part] + rng.normal(0, 1, (N, table.shape[1]))).astype(np.float16)


# ------------------------------------------------------------------------------------------------ CPU: wrappers
def test_mask_flags_select_what_bool_selects():
    rng = np.random.default_rng(0)
    fm = rng.choice(np.array([0.0, 0.5, -1.0, np.nan, 1.0, 1e-30, -0.0], F32), (4, 5, 6))
    im = rng.choice(np.array([0, 1, 2, 255, 256, -1, 512], np.int64), (4, 5, 6))
    for m in (torch.from_numpy(fm), torch.from_numpy(fm).half(), torch.from_numpy(im), torch.from_numpy(fm != 0)):
        got = S.mask_flags(m, "cpu")
        assert got.dtype == torch.uint8 and got.is_contiguous() and got.shape == (m.numel(),)
        assert torch.equal(got, m.reshape(-1).bool().to(torch.uint8))
    for m, v in ((fm, 0.5), (im, 256)):                          # the entries a direct uint8 cast turns into 0
        assert (m == v).any() and S.mask_flags(torch.from_numpy(m), "cpu")[torch.from_numpy((m == v).reshape(-1))].all()


def test_vote_argument_checks_before_device():
    c, lab = torch.zeros(5, 3), torch.zeros(5, dtype=torch.int64)
    for k in (0, -1):
        with pytest.raises(ValueError, match="k must be"):
            S.knn_label_vote(c, lab, k)
    with pytest.raises(ValueError, match="n_neighbors"):
        S.knn_label_vote(c, lab, 6)
    with pytest.raises(ValueError, match="n_neighbors"):
        S.knn_label_vote(torch.zeros(0, 3), torch.zeros(0, dtype=torch.int64), 1)
    for bad in (torch.zeros(5, 2), torch.zeros(5, 4), torch.zeros(15)):
        with pytest.raises(ValueError, match="coords"):
            S.knn_label_vote(bad, lab, 1)
    for bad in (torch.zeros(4, dtype=torch.int64), torch.zeros(6, dtype=torch.int64), torch.zeros(5, 1, dtype=torch.int64)):
        with pytest.raises(ValueError, match="labels"):
            S.knn_label_vote(c, bad, 1)


def test_nearest_vertex_shape_checks_before_device():
    with pytest.raises(ValueError, match="vertices"):
        S.nearest_vertex(np.zeros((4, 2)), torch.zeros(3, 3))
    with pytest.raises(ValueError, match="vertices"):
        S.nearest_vertex(np.zeros(12), torch.zeros(3, 3))
    with pytest.raises(ValueError, match="vertices"):
        S.nearest_vertex(np.zeros((4, 3)), torch.zeros(9))


# ------------------------------------------------------------------------------------------------ GPU: similarity
TIER_PS = (8, 9, 16, 17, 32, 33, 63)
TIER_CS = (1, 7, 8, 256, 257, 768)


@gpu
@pytest.mark.parametrize("C", TIER_CS)
@pytest.mark.parametrize("P", TIER_PS)
def test_similarity_tiers(cuda_dev, P, C):
    """Every tier at its edges, with a mask and without, aligned (16 B loads where C % 8 == 0) and one half off (2 B loads):
    the oracle's bounds, and the two load paths bit for bit."""
    feats, _, table = make_grid(7, C, P, "full", seed=P * 1000 + C)
    f = torch.from_numpy(feats).to(cuda_dev).reshape(-1, C)
    q = unit(table)
    g = group(P)
    m = torch.from_numpy(pick(len(f), 4 * g + (P + C) % g, P + C)).to(cuda_dev)
    n_rows = g + (3 * P + C) % g
    outs = []
    for x in (f, unaligned(f)):
        a = S.part_similarity(x, q, 0.1, mask=m)
        check_outputs(x[m], table, 0.1, *a)
        b = S.part_similarity(x[:n_rows], q, 0.1)
        check_outputs(x[:n_rows], table, 0.1, *b)
        outs.append(a + b)
    for u, v in zip(*outs):
        assert torch.equal(u, v)


@gpu
@pytest.mark.parametrize("C", (256, 257))
@pytest.mark.parametrize("P", (8, 16, 32, 63))
def test_similarity_every_group_remainder(cuda_dev, P, C):
    """n = 1 .. 2 * 8V occupied voxels: counts below one block step, and every remainder of the last one."""
    g = group(P)
    feats, _, table = make_grid(6, C, P, "full", seed=7 * P + C)
    f = torch.from_numpy(feats).to(cuda_dev).reshape(-1, C)
    q = unit(table)
    for n in range(1, 2 * g + 1):
        m = torch.from_numpy(pick(len(f), n, n)).to(cuda_dev)
        check_outputs(f[m], table, 0.1, *S.part_similarity(f, q, 0.1, mask=m))


@gpu
@pytest.mark.parametrize("P,C", [(9, 6000), (26, 2048), (8, 6656), (50, 1024), (51, 1024)])
def test_similarity_query_residency(cuda_dev, P, C):
    """Query tiles re-staged per voxel group in tiers 16, 32, 8 and 64, and exactly at the 200 KiB residency limit."""
    assert resident(P, C) == (P == 50)
    feats, mask, table = make_grid(8, C, P, "ragged", seed=P * 31 + C)
    f = torch.from_numpy(feats).to(cuda_dev).reshape(-1, C)
    m = torch.from_numpy(mask).to(cuda_dev).reshape(-1)
    check_outputs(f[m], table, 0.1, *S.part_similarity(f, unit(table), 0.1, mask=m))


@gpu
def test_similarity_resident_and_restaged_agree(cuda_dev):
    """The same rows against 50 queries (resident, 200 KiB) and the same 50 plus one (re-staged): both within the oracle's
    bounds, and the 50 shared similarity columns bit-identical (one FMA order, one shuffle tree)."""
    C = 1024
    feats, mask, table = make_grid(8, C, 51, "ragged", seed=5)
    f = torch.from_numpy(feats).to(cuda_dev).reshape(-1, C)
    m = torch.from_numpy(mask).to(cuda_dev).reshape(-1)
    q = unit(table)
    a = S.part_similarity(f, q[:50].contiguous(), 0.1, mask=m)
    b = S.part_similarity(f, q, 0.1, mask=m)
    check_outputs(f[m], table[:50], 0.1, *a)
    check_outputs(f[m], table, 0.1, *b)
    assert torch.equal(a[0], b[0][:, :50])


@gpu
@pytest.mark.parametrize("P,a,b,c", [(8, 2, 4, 0), (16, 9, 11, 3), (32, 20, 22, 5), (64, 40, 42, 10)])
def test_similarity_duplicate_and_negated_queries(cuda_dev, P, a, b, c):
    """Query a + 1 repeats query a and query b is -query c. Every part runs through the same FMA chain and shuffle tree, so
    the duplicate columns are bit-identical, the negated ones exact negatives, and the label goes to the lower duplicate."""
    rng = np.random.default_rng(P)
    C, N = 256, 400
    table = rng.normal(0, 1, (P, C)).astype(F32)
    table[a + 1] = table[a]
    table[b] = -table[c]
    part = rng.integers(0, P, N)
    part[: N // 2] = a
    f = torch.from_numpy(rows_near(table, N, P, part)).to(cuda_dev)
    sims, labels, scores, probs = S.part_similarity(f, unit(table), 0.1)
    check_outputs(f, table, 0.1, sims, labels, scores, probs)
    assert torch.equal(sims[:, a], sims[:, a + 1]) and torch.equal(probs[:, a], probs[:, a + 1])
    assert torch.equal(sims[:, b], -sims[:, c])
    assert (labels == a).sum().item() >= N // 4 and not (labels == a + 1).any()


@gpu
@pytest.mark.parametrize("T", (0.01, 0.1, 1.0, 10.0))
@pytest.mark.parametrize("P", (8, 33))
def test_similarity_temperatures(cuda_dev, P, T):
    """Temperatures 0.01 to 10. Query 1 is -query 0 and many rows sit close to query 0, so at T = 0.01 their softmax
    underflows to exact zeros."""
    rng = np.random.default_rng(int(T * 100) + P)
    table = rng.normal(0, 1, (P, 300)).astype(F32)
    table[1] = -table[0]
    part = rng.integers(0, P, 500)
    part[::2] = 0
    f = torch.from_numpy(rows_near(table, 500, P, part, scale=4.0)).to(cuda_dev)
    sims, labels, scores, probs = S.part_similarity(f, unit(table), T)
    check_outputs(f, table, T, sims, labels, scores, probs)
    if T == 0.01:
        assert (torch.softmax(sims / T, dim=1) == 0).any() and (probs == 0).any()


@gpu
@pytest.mark.parametrize("P", (7, 40))
def test_similarity_fp16_extremes(cuda_dev, P):
    """Rows of +-65504, of subnormal halves, and both mixed, within the oracle's bounds; a row with a +-Inf element gives
    NaN similarities and probabilities, label 0 and a NaN score, as torch's expression does."""
    rng = np.random.default_rng(P)
    C = 264
    table = rng.normal(0, 1, (P, C)).astype(F32)
    big = np.float16(65504)
    sub = (rng.integers(1, 1024, C) * 2.0 ** -24 * rng.choice([-1, 1], C)).astype(np.float16)     # every subnormal half
    special = [np.full(C, big), big * np.where(np.arange(C) % 2, 1, -1).astype(np.float16), sub,
               np.where(np.arange(C) == 17, big, sub).astype(np.float16), np.where(np.arange(C) == 3, np.float16(2.0 ** -24), 0),
               np.full(C, np.float16(-1023 * 2.0 ** -24)), np.where(np.arange(C) < 8, -big, sub).astype(np.float16)]
    inf_rows = [rows_near(table, 1, 1)[0], np.full(C, big)]
    inf_rows[0][5], inf_rows[1][C - 1] = np.inf, -np.inf
    feats = np.concatenate([rows_near(table, 40, P), np.stack(special), np.stack(inf_rows)]).astype(np.float16)
    assert np.all(np.abs(sub) < 2.0 ** -14) and np.all(sub != 0)
    f = torch.from_numpy(feats).to(cuda_dev)
    sims, labels, scores, probs = S.part_similarity(f, unit(table), 0.1)
    fin = len(feats) - len(inf_rows)
    check_outputs(f[:fin], table, 0.1, sims[:fin], labels[:fin], scores[:fin], probs[:fin])
    x = f[fin:].float()
    p_t = torch.softmax(((x / x.norm(dim=-1, keepdim=True)) @ unit(table).T) / 0.1, dim=1)
    assert torch.isnan(sims[fin:]).all() and torch.isnan(probs[fin:]).all() and torch.isnan(scores[fin:]).all()
    assert labels[fin:].tolist() == [0, 0] == torch.argmax(p_t, dim=1).tolist()


@gpu
@pytest.mark.parametrize("P", (8, 17, 64))
def test_similarity_without_probs_is_bit_identical(cuda_dev, P):
    """with_probs=False (the command line's call, with the caller's count) gives the same similarities, labels and scores."""
    feats, mask, table = make_grid(8, 300, P, "ragged", seed=P + 11)
    f = torch.from_numpy(feats).to(cuda_dev)
    m = torch.from_numpy(mask).to(cuda_dev)
    q = unit(table)
    a = S.part_similarity(f, q, 0.1, mask=m)
    b = S.part_similarity(f, q, 0.1, mask=torch.from_numpy(mask), n_occupied=int(mask.sum()), with_probs=False)
    assert b[3] is None
    for x, y in zip(a[:3], b[:3]):
        assert torch.equal(x, y)


@gpu
def test_similarity_float_mask_selects_as_bool(cuda_dev):
    """A float mask of 0.5, -1 and NaN entries, and an integer one with 256, select the rows that mask.bool() selects."""
    rng = np.random.default_rng(21)
    feats, _, table = make_grid(8, 64, 9, "full", seed=21)
    f = torch.from_numpy(feats).to(cuda_dev)
    q = unit(table)
    fm = rng.choice(np.array([0.0, 0.5, -1.0, np.nan, 1.0], F32), (8, 8, 8))
    im = rng.choice(np.array([0, 256, -1, 1, 512], np.int64), (8, 8, 8))
    for m, v in ((torch.from_numpy(fm), 0.5), (torch.from_numpy(im), 256)):
        bm = m.bool()
        a = S.part_similarity(f, q, 0.1, mask=m.to(cuda_dev))
        b = S.part_similarity(f, q, 0.1, mask=bm.to(cuda_dev))
        assert (m == v).any() and a[0].shape[0] == int(bm.sum())
        for x, y in zip(a, b):
            assert torch.equal(x, y)
        check_outputs(f.reshape(-1, 64)[bm.reshape(-1).to(cuda_dev)], table, 0.1, *a)


# ------------------------------------------------------------------------------------------------ k-NN vote: point sets
VOTE_KS = (31, 32, 33, 47, 48, 49, 111, 112, 113, 240, 241, 496, 497)


def cloud(n, seed):
    """Jittered float32 points in [-1, 1]^3 with spatially coherent labels in [0, 5), a quarter of them random."""
    rng = np.random.default_rng(seed)
    pts = rng.uniform(-1.0, 1.0, (n, 3)).astype(F32)
    labels = ((pts[:, 0] > 0).astype(np.int64) + 2 * (pts[:, 1] > 0.3)) % 5
    return pts, np.where(rng.uniform(size=n) < 0.25, rng.integers(0, 5, n), labels).astype(np.int64)


def coincident():
    """1000 copies of one point: every distance ties, so every vote is the mode of labels[:k]."""
    return np.tile(np.array([[0.25, -0.5, 0.125]], F32), (1000, 1)), np.random.default_rng(1).integers(0, 6, 1000)


def doubled():
    """A cloud followed by its own reverse, the copies labelled independently: which of two equal points is kept matters."""
    c, l1 = cloud(2000, 2)
    return np.concatenate([c, c[::-1]]), np.concatenate([l1, np.random.default_rng(3).integers(0, 5, 2000)])


def plane():
    """A 48 x 48 x 1 lattice: the Morton scale of the flat axis is 0."""
    x = np.linspace(-0.7, 0.6, 48, dtype=F32)
    g = np.stack(np.meshgrid(x, x, indexing="ij"), -1).reshape(-1, 2)
    pts = np.column_stack([g, np.full(len(g), 0.3, F32)]).astype(F32)
    rng = np.random.default_rng(4)
    labels = (g[:, 0] > 0).astype(np.int64) * 2 + (g[:, 1] > 0.2)
    return pts, np.where(rng.uniform(size=len(g)) < 0.3, rng.integers(0, 4, len(g)), labels).astype(np.int64)


def line():
    """1500 collinear points at exact spacing 2^-8: each interior point has two neighbours at every distance."""
    x = (np.arange(1500) * 2.0 ** -8 - 2.0).astype(F32)
    pts = np.column_stack([x, np.full(1500, 0.5, F32), np.full(1500, -0.25, F32)]).astype(F32)
    return pts, np.random.default_rng(5).integers(0, 4, 1500)


def far_clusters():
    """Two 10^3 lattices at spacing 2^-10 (~1e-3), 1e4 apart in x, every coordinate exact in float32."""
    i = np.arange(10) * 2.0 ** -10
    g = np.stack(np.meshgrid(i, i, i, indexing="ij"), -1).reshape(-1, 3)
    pts64 = np.concatenate([g, g + np.array([1e4, 0.0, 0.0])])
    pts = pts64.astype(F32)
    assert np.array_equal(pts.astype(F64), pts64)
    return pts, np.random.default_rng(6).integers(0, 4, len(pts))


DEGENERATE_SETS = {"coincident": coincident, "doubled": doubled, "plane": plane, "line": line, "far": far_clusters}
DEGENERATE = [("coincident", k) for k in (1, 33, 200, 497)] + [("doubled", k) for k in (1, 2, 33, 200, 497)] + \
             [("plane", k) for k in (5, 9, 33, 200, 497)] + [("line", k) for k in (2, 3, 33, 200, 497)] + \
             [("far", k) for k in (1, 33, 497, 1000, 1001, 1500)]


@pytest.fixture(scope="module")
def sweep_sets():
    """The jittered cloud and the dense lattice of the k sweep, with the oracle's neighbour table up to max(k) + 1."""
    sets = {"cloud": cloud(4000, 11), "lattice": lattice(16, "solid", seed=5)}
    return {name: (c, lab, O.knn_table(c, max(VOTE_KS) + 1)) for name, (c, lab) in sets.items()}


@pytest.fixture(scope="module")
def degenerate_sets():
    out = {}
    for name, make in DEGENERATE_SETS.items():
        c, lab = make()
        kmax = max(k for n, k in DEGENERATE if n == name)
        out[name] = (c, lab, O.knn_table(c, kmax + 1))
    return out


def device_vote(coords, labels, k, dev):
    return S.knn_label_vote(torch.from_numpy(np.ascontiguousarray(coords)).to(dev), torch.from_numpy(np.asarray(labels, np.int64)).to(dev),
                            k).cpu().numpy()


# ------------------------------------------------------------------------------------------------ CPU: vote oracle
@pytest.mark.parametrize("name,k", DEGENERATE)
def test_oracle_vote_matches_scikit_learn_on_degenerate_sets(degenerate_sets, name, k):
    """The brute-force vote is scikit-learn's wherever the k-th distance is not tied; on the coincident set it is the mode of
    labels[:k] everywhere."""
    c, lab, (idx, dist) = degenerate_sets[name]
    want = O.vote_of(lab, idx[:, :k])
    clear = O.gap_of(dist, k)
    if len(c) <= 2000:                                          # the table's prefixes are the per-k oracles
        assert np.array_equal(want, O.vote_exact(c, lab, k)) and np.array_equal(clear, O.kth_distance_gap(c, k))
    if clear.any():
        assert np.array_equal(want[clear], O.vote_reference(c, lab, k)[clear])
    if name == "coincident":
        vals, counts = np.unique(lab[:k], return_counts=True)
        assert not clear.any() and (want == vals[np.argmax(counts)]).all()


# ------------------------------------------------------------------------------------------------ GPU: k-NN vote
@gpu
@pytest.mark.parametrize("k", VOTE_KS)
@pytest.mark.parametrize("name", ("cloud", "lattice"))
def test_vote_k_at_buffer_edges(cuda_dev, sweep_sets, name, k):
    """k on both sides of each doubling of the candidate buffer and of its move from shared to global memory (k = 496 | 497)."""
    c, lab, (idx, dist) = sweep_sets[name]
    got = device_vote(c, lab, k, cuda_dev)
    assert np.array_equal(got, O.vote_of(lab, idx[:, :k]))
    clear = O.gap_of(dist, k)
    assert clear.any()
    assert np.array_equal(got[clear], O.vote_reference(c, lab, k)[clear])


@gpu
@pytest.mark.parametrize("name,k", DEGENERATE)
def test_vote_on_degenerate_sets(cuda_dev, degenerate_sets, name, k):
    c, lab, (idx, _) = degenerate_sets[name]
    assert np.array_equal(device_vote(c, lab, k, cuda_dev), O.vote_of(lab, idx[:, :k]))


@gpu
@pytest.mark.parametrize("n", (1, 5, 31, 32, 33))
def test_vote_small_sets(cuda_dev, n):
    """Fewer points than a leaf, one leaf exactly and one past it, with k = n and k = n - 1."""
    c, lab = cloud(n, seed=n)
    for k in sorted({n, max(n - 1, 1)}):
        got = device_vote(c, lab, k, cuda_dev)
        assert np.array_equal(got, O.vote_exact(c, lab, k))
        clear = O.kth_distance_gap(c, k)
        assert np.array_equal(got[clear], O.vote_reference(c, lab, k)[clear])


@gpu
@pytest.mark.parametrize("k", (1, 33, 700))
def test_vote_labels_on_the_sorting_path(cuda_dev, k):
    """Labels outside [0, 256) are counted by sorting: shifted, negative, one 256 among small labels (only the queries that
    see it leave the histogram), and labels taking LLONG_MIN and LLONG_MAX."""
    c, lab = cloud(1500, seed=7)
    idx = O.knn_exact(c, k)
    rng = np.random.default_rng(k)
    extreme = rng.choice(np.array([LLONG_MIN, -1, 0, 3, LLONG_MAX], np.int64), len(lab))
    for labels in (lab * 1000 - 7, lab - 9, np.where(np.arange(len(lab)) == 777, 256, lab), extreme):
        assert np.array_equal(device_vote(c, labels, k, cuda_dev), O.vote_of(labels, idx))


@gpu
def test_vote_extreme_labels_mode_and_count_tie(cuda_dev):
    """k = n = 100 (the sort pads 28 slots): LLONG_MAX, the padding value, wins as the mode; loses a count tie to a smaller
    label; and LLONG_MIN wins as the mode."""
    c, _ = cloud(100, seed=9)
    rng = np.random.default_rng(9)
    cases = [([LLONG_MAX] * 40 + [LLONG_MIN] * 35 + [7] * 25, LLONG_MAX), ([LLONG_MAX] * 40 + [3] * 40 + [LLONG_MIN] * 20, 3),
             ([LLONG_MIN] * 45 + [LLONG_MAX] * 30 + [300] * 25, LLONG_MIN)]
    for labels, mode in cases:
        labels = rng.permutation(np.array(labels, np.int64))
        assert (device_vote(c, labels, 100, cuda_dev) == mode).all()
    c3, _ = cloud(300, seed=10)
    labels = rng.choice(np.array([LLONG_MIN, LLONG_MAX, 5], np.int64), 300)
    assert np.array_equal(device_vote(c3, labels, 100, cuda_dev), O.vote_exact(c3, labels, 100))


@gpu
def test_vote_rounds_float64_coordinates_to_float32(cuda_dev):
    """float64 coordinates a sub-ulp away from a float32 lattice vote as the lattice itself, ties included."""
    c32, lab = lattice(10, "solid", seed=3)
    c64 = c32.astype(F64) + np.random.default_rng(3).uniform(-1e-12, 1e-12, c32.shape)
    assert np.array_equal(c64.astype(F32), c32) and not np.array_equal(c64, c32.astype(F64))
    got = S.knn_label_vote(torch.from_numpy(c64).to(cuda_dev), torch.from_numpy(lab).to(cuda_dev), 33).cpu().numpy()
    assert np.array_equal(got, O.vote_exact(c32, lab, 33))
    assert not O.kth_distance_gap(c32, 33).all()


# ------------------------------------------------------------------------------------------------ nearest vertex: sets
FLT_MAX = float(np.finfo(F32).max)
BAD_QUERIES = np.array([[np.nan, 0, 0], [0, np.inf, 0], [0, 0, -np.inf], [np.nan] * 3], F32)


def sub_float32_set(m=400, seed=1):
    """Around each float32 query q, four fp64 vertices q + delta u, delta = 1e-9, 3e-10, 1e-10, 1e-12, all rounding to q in
    float32; the nearest has the highest index of the four. 2000 ordinary vertices come first."""
    rng = np.random.default_rng(seed)
    q = (rng.uniform(0.5, 1.0, (m, 3)) * rng.choice([-1.0, 1.0], (m, 3))).astype(F32)
    u = rng.normal(size=(m, 4, 3))
    u /= np.linalg.norm(u, axis=-1, keepdims=True)
    near = q[:, None, :].astype(F64) + np.array([1e-9, 3e-10, 1e-10, 1e-12])[None, :, None] * u
    assert (near.astype(F32) == q[:, None, :]).all()
    v = np.concatenate([rng.uniform(-1, 1, (2000, 3)), near.reshape(-1, 3)])
    return v, q, 2000 + 4 * np.arange(m) + 3


def nonfinite_set(seed=2):
    """3000 finite vertices and 80 with NaN or +-Inf coordinates: 40 before every finite one (the lowest indices) and 40
    among them; sorted last, they fill whole leaves. The queries include the finite parts of the non-finite vertices."""
    rng = np.random.default_rng(seed)
    bad = rng.uniform(-1, 1, (80, 3))
    kinds = np.array([np.nan, np.inf, -np.inf])
    for r in range(80):
        bad[r, r % 3] = kinds[r % 3]
        if r % 5 == 0:
            bad[r, (r + 1) % 3] = kinds[(r + 1) % 3]
    fin = rng.uniform(-1, 1, (3000, 3))
    v = np.concatenate([bad[:40], fin[:1500], bad[40:], fin[1500:]])
    q = np.concatenate([rng.uniform(-1.2, 1.2, (1500, 3)), np.nan_to_num(bad, nan=0.1, posinf=0.2, neginf=-0.2)]).astype(F32)
    return v, q


def far_sets():
    """Finite vertices past the float32 range: with an ordinary cloud; alone (the +-1e39 ones are nearest); and only 1e300
    magnitudes behind a NaN and an Inf vertex, where every d2 overflows to Inf and the lowest finite index (2) is nearest."""
    rng = np.random.default_rng(3)
    far = np.array([[1e39, 0, 0], [-1e39, 0.5, 0], [0, 1e300, 0], [0, 0, -1e300], [1e300, 1e300, 1e300], [-1e300, 0, 0],
                    [0, -1e39, 1e39]])
    q = np.concatenate([rng.uniform(-2, 2, (300, 3)),
                        [[FLT_MAX, 0, 0], [-FLT_MAX, 0, 0], [0, FLT_MAX, -FLT_MAX], [FLT_MAX] * 3, [0, -FLT_MAX, FLT_MAX]]]).astype(F32)
    overflow = np.concatenate([[[np.nan, 0, 0], [0, np.inf, 0]], far[2:6]])
    return {"with_cloud": (np.concatenate([rng.uniform(-1, 1, (500, 3)), far]), q), "alone": (far, q), "overflow": (overflow, q)}


def small_and_flat_sets():
    rng = np.random.default_rng(4)
    sets = {f"n{n}": rng.uniform(-1, 1, (n, 3)) for n in (1, 31, 32, 33)}
    xy = rng.uniform(-1, 1, (3000, 2))
    sets["coplanar"] = np.column_stack([xy, np.full(3000, 0.25)])
    g = np.linspace(-1, 1, 20)
    sets["coplanar_lattice"] = np.column_stack([np.stack(np.meshgrid(g, g, indexing="ij"), -1).reshape(-1, 2), np.zeros(400)])
    return sets, rng.uniform(-1.2, 1.2, (1000, 3)).astype(F32)


def kdtree_agrees(v, q, want):
    """cKDTree over the finite vertices gives the oracle's index wherever its distance is finite and the nearest is unique."""
    from scipy.spatial import cKDTree
    ok = np.isfinite(v).all(1)
    fin = np.flatnonzero(ok)
    qf = np.isfinite(q).all(1)
    d, i = cKDTree(v[ok]).query(q[qf].astype(F64), k=2 if ok.sum() > 1 else 1)
    d, i = d.reshape(len(d), -1), i.reshape(len(i), -1)
    unique = np.isfinite(d[:, 0]) & ((d[:, 0] < d[:, 1]) if d.shape[1] > 1 else True)
    assert unique.any()
    assert np.array_equal(fin[i[unique, 0]], want[qf][unique])


# ------------------------------------------------------------------------------------------------ CPU: nearest-vertex oracle
def test_oracle_nearest_on_edge_sets():
    v, q, nearest = sub_float32_set()
    want = O.nearest_exact(v, q)
    assert np.array_equal(want, nearest)
    kdtree_agrees(v, q, want)
    v, q = nonfinite_set()
    want = O.nearest_exact(v, q)
    assert np.isfinite(v[want]).all()
    kdtree_agrees(v, q, want)
    for name, (v, q) in far_sets().items():
        want = O.nearest_exact(v, q)
        if name == "overflow":
            assert (want == 2).all()
        else:
            kdtree_agrees(v, q, want)
    sets, q = small_and_flat_sets()
    for name, v in sets.items():
        if name != "coplanar_lattice":
            kdtree_agrees(v, q, O.nearest_exact(v, q))
    assert (O.nearest_exact(np.zeros((0, 3)), q) == -1).all()
    assert (O.nearest_exact(sets["n33"], BAD_QUERIES) == -1).all()
    assert (O.nearest_exact(np.full((40, 3), np.nan), q) == -1).all()


# ------------------------------------------------------------------------------------------------ GPU: nearest vertex
def device_nearest(v, q, dev):
    return S.nearest_vertex(v, torch.from_numpy(np.ascontiguousarray(q)).to(dev)).numpy()


@gpu
def test_nearest_vertex_below_float32_resolution(cuda_dev):
    """Vertices that share one float32 point are told apart by their fp64 coordinates."""
    v, q, nearest = sub_float32_set()
    assert np.array_equal(device_nearest(v, q, cuda_dev), nearest)


@gpu
def test_nearest_vertex_non_finite_vertices_never_win(cuda_dev):
    v, q = nonfinite_set()
    got = device_nearest(v, q, cuda_dev)
    assert np.array_equal(got, O.nearest_exact(v, q)) and np.isfinite(v[got]).all()
    assert (device_nearest(np.full((70, 3), np.nan), q, cuda_dev) == -1).all()
    assert (device_nearest(np.tile([[np.inf, 0, 0], [0, -np.inf, 0]], (40, 1)), q, cuda_dev) == -1).all()


@gpu
@pytest.mark.parametrize("name", ("with_cloud", "alone", "overflow"))
def test_nearest_vertex_past_float32_range(cuda_dev, name):
    """Finite vertices at +-1e39 and +-1e300 are candidates like any other, also where their d2 overflows to Inf."""
    v, q = far_sets()[name]
    got = device_nearest(v, q, cuda_dev)
    assert np.array_equal(got, O.nearest_exact(v, q))
    if name == "overflow":
        assert (got == 2).all()


@gpu
def test_nearest_vertex_non_finite_queries_and_no_vertices(cuda_dev):
    v, q = nonfinite_set()
    mixed = np.concatenate([q[:100], BAD_QUERIES, q[100:200]])
    got = device_nearest(v, mixed, cuda_dev)
    assert np.array_equal(got, O.nearest_exact(v, mixed))
    assert (got[100:104] == -1).all() and (got[:100] >= 0).all()
    assert (device_nearest(np.zeros((0, 3)), q, cuda_dev) == -1).all()


@gpu
@pytest.mark.parametrize("name", ("n1", "n31", "n32", "n33", "coplanar", "coplanar_lattice"))
def test_nearest_vertex_small_and_flat_sets(cuda_dev, name):
    sets, q = small_and_flat_sets()
    v = sets[name]
    assert np.array_equal(device_nearest(v, q, cuda_dev), O.nearest_exact(v, q))
