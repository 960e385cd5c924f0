"""The VLM part segmentation (pixie_b200.segmentation, csrc/part_segmentation.cu and the searches of csrc/nearest.cu):
the fp64 oracle against the reference's own outputs (tests/golden/segmentation_golden.npz, make_segmentation_golden.py),
the host side and the command line on the CPU; the kernels against the oracle and the reference's expressions, and the
command line end to end, on the GPU."""
import io
import json
import os
import re
import shutil
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import make_segmentation_golden as G  # noqa: E402
from oracle import segmentation_ref as O  # noqa: E402
from pixie_b200 import segmentation as S  # noqa: E402

GOLD = np.load(os.path.join(ROOT, "tests", "golden", "segmentation_golden.npz"))
CASES = G.cases()
U32 = 2.0 ** -24
gpu = pytest.mark.gpu


def occupied_features(c):
    m = c["mask"].astype(bool)
    return c["feats"][m], m


def files_of(d):
    return {f: open(os.path.join(d, f), "rb").read() for f in sorted(os.listdir(d))}


def golden_files(prefix):
    return {k.split("/", 1)[1]: GOLD[k].tobytes() for k in GOLD.files if k.startswith(prefix + "/")}


def golden_labels(prefix):
    return torch.from_numpy(np.load(io.BytesIO(GOLD[f"{prefix}/part_labels.npy"].tobytes())))


def _cpu_nearest(monkeypatch):
    """The device colour lookup replaced by the brute-force oracle, so the host side runs without a GPU."""
    monkeypatch.setattr(S, "nearest_vertex", lambda v, q: torch.from_numpy(O.nearest_exact(v, q.cpu().numpy())))


# ------------------------------------------------------------------------------------------------ CPU: oracle vs reference
@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_similarities_match_reference(name):
    c = CASES[name]
    f, _ = occupied_features(c)
    sims, probs, labels, scores = O.similarities(f, c["table"])
    ref_p, ref_s = GOLD[f"clip64_{name}/probs"], GOLD[f"clip64_{name}/sims"]
    nan = np.isnan(ref_p).any(1)
    assert np.array_equal(np.isnan(probs.numpy()), np.isnan(ref_p)) and np.array_equal(np.isnan(sims.numpy()), np.isnan(ref_s))
    assert np.abs(probs.numpy()[~nan] - ref_p[~nan]).max() <= 1e-12
    assert np.abs(sims.numpy()[~nan] - ref_s[~nan]).max() <= 1e-12
    assert np.array_equal(labels.numpy(), GOLD[f"clip64_{name}/labels32"])        # the fp32 run: no label near a tie
    assert labels.numpy()[nan].tolist() == [0] * int(nan.sum())
    np.testing.assert_allclose(scores.numpy()[~nan], GOLD[f"clip64_{name}/scores32"][~nan], rtol=1e-5)


@pytest.mark.parametrize("k", G.VOTE_KS)
def test_oracle_vote_matches_reference(k):
    coords, labels = G.vote_inputs()
    assert np.array_equal(O.vote_reference(coords, labels, k), GOLD[f"vote_k{k}"])
    assert np.array_equal(O.vote_exact(coords, labels, k), GOLD[f"vote_k{k}"])


def test_smoothing_case_does_not_depend_on_knn_ties():
    """The golden smoothing case is one where the vote with the k nearest by (distance, index) equals scikit-learn's, whichever
    of the points tied at the 200th distance its tree keeps: there the device vote must write the reference's bytes."""
    c = CASES["smooth"]
    f, m = occupied_features(c)
    labels = O.similarities(f, c["table"])[2].numpy()
    lo, hi = c["bounds"]
    axes = [torch.linspace(lo[i], hi[i], c["D"]).numpy() for i in range(3)]
    idx = np.argwhere(m)
    coords = np.stack([axes[a][idx[:, a]] for a in range(3)], 1)
    assert (~O.kth_distance_gap(coords, 200)).any()               # ties at the 200th distance exist ...
    assert np.array_equal(O.vote_exact(coords, labels, 200), O.vote_reference(coords, labels, 200))     # ... and change no vote


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_files_match_reference(tmp_path, name):
    """The oracle's pipeline (fp64 labels, scikit-learn vote, cKDTree colours) writes the reference's bytes."""
    c = CASES[name]
    f, m = occupied_features(c)
    _, _, labels, _ = O.similarities(f, c["table"])
    labels = labels.numpy()
    lo, hi = c["bounds"]
    axes = [torch.linspace(lo[i], hi[i], c["D"]).numpy() for i in range(3)]
    idx = np.argwhere(m)
    coords = np.stack([axes[a][idx[:, a]] for a in range(3)], 1)
    if c["smooth"]:
        labels = O.vote_reference(coords, labels, 200)
    cols = np.column_stack([c["colors"], np.full(len(c["colors"]), 255, np.uint8)])
    O.save_files(coords, labels, str(tmp_path), c["verts"], cols, list(c["props"]), c["props"], (c["D"],) * 3, c["mask"])
    got = files_of(tmp_path)
    want = golden_files(f"cli_{name}")
    want.pop("part_labels.npy")
    assert got.keys() == want.keys()
    for k in want:
        assert got[k] == want[k], k


def test_str2bool_matches_reference():
    import argparse
    got = []
    for v in G.STR2BOOL_INPUTS:
        try:
            got.append(int(S.str2bool(v)))
        except argparse.ArgumentTypeError:
            got.append(-1)
    assert got == GOLD["str2bool"].tolist()
    assert S.str2bool(True) is True and S.str2bool(False) is False


def test_tab10_is_matplotlibs():
    assert S.TAB10 == [G._Colormap()(i) for i in range(10)]


# ------------------------------------------------------------------------------------------------ CPU: host side, command line
def test_cached_labels_path_reads_labels_and_ply(tmp_path, monkeypatch):
    """part_labels.npy present and --overwrite false: the labels are read, the coordinates come from the occupancy PLY, and
    every file is the reference's."""
    _cpu_nearest(monkeypatch)
    real = S.load_occupancy_grid
    monkeypatch.setattr(S, "load_occupancy_grid", lambda p, device="cuda": real(p, device="cpu"))
    monkeypatch.setattr(S, "clip_part_segmentation", lambda *a, **k: pytest.fail("the cached path ran the segmentation"))
    p = G.write_inputs(CASES["plain"], str(tmp_path / "in"))
    od = tmp_path / "out"
    od.mkdir()
    (od / "part_labels.npy").write_bytes(GOLD["cache/part_labels.npy"].tobytes())
    S.main(["--grid_feature_path", p["grid"], "--occupancy_path", p["occ"], "--output_dir", str(od), "--material_dict_path", p["mat"],
            "--overwrite", "False", "--query_embeddings", p["emb"]])
    assert files_of(od) == golden_files("cache")


def test_host_writer_matches_reference(tmp_path, monkeypatch):
    """save_segmented_point_cloud from the reference's labels and the grid's coordinates writes the reference's bytes."""
    _cpu_nearest(monkeypatch)
    for name, c in CASES.items():
        p = G.write_inputs(c, str(tmp_path / name))
        labels = golden_labels(f"cli_{name}")
        with np.load(p["grid"]) as md:
            coords = S._grid_coords(md["min_bounds"], md["max_bounds"], md["grid_shape"], "cpu")[torch.from_numpy(c["mask"].astype(bool))]
        od = tmp_path / f"{name}_out"
        S.save_segmented_point_cloud(coords, labels, str(od), original_pc_path=p["occ"], part_queries=list(c["props"]),
                                     material_props=c["props"], grid_feature_path=p["grid"])
        want = golden_files(f"cli_{name}")
        want.pop("part_labels.npy")
        assert files_of(od) == want


def test_segmented_cloud_equals_semantics_ply(tmp_path, monkeypatch):
    from pixie_b200 import scene_files as SF
    _cpu_nearest(monkeypatch)
    c = CASES["smooth"]
    p = G.write_inputs(c, str(tmp_path / "in"))
    labels = golden_labels("cli_smooth")
    with np.load(p["grid"]) as md:
        coords = S._grid_coords(md["min_bounds"], md["max_bounds"], md["grid_shape"], "cpu")[torch.from_numpy(c["mask"].astype(bool))]
    S.save_segmented_point_cloud(coords, labels, str(tmp_path / "out"), original_pc_path=p["occ"], part_queries=list(c["props"]),
                                 material_props=c["props"])
    got = S.segmented_point_cloud(coords, labels, list(c["props"]), c["props"], device="cpu")
    ref = SF.load_point_cloud(str(tmp_path / "out" / "segmented_semantics.ply"), device="cpu")
    assert got.keys() == ref.keys()
    for k in ref:
        assert got[k].dtype == ref[k].dtype and torch.equal(got[k], ref[k]), k


def _argv(p, od, *extra):
    return ["--grid_feature_path", p["grid"], "--occupancy_path", p["occ"], "--output_dir", str(od), "--material_dict_path", p["mat"],
            *extra]


@pytest.mark.parametrize("extra", [["--use_spatial_smoothing", "maybe"], ["--overwrite", "2"], ["--background_id", "x"],
                                   ["--no_such_flag", "1"]])
def test_cli_rejects_bad_flags(tmp_path, extra):
    p = G.write_inputs(CASES["plain"], str(tmp_path / "in"))
    with pytest.raises(SystemExit):
        S.main(_argv(p, tmp_path / "out", *extra))
    assert not (tmp_path / "out").exists()


def test_cli_requires_its_paths(tmp_path):
    with pytest.raises(SystemExit):
        S.main(["--grid_feature_path", "a.npz", "--occupancy_path", "b.ply", "--output_dir", str(tmp_path)])


def test_cli_rejects_inputs_before_device_work(tmp_path, monkeypatch):
    monkeypatch.setattr(S, "part_similarity", lambda *a, **k: pytest.fail("device work started"))
    p = G.write_inputs(CASES["plain"], str(tmp_path / "in"))
    od = tmp_path / "out"
    # embeddings with a row count other than the dict's keys
    np.save(tmp_path / "q2.npy", CASES["plain"]["table"][:2])
    with pytest.raises(ValueError, match="one row per key"):
        S.main(_argv(p, od, "--query_embeddings", str(tmp_path / "q2.npy")))
    # embeddings of another width than the features
    np.save(tmp_path / "qw.npy", np.ones((3, 5), np.float32))
    with pytest.raises(ValueError, match="C = 16"):
        S.main(_argv(p, od, "--query_embeddings", str(tmp_path / "qw.npy")))
    # a cached label with no key in the material dict
    od.mkdir()
    np.save(od / "part_labels.npy", np.array([0, 1, 3], np.int64))
    with pytest.raises(ValueError, match="no part"):
        S.main(_argv(p, od, "--query_embeddings", p["emb"]))
    # a missing material dict, and one with no parts
    with pytest.raises(AssertionError, match="does not exist"):
        S.main(_argv(dict(p, mat=str(tmp_path / "none.json")), tmp_path / "o2"))
    (tmp_path / "empty.json").write_text(json.dumps({"material_dict": {}}))
    with pytest.raises(ValueError, match="no parts"):
        S.main(_argv(dict(p, mat=str(tmp_path / "empty.json")), tmp_path / "o3"))
    assert sorted(os.listdir(od)) == ["part_labels.npy"]


def test_cli_without_embeddings_names_the_flag(tmp_path, monkeypatch):
    import builtins
    real = builtins.__import__

    def no_f3rm(name, *a, **k):
        if name.startswith("f3rm"):
            raise ImportError(name)
        return real(name, *a, **k)
    monkeypatch.setattr(builtins, "__import__", no_f3rm)
    monkeypatch.setattr(S, "part_similarity", lambda *a, **k: pytest.fail("device work started"))
    p = G.write_inputs(CASES["plain"], str(tmp_path / "in"))
    with pytest.raises(RuntimeError, match="--query_embeddings"):
        S.main(_argv(p, tmp_path / "out"))


def test_library_exports_segmentation_symbols():
    from pixie_b200 import _lib
    header = open(os.path.join(ROOT, "include", "pixie_b200.h")).read()
    for sym in ("pixie_part_similarity", "pixie_knn_label_vote", "pixie_nearest_vertex"):
        assert re.search(rf"\b{sym}\(", header) and sym in _lib._SIGNATURES
    if os.path.exists(_lib.LIB_PATH):
        lib = _lib.load()
        for sym in ("pixie_part_similarity", "pixie_knn_label_vote", "pixie_nearest_vertex"):
            assert getattr(lib, sym) is not None


def test_vote_rejects_k_above_n():
    with pytest.raises(ValueError, match="n_neighbors"):
        S.knn_label_vote(torch.zeros(5, 3), torch.zeros(5, dtype=torch.int64), k=6)


# ------------------------------------------------------------------------------------------------ GPU: similarity kernel
DEV = "cuda:0"


def sim_bound(C: int) -> float:
    """DESIGN.md: |sim - sim64| <= 2 (2C + 8) 2^-24 for unit queries (fp32 accumulation of C products, the fp32 norm and
    the fp32-normalised queries)."""
    return 2.0 * (2 * C + 8) * U32


def make_grid(D, C, P, kind, seed):
    rng = np.random.default_rng(seed)
    table = rng.normal(0, 1, (P, C)).astype(np.float32)
    part = rng.integers(0, P, (D, D, D))
    feats = (2.0 * table[part] + rng.normal(0, 1, (D, D, D, C))).astype(np.float16)
    if kind == "empty":
        mask = np.zeros((D, D, D), bool)
    elif kind == "one":
        mask = np.zeros((D, D, D), bool)
        mask[D // 2, D - 1, 1] = True
    elif kind == "full":
        mask = np.ones((D, D, D), bool)
    else:
        mask = rng.uniform(size=(D, D, D)) < 0.37
    return feats, mask, table


def _check_similarity(feats, mask, table, T=0.1):
    C = feats.shape[-1]
    f_dev = torch.from_numpy(feats).to(DEV)
    m_dev = torch.from_numpy(mask).to(DEV)
    q = S.normalize_queries(torch.from_numpy(table), DEV)
    sims, labels, scores, probs = S.part_similarity(f_dev, q, T, mask=m_dev)
    check_outputs(f_dev.reshape(-1, C)[m_dev.reshape(-1)], table, T, sims, labels, scores, probs)


def check_outputs(rows, table, T, sims, labels, scores, probs):
    """part_similarity's outputs for the float16 feature rows (n, C) on the device against the fp64 oracle, the label rule
    and torch's softmax of the kernel's similarities."""
    n, C = rows.shape
    assert sims.shape == (n, table.shape[0]) and labels.dtype == torch.int64
    if n == 0:
        return
    s64, _, _, _ = O.similarities(rows, table, T)
    err = (sims.double() - s64).abs().max().item()
    assert err <= sim_bound(C), (err, sim_bound(C))
    # labels: the oracle's wherever the top-two gap is clear of the bound, else one of its two best
    top2 = torch.topk(s64, min(2, s64.shape[1]), dim=1)
    gap = (top2.values[:, 0] - top2.values[:, 1]) if s64.shape[1] > 1 else torch.full((n,), np.inf, device=DEV, dtype=torch.float64)
    clear = gap > 2 * sim_bound(C)
    assert torch.equal(labels[clear], top2.indices[clear, 0])
    if (~clear).any():
        amb = labels[~clear]
        assert ((amb == top2.indices[~clear, 0]) | (amb == top2.indices[~clear, 1])).all()
    # the softmax of the kernel's similarities by the reference's own expression, on the same device
    p_ref = torch.nn.functional.softmax(sims / T, dim=1)
    P = table.shape[0]
    assert ((probs - p_ref).abs() <= (P + 4) * U32 * p_ref + 1e-30).all()
    assert torch.equal(scores, torch.gather(probs, 1, labels[:, None])[:, 0])
    assert torch.equal(labels, torch.argmax(probs, dim=1))


SIM_CASES = [(D, C, P, kind) for C in (512, 768, 100) for P in (1, 2, 7, 64) for D, kind in ((8, "ragged"), (8, "one"))] + \
            [(33, C, P, kind) for C, P in ((768, 7), (100, 64), (512, 2)) for kind in ("empty", "ragged", "full")] + \
            [(64, 768, 7, "ragged"), (64, 512, 64, "full"), (64, 768, 1, "full"), (64, 100, 2, "ragged")] + \
            [(8, 1024, 64, "ragged"), (8, 1000, 64, "full")]          # queries past 200 KB: one tile in shared memory at a time


@gpu
@pytest.mark.parametrize("D,C,P,kind", SIM_CASES)
def test_similarity_against_oracle(D, C, P, kind):
    feats, mask, table = make_grid(D, C, P, kind, seed=D * 1000 + C + P)
    _check_similarity(feats, mask, table)


@gpu
def test_similarity_scalar_path_on_unaligned_features():
    """C % 8 == 0 but the rows start off 16 B alignment: the 2 B-load path, same results as the aligned call."""
    feats, mask, table = make_grid(8, 512, 7, "ragged", seed=9)
    q = S.normalize_queries(torch.from_numpy(table), DEV)
    buf = torch.empty(feats.size + 1, dtype=torch.float16, device=DEV)
    off = buf[1:].view(feats.shape)
    off.copy_(torch.from_numpy(feats))
    a = S.part_similarity(torch.from_numpy(feats).to(DEV), q, 0.1, mask=torch.from_numpy(mask).to(DEV))
    b = S.part_similarity(off, q, 0.1, mask=torch.from_numpy(mask).to(DEV))
    for x, y in zip(a, b):
        assert torch.equal(x, y)


@gpu
def test_similarity_zero_and_nan_rows_behave_as_torch():
    feats, mask, table = make_grid(8, 100, 7, "full", seed=3)
    feats[0, 0, 0] = 0
    feats[1, 2, 3, 5] = np.nan
    flat = torch.from_numpy(feats).to(DEV).reshape(-1, 100)
    q = S.normalize_queries(torch.from_numpy(table), DEV)
    sims, labels, scores, probs = S.part_similarity(flat, q, 0.1)
    f = flat.float()
    f = f / f.norm(dim=-1, keepdim=True)
    p_t = torch.softmax((f @ q.T) / 0.1, dim=1)
    bad = [0, (1 * 8 + 2) * 8 + 3]
    for r in bad:
        assert torch.isnan(sims[r]).all() and torch.isnan(probs[r]).all() and torch.isnan(scores[r])
        assert labels[r].item() == 0 == torch.argmax(p_t[r]).item()
    assert not torch.isnan(sims[1]).any()


@gpu
def test_similarity_rejects_too_many_parts():
    q = torch.ones(65, 16, device=DEV) / 4
    with pytest.raises(ValueError, match="64"):
        S.part_similarity(torch.ones(4, 16, dtype=torch.float16, device=DEV), q)


@gpu
def test_similarity_fp16_accumulation_would_fail_the_bound():
    """The bound is tight enough to catch an fp16 accumulator: emulate one and check it breaks the bound."""
    feats, mask, table = make_grid(8, 768, 7, "full", seed=4)
    rows = torch.from_numpy(feats).to(DEV).reshape(-1, 768)[:256]
    q = S.normalize_queries(torch.from_numpy(table), DEV)
    acc = torch.zeros(rows.shape[0], 7, dtype=torch.float16, device=DEV)
    for c in range(768):
        acc = acc + (rows[:, c:c + 1].float() * q[:, c][None, :]).half()
    sims_h = acc.float() / rows.float().norm(dim=1, keepdim=True)
    s64, _, _, _ = O.similarities(rows, table)
    assert (sims_h.double() - s64).abs().max().item() > sim_bound(768)


# ------------------------------------------------------------------------------------------------ GPU: k-NN vote
@gpu
@pytest.mark.parametrize("k", G.VOTE_KS)
def test_vote_equals_reference_on_jittered_points(k):
    coords, labels = G.vote_inputs()
    got = S.local_post_process_segmentation(torch.from_numpy(coords).to(DEV), torch.from_numpy(labels).to(DEV), k=k)
    assert got.dtype == torch.int64 and got.device.type == "cuda"
    assert np.array_equal(got.cpu().numpy(), GOLD[f"vote_k{k}"])
    assert np.array_equal(got.cpu().numpy(), O.vote_reference(coords, labels, k))


def lattice(D, kind, seed, bounds=((-0.6, -0.5, -0.4), (0.7, 0.5, 0.45))):
    rng = np.random.default_rng(seed)
    lo, hi = bounds
    axes = [torch.linspace(lo[i], hi[i], D) for i in range(3)]
    grid = torch.stack(torch.meshgrid(*axes, indexing="ij"), -1)
    ii = np.indices((D, D, D))
    if kind == "solid":
        m = np.ones((D, D, D), bool)
    elif kind == "shell":
        r = np.sqrt(sum((a - (D - 1) / 2) ** 2 for a in ii))
        m = np.abs(r - D / 3) < 0.5
    else:
        m = rng.uniform(size=(D, D, D)) < 0.5
    coords = grid[torch.from_numpy(m)].numpy()
    labels = ((ii[0] * 3 // D) + (ii[1] * 2 // D))[m] % 4
    flip = rng.uniform(size=len(coords)) < 0.3
    labels = np.where(flip, rng.integers(0, 4, len(coords)), labels).astype(np.int64)
    return coords, labels


@gpu
@pytest.mark.parametrize("D,kind,k", [(12, "solid", 200), (16, "ragged", 200), (24, "shell", 200), (12, "solid", 16), (16, "ragged", 1),
                                      (12, "shell", 27), (10, "ragged", 2)])
def test_vote_on_lattice(D, kind, k):
    coords, labels = lattice(D, kind, seed=D + k)
    got = S.knn_label_vote(torch.from_numpy(coords).to(DEV), torch.from_numpy(labels).to(DEV), k).cpu().numpy()
    assert np.array_equal(got, O.vote_exact(coords, labels, k))
    clear = O.kth_distance_gap(coords, k)
    assert np.array_equal(got[clear], O.vote_reference(coords, labels, k)[clear])


@gpu
@pytest.mark.parametrize("k", (16, 200))
def test_vote_with_labels_outside_the_histogram(k):
    """Labels outside [0, 256) are counted by sorting them; the vote is the same (the map keeps the order of labels)."""
    coords, labels = G.vote_inputs()
    big = labels * 1000 - 7
    got = S.knn_label_vote(torch.from_numpy(coords).to(DEV), torch.from_numpy(big).to(DEV), k).cpu().numpy()
    assert np.array_equal(got, GOLD[f"vote_k{k}"] * 1000 - 7)


@gpu
def test_vote_large_k_uses_global_buffers():
    """k = 700 needs a candidate buffer past shared memory; k = N takes every point."""
    coords, labels = G.vote_inputs()
    c, l_ = torch.from_numpy(coords).to(DEV), torch.from_numpy(labels).to(DEV)
    assert np.array_equal(S.knn_label_vote(c, l_, 700).cpu().numpy(), O.vote_exact(coords, labels, 700))
    full = S.knn_label_vote(c[:300], l_[:300], 300).cpu().numpy()
    assert (full == np.bincount(labels[:300]).argmax()).all()


@gpu
def test_vote_rejects_k_out_of_range_on_device():
    c = torch.zeros(4, 3, device=DEV)
    with pytest.raises(ValueError):
        S.local_post_process_segmentation(c, torch.zeros(4, dtype=torch.int64, device=DEV), k=5)
    with pytest.raises(ValueError):
        S.knn_label_vote(c, torch.zeros(4, dtype=torch.int64, device=DEV), k=0)
    one = S.knn_label_vote(torch.ones(1, 3, device=DEV), torch.full((1,), 3, dtype=torch.int64, device=DEV), 1)
    assert one.tolist() == [3]


# ------------------------------------------------------------------------------------------------ GPU: nearest vertex
@gpu
def test_nearest_vertex_against_oracle():
    rng = np.random.default_rng(8)
    verts = rng.uniform(-1, 1, (5000, 3))
    q = np.concatenate([rng.uniform(-1.2, 1.2, (3000, 3)), verts[:500]]).astype(np.float32)
    dup = np.concatenate([verts, verts[::-1]])                       # every distance tied: the lower index wins
    for v in (verts, dup):
        got = S.nearest_vertex(v, torch.from_numpy(q).to(DEV)).numpy()
        assert np.array_equal(got, O.nearest_exact(v, q))


# ------------------------------------------------------------------------------------------------ GPU: files end to end
@gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_cli_writes_the_reference_files(tmp_path, name):
    c = CASES[name]
    p = G.write_inputs(c, str(tmp_path / "in"))
    od = tmp_path / "out"
    extra = ["--use_spatial_smoothing", "true" if c["smooth"] else "false", "--query_embeddings", p["emb"]]
    S.main(_argv(p, od, *extra))
    assert files_of(od) == golden_files(f"cli_{name}")
    if name == "plain":
        for f in os.listdir(od):
            if f != "part_labels.npy":
                os.remove(od / f)
        S.main(_argv(p, od, "--overwrite", "False"))                 # no embeddings needed on the cached path
        assert files_of(od) == golden_files("cache")
        shutil.rmtree(od)
        S.main(_argv(p, od, "--overwrite", "true", "--query_embeddings", p["emb"]))
        assert files_of(od) == golden_files("cli_plain")


@gpu
def test_segmented_cloud_runs_the_simulation(tmp_path):
    from oracle import unet_ref as OU
    from pixie_b200 import scene_driver as SD
    from pixie_b200 import scene_files as SF
    c = CASES["smooth"]
    p = G.write_inputs(c, str(tmp_path / "in"))
    queries = list(c["props"])
    coords, labels, scores, metrics = S.clip_part_segmentation(p["grid"], queries, query_embs=c["table"])
    assert metrics["masked_voxels"] == len(coords) == int(c["mask"].astype(bool).sum())
    assert sum(metrics[f"part_{i}_{q}"] for i, q in enumerate(queries)) == len(coords)
    labels = S.local_post_process_segmentation(coords, labels)
    S.save_segmented_point_cloud(coords, labels, str(tmp_path / "out"), original_pc_path=p["occ"], part_queries=queries,
                                 material_props=c["props"], grid_feature_path=p["grid"])
    cloud = S.segmented_point_cloud(coords, labels, queries, c["props"], device=DEV)
    ref = SF.load_point_cloud(str(tmp_path / "out" / "segmented_semantics.ply"), device=DEV)
    for k in ref:
        assert torch.equal(cloud[k], ref[k]), k
    seg, reg = OU.build_pair(64, 16, seed=3)
    drv = SD.SceneBatchDriver(feature_channels=64, grid_size=16, device=DEV, seg_state_dict=seg.state_dict(),
                              cont_state_dict=reg.state_dict(), **OU.DEFAULT_CFG)
    rng = np.random.default_rng(1)
    pos = (coords.cpu().numpy() + rng.uniform(-0.01, 0.01, coords.shape)).astype(np.float32)
    sc = SD.Scene(name="vlm", grid=None, mask=None, min_bounds=c["bounds"][0], max_bounds=c["bounds"][1], particles=torch.from_numpy(pos),
                  material_params={"n_grid": 32, "grid_lim": 2.0, "material": "jelly", "g": [0.0, 0.0, -9.8], "density": 1000.0,
                                   "E": 1e5, "nu": 0.3},
                  bc_params=[{"type": "bounding_box"}], time_params={"substep_dt": 1e-4, "frame_dt": 2e-3, "frame_num": 2})
    rec = drv.run_physics_simulation(sc, cloud)
    assert len(rec["frames_pos"]) == 2 and all(torch.isfinite(f).all() for f in rec["frames_pos"])
