"""Image metrics (pixie_b200.gs_metrics): the fp64 oracle (oracle/image_metrics_ref.py) against the reference's float32
ssim / psnr (golden vectors) on the CPU; the device kernel against the oracle and the command line's files on the GPU."""
from __future__ import annotations

import json
import math
import os
import sys

import numpy as np
import pytest
import torch
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import image_metrics_ref as M  # noqa: E402
from pixie_b200 import gs_metrics as G  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "gs_views_golden.npz")

U32 = 2.0 ** -24


def ulp32(v: float) -> float:
    return float(np.spacing(np.float32(abs(v)))) if math.isfinite(v) else 0.0


def to_float(u8: np.ndarray) -> np.ndarray:
    """to_tensor: (H, W, 3) uint8 -> (3, H, W) float32 k / 255."""
    return np.ascontiguousarray((torch.from_numpy(u8).permute(2, 0, 1).float() / 255).numpy())


def pairs(rng, H, W):
    a = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    noisy = np.clip(a.astype(np.int64) + rng.integers(-20, 21, a.shape), 0, 255).astype(np.uint8)
    flat = np.full((H, W, 3), 200, np.uint8)
    flat2 = flat.copy()
    flat2[rng.random((H, W)) < 0.02] = 201                  # near-flat: sigma^2 ~ 1e-7 against C2 = 9e-4
    flat2[H // 2, W // 2] = 201
    return {"random": (a, rng.integers(0, 256, (H, W, 3), dtype=np.uint8)), "noisy": (a, noisy), "near_flat": (flat, flat2)}


# ------------------------------------------------------------------------------------------------ CPU
def test_window_is_the_reference_construction():
    g = G.ssim_window()
    gauss = torch.Tensor([math.exp(-(x - 5) ** 2 / float(2 * 1.5 ** 2)) for x in range(11)])
    assert g.dtype == torch.float32 and torch.equal(g, gauss / gauss.sum())


def test_oracle_agrees_with_reference_float32():
    """Against loss_utils.ssim and image_utils.psnr themselves (tests/golden/gs_views_golden.npz, run on the CPU in float32).
    The oracle evaluates the same formulas in fp64 over the same float32 inputs, with the 2D window g_i g_j exact where
    the reference rounds it to float32. Every quantity of the map is a sum of at most 121 products of values in [0, 1]
    with weights summing to 1, so each float32 convolution is within 2 * 121 u (u = 2^-24) of its exact value, the window
    rounding adding u per weight. A map entry's error is then at most 4 * 121 u times (|E[x^2]| + |E[y^2]| + |E[xy]| +
    mu1^2 + mu2^2 + 1) over its smallest denominator factor (sigma1^2 + sigma2^2 + C2), plus the same bound times the
    entry for the numerator; the mean carries that average plus n u. PSNR: the float32 mean of n squares is within n u
    relative, so 20 log10 moves by at most 10 / ln(10) * n u; the stored value adds half a float32 ulp."""
    gold = np.load(GOLDEN)
    g = G.ssim_window().numpy()
    k = 0
    while f"metric_{k}_0_a" in gold.files:
        for j in range(3):
            a, b = to_float(gold[f"metric_{k}_{j}_a"]), to_float(gold[f"metric_{k}_{j}_b"])
            ref_s, ref_p = float(gold[f"metric_{k}_{j}_ssim"]), float(gold[f"metric_{k}_{j}_psnr"])
            x, y = a.astype(np.float64), b.astype(np.float64)
            w2 = M.window(g)
            mu1, mu2 = M._filter(x, w2), M._filter(y, w2)
            exx, eyy, exy = M._filter(x * x, w2), M._filter(y * y, w2), M._filter(x * y, w2)
            den = (exx - mu1 ** 2) + (eyy - mu2 ** 2) + M.C2
            mag = np.abs(exx) + np.abs(eyy) + np.abs(exy) + mu1 ** 2 + mu2 ** 2 + 1
            bound = float(np.mean(2 * 4 * 121 * U32 * mag / den)) + a.size * U32
            o = M.ssim(a, b, g)
            assert abs(ref_s - o) <= bound + ulp32(o), (k, j, ref_s, o, bound)
            p = M.psnr(a, b)
            assert abs(ref_p - p) <= 10 / math.log(10) * a.size * U32 * abs(p) + ulp32(p), (k, j, ref_p, p)
        k += 1
    assert k == 3
    assert M.psnr(a, a) == math.inf and M.ssim(a, a, g) == 1.0


def test_cli_reports_failed_scenes(tmp_path, capsys):
    missing = str(tmp_path / "no_such_model")
    assert G.main(["-m", missing]) == 1
    err = capsys.readouterr().err
    assert "Unable to compute metrics for model " + missing in err and "FileNotFoundError" in err


def test_help_mentions_lpips(capsys):
    with pytest.raises(SystemExit):
        G.main(["--help"])
    assert "LPIPS is not computed" in " ".join(capsys.readouterr().out.split())
    assert "LPIPS is not computed" in G.__doc__


# ------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("hw", [(5, 7), (11, 11), (37, 53), (800, 800), (577, 801)])
def test_kernel_matches_oracle(built_lib, cuda_dev, hw):
    rng = np.random.default_rng(sum(hw))
    g = G.ssim_window().numpy()
    cases = pairs(rng, *hw)
    cases["identical"] = (cases["random"][0], cases["random"][0].copy())
    for name, (a8, b8) in cases.items():
        r = G.image_metrics(torch.from_numpy(a8).to(cuda_dev), torch.from_numpy(b8).to(cuda_dev)).cpu().numpy()
        a, b = to_float(a8), to_float(b8)
        o_s, o_p = M.ssim(a, b, g), M.psnr(a, b)
        if name == "identical":
            assert r[0] == math.inf and r[1] == 1.0
            continue
        assert abs(r[1] - o_s) <= 2 * ulp32(o_s), (hw, name, r[1], o_s)
        assert r[0] == o_p if math.isinf(o_p) else abs(r[0] - o_p) <= 2 * ulp32(o_p), (hw, name, r[0], o_p)
        again = G.image_metrics(torch.from_numpy(a8).to(cuda_dev), torch.from_numpy(b8).to(cuda_dev)).cpu().numpy()
        assert np.array_equal(r, again)


@pytest.mark.gpu
def test_cli_results_files(built_lib, cuda_dev, tmp_path):
    rng = np.random.default_rng(4)
    model = tmp_path / "model"
    g = G.ssim_window().numpy()
    want = {}
    for method, n in (("ours_30000", 3), ("ours_7000", 0)):
        for kind in ("renders", "gt"):
            (model / "test" / method / kind).mkdir(parents=True)
        for i in range(n):
            a8 = rng.integers(0, 256, (40, 56, 3), dtype=np.uint8)
            b8 = a8 if i == 1 else np.clip(a8.astype(int) + rng.integers(-9, 10, a8.shape), 0, 255).astype(np.uint8)
            Image.fromarray(a8).save(model / "test" / method / "renders" / f"{i:05d}.png")
            Image.fromarray(b8).save(model / "test" / method / "gt" / f"{i:05d}.png")
            want[f"{i:05d}.png"] = (M.ssim(to_float(a8), to_float(b8), g), M.psnr(to_float(a8), to_float(b8)))
    bad = tmp_path / "bad"
    (bad / "test" / "m" / "renders").mkdir(parents=True)
    Image.fromarray(np.zeros((4, 4, 3), np.uint8)).save(bad / "test" / "m" / "renders" / "00000.png")
    assert G.main(["-m", str(model), str(bad)]) == 1                  # the bad scene has no gt/ image
    res = json.load(open(model / "results.json"))
    per = json.load(open(model / "per_view.json"))
    assert sorted(res) == ["ours_30000", "ours_7000"] and sorted(res["ours_30000"]) == ["PSNR", "SSIM"]
    assert math.isnan(res["ours_7000"]["SSIM"]) and math.isnan(res["ours_7000"]["PSNR"])
    assert per["ours_7000"] == {"SSIM": {}, "PSNR": {}}
    for name, (s, p) in want.items():
        assert abs(per["ours_30000"]["SSIM"][name] - s) <= 2 * ulp32(s)
        assert per["ours_30000"]["PSNR"][name] == p if math.isinf(p) else abs(per["ours_30000"]["PSNR"][name] - p) <= 2 * ulp32(p)
    ms = float(np.mean([s for s, _ in want.values()]))
    assert abs(res["ours_30000"]["SSIM"] - ms) <= 2 * ulp32(ms)
    assert res["ours_30000"]["PSNR"] == math.inf
    text = (model / "results.json").read_text()
    assert text.startswith("{\n \"ours_30000\": {\n  \"SSIM\": ") and "Infinity" in text and "NaN" in text
    assert not (bad / "results.json").exists()
