"""GPU parity tests of the U-Net path (needs an H100: pytest -m gpu). Every call goes through
the C ABI (pixie_b200/_lib.py -> libpixie_b200.so); the oracle is only the checker.

Tolerances (max-abs on outputs of magnitude ~3):
  fp16x3  : < 1e-3   — the north-star material-field tolerance (measured ~5e-5)
  fp16e5  : < 1e-3   — one fp16 pass + one E5M2 pass carrying a_lo*w + a*w_lo (2 pass-equivalents; predicted 3e-4 by a CPU
                       emulation of the rounding points, see DESIGN.md "Numerics") — the default mode of bench.py
  fp16    : < 2e-2   — one tensor-core pass with fp16 operands has a 2^-11 relative rounding per operand,
                       the same mantissa as the TF32 arithmetic the reference's own GPU run uses
                       (torch default cudnn.allow_tf32); measured ~5e-3 (see DESIGN.md, "Numerics").
"""
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import unet_ref as O

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL = {"fp16x3": 1e-3, "fp16e5": 1e-3, "fp16": 2e-2}


def _mine(cls_name, C, G, out, precision, sd, max_batch=2, cfg=None):
    from pixie_b200 import unet as U
    cfg = dict(O.DEFAULT_CFG if cfg is None else cfg)
    kw = dict(num_classes=out) if cls_name == "SegmentationUNet" else dict(out_channels=out)
    net = getattr(U, cls_name)(feature_channels=C, grid_size=G, max_batch=max_batch, precision=precision, **cfg, **kw).to("cuda:0")
    net.load_state_dict(sd)
    return net.eval()


def test_conv_bringup_binary(built_lib, cuda_dev):
    """build/conv_test: every kernel instance, ragged and 64^3 geometry, short batches, the three statistics modes and the
    three numerics against an fp64 host reference of the products the kernel computes, under a per-element fp32
    accumulation bound, through the same host planner the library uses (see pixie_b200/csrc/conv_test.cu)."""
    exe = os.path.join(ROOT, "build", "conv_test")
    assert os.path.exists(exe)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=1200)
    summary = r.stdout[r.stdout.find("INSTANCES"):]
    print(summary)
    fails = [line for line in r.stdout.splitlines() if " FAIL" in line or line.startswith("FAIL")]
    assert r.returncode == 0 and "fail=0" in r.stdout, "\n".join(fails[:40]) + "\n" + summary + r.stderr[-2000:]


def test_unet_kernels_binary(built_lib, cuda_dev):
    """build/unet_kernels_test: moments, norm_act, upsample2 and attention against fp64 host references, including
    offset data, every normalisation x activation x lo layout, channel slices and logits up to +-60
    (see pixie_b200/csrc/unet_kernels_test.cu)."""
    exe = os.path.join(ROOT, "build", "unet_kernels_test")
    assert os.path.exists(exe)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    print(r.stdout[-6000:])
    fails = [line for line in r.stdout.splitlines() if " FAIL" in line]
    assert r.returncode == 0 and "fail=0" in r.stdout, "\n".join(fails[:40]) + r.stdout[-500:] + r.stderr[-2000:]


@pytest.mark.parametrize("precision", ["fp16e5", "fp16x3", "fp16"])
def test_short_batch_writes_only_the_callers_items(built_lib, cuda_dev, precision):
    """A network built for max_batch = 2 and run on one item writes into that item only. At G = 16 the head convolution
    uses split-K and clears its output before accumulating; the clear must cover the launched items, not max_batch of
    them (big[1] lies right after the caller's one-item output). N = 3 runs as chunks of 2 and 1."""
    C, G = 64, 16
    seg, reg = O.build_pair(C, G, seed=12)
    x = O.synthetic_features(3, C, G, seed=13)
    with torch.no_grad():
        refs = {"SegmentationUNet": (8, seg, seg(x)), "RegressionUNet": (3, reg, reg(x))}
    x_cl = x.permute(0, 2, 3, 4, 1).contiguous().to(torch.float16).cuda()
    for cls, (out, oracle, y_ref) in refs.items():
        net = _mine(cls, C, G, out, precision, oracle.state_dict(), max_batch=2)
        big = torch.full((2, out, G, G, G), float("nan"), device="cuda:0")
        net.forward_channels_last_f16(x_cl[:1], out=big[:1])
        net.check()
        assert torch.isnan(big[1]).all(), f"{cls} {precision}: wrote past the end of a one-item output"
        assert (big[0].cpu() - y_ref[0]).abs().max() < TOL[precision]
        y3 = net(x.cuda()).cpu()
        net.check()
        for i in range(3):
            assert (y3[i] - y_ref[i]).abs().max() < TOL[precision], (cls, i)


@pytest.mark.parametrize("precision", ["fp16e5", "fp16x3", "fp16"])
def test_golden_vectors(built_lib, cuda_dev, precision):
    """Outputs of the REFERENCE modules (tests/golden/make_unet_golden.py) on seeded inputs."""
    g = np.load(os.path.join(ROOT, "tests", "golden", "unet_small.npz"))
    x = torch.from_numpy(g["x"])
    for name, out, cls in (("reg", 3, "RegressionUNet"), ("seg", 8, "SegmentationUNet")):
        ref = (O.RegressionUNet if out == 3 else O.SegmentationUNet)(64, 32, 64, 3, (1, 1, 2, 4), (), 8, out)
        sd = O.seeded_state_dict(ref, int(g[f"{name}_seed"]))
        net = _mine(cls, 64, 8, out, precision, sd)
        y = net(x.cuda()).cpu().numpy()
        net.check()
        assert np.abs(y - g[f"{name}_y"]).max() < TOL[precision]


@pytest.mark.parametrize("precision", ["fp16e5", "fp16x3", "fp16"])
@pytest.mark.parametrize("C,G", [(128, 16), (512, 32)])
def test_parity_vs_oracle_both_networks(built_lib, cuda_dev, precision, C, G):
    """BASELINE config 1 (32^3 x 512) and a smaller grid; segmentation argmax must agree wherever the
    oracle's top-2 logit gap exceeds 10x the tolerance."""
    seg, reg = O.build_pair(C, G, seed=0)
    x = O.synthetic_features(1, C, G, seed=1)
    with torch.no_grad():
        ys, yr = seg(x), reg(x)
    ns = _mine("SegmentationUNet", C, G, 8, precision, seg.state_dict(), max_batch=1)
    nr = _mine("RegressionUNet", C, G, 3, precision, reg.state_dict(), max_batch=1)
    zs, zr = ns(x.cuda()).cpu(), nr(x.cuda()).cpu()
    ns.check(); nr.check()
    assert (zr - yr).abs().max() < TOL[precision]
    assert (zs - ys).abs().max() < TOL[precision]
    top2 = ys.topk(2, dim=1).values
    confident = (top2[:, 0] - top2[:, 1]) > 10 * TOL[precision]
    assert (zs.argmax(1) == ys.argmax(1))[confident].all()
    assert confident.float().mean() > 0.5


def test_input_layout_paths_agree(built_lib, cuda_dev):
    """fp32 NCDHW (reference dataset layout), fp16 NDHWC device (on-disk layout) and the host-buffer
    end-to-end call give the same result; batch of 2 equals two single forwards."""
    C, G = 64, 16
    _, reg = O.build_pair(C, G, seed=2)
    # fp16x3: the three paths agree to fp32 round-off. (In single-pass fp16 mode 1-ulp differences in the
    # fp64-atomic statistics flip individual fp16 roundings, so two runs of the SAME path differ at the
    # mode's own noise level, ~2.5e-3; that mode is covered by its stated tolerance in the parity tests.)
    net = _mine("RegressionUNet", C, G, 3, "fp16x3", reg.state_dict(), max_batch=2)
    x = O.synthetic_features(2, C, G, seed=4)                    # exactly fp16-representable values
    y_ncdhw = net(x.cuda()).cpu()
    x_cl = x.permute(0, 2, 3, 4, 1).contiguous().to(torch.float16)
    y_cl = net.forward_channels_last_f16(x_cl.cuda()).cpu()
    y_host = net.forward_host(x_cl.pin_memory()).clone()
    net.check()
    assert (y_ncdhw - y_cl).abs().max() < 1e-4
    assert (y_host - y_cl).abs().max() < 1e-4
    y0 = net(x[:1].cuda()).cpu()
    y1 = net(x[1:].cuda()).cpu()
    assert (torch.cat([y0, y1]) - y_ncdhw).abs().max() < 1e-4
    with pytest.raises(ValueError):
        net(torch.zeros(1, C + 1, G, G, G))
    with pytest.raises(ValueError):
        net.forward_host(torch.zeros(3, G, G, G, C, dtype=torch.float16))


def test_pack_predictions_matches_reference_packing(built_lib, cuda_dev):
    """`pixie_pack_predictions` against the reference's own statements: `th.argmax(seg_logits, dim=1)`
    (inference_combined.py:125) and the one-hot packing of save_predictions (:173-199: continuous channels first, then
    np.eye(n_classes)[label] moved to channel-first). Exact ties between class logits must resolve to the FIRST maximum,
    like torch.argmax / np.argmax."""
    from pixie_b200.inference import MaterialFieldPredictor
    G, K = 16, 8
    pred = MaterialFieldPredictor(feature_channels=64, grid_size=G, device="cuda:0", max_batch=2, precision="fp16x3", **O.DEFAULT_CFG)
    g = torch.Generator().manual_seed(3)
    seg = torch.randn(2, K, G, G, G, generator=g)
    cont = torch.randn(2, 3, G, G, G, generator=g)
    # ties: two, three and all classes equal to the maximum, at known voxels
    seg[0, :, 0, 0, 0] = 1.5
    seg[0, :, 0, 0, 1] = torch.tensor([0.1, 2.0, -1.0, 2.0, 0.3, 2.0, 0.0, 1.0])
    seg[1, :, 3, 2, 1] = torch.tensor([-3.0, -3.0, 7.0, 0.0, 0.0, 0.0, 0.0, 7.0])
    seg[1, :, 5, 5, 5] = float("-inf"); seg[1, 6, 5, 5, 5] = -1e30
    out = pred.pack(seg.cuda(), cont.cuda()).cpu()
    labels = torch.argmax(seg, dim=1)                                                      # inference_combined.py:125
    onehot = torch.from_numpy(np.eye(K, dtype=np.float32)[labels.numpy()]).permute(0, 4, 1, 2, 3)   # :186-191
    want = torch.cat([cont, onehot], dim=1)
    assert torch.equal(out, want)
    assert labels[0, 0, 0, 0] == 0 and labels[0, 0, 0, 1] == 1 and labels[1, 3, 2, 1] == 2 and labels[1, 5, 5, 5] == 6


def test_pipelined_host_stream_equals_single_calls(built_lib, cuda_dev):
    """predict_packed_host_stream (double-buffered H2D overlapping the networks) = predict_packed_host scene by scene,
    including when the two input slots and the graph cache are cycled more than once."""
    from pixie_b200.inference import MaterialFieldPredictor
    C, G = 64, 16
    seg, reg = O.build_pair(C, G, seed=6)
    pred = MaterialFieldPredictor(feature_channels=C, grid_size=G, device="cuda:0", max_batch=1, precision="fp16x3", **O.DEFAULT_CFG)
    pred.load_state_dicts(seg.state_dict(), reg.state_dict())
    scenes = [O.synthetic_features(1, C, G, seed=10 + i).permute(0, 2, 3, 4, 1).contiguous().to(torch.float16).pin_memory() for i in range(5)]
    single = [pred.predict_packed_host(s).clone() for s in scenes]
    # the first scene also against the oracle networks + the reference's packing (not only against ourselves)
    with torch.no_grad():
        x0 = scenes[0].float().permute(0, 4, 1, 2, 3).contiguous()
        ys, yr = seg(x0), reg(x0)
    assert (single[0][:, :3] - yr).abs().max() < TOL["fp16x3"]
    top2 = ys.topk(2, dim=1).values
    confident = (top2[:, 0] - top2[:, 1]) > 10 * TOL["fp16x3"]
    assert (single[0][:, 3:].argmax(1) == ys.argmax(1))[confident].all() and (single[0][:, 3:].sum(1) == 1).all()
    piped = pred.predict_packed_host_stream(scenes)
    piped2 = pred.predict_packed_host_stream(iter(scenes[::-1]))                          # a generator: consumed lazily
    for i in range(5):
        assert (piped[i][:, :3] - single[i][:, :3]).abs().max() < 1e-4
        assert (piped[i][:, 3:] == single[i][:, 3:]).float().mean() > 0.9999          # one-hot argmax
        assert (piped2[4 - i][:, :3] - single[i][:, :3]).abs().max() < 1e-4


def test_scene_stream_from_npy_files_through_host_pipeline(built_lib, cuda_dev, tmp_path):
    """voxel_io.scene_stream -> predict_packed_host_stream from real clip_features_features.npy files, with MORE scenes than
    pinned buffers: every scene's output must equal its own single-scene result (a recycled pinned buffer must not be
    rewritten before the device has read it)."""
    from pixie_b200 import voxel_io as V
    from pixie_b200.inference import MaterialFieldPredictor
    C, G, n_scenes = 64, 16, 7
    seg, reg = O.build_pair(C, G, seed=8)
    pred = MaterialFieldPredictor(feature_channels=C, grid_size=G, device="cuda:0", max_batch=1, precision="fp16x3", **O.DEFAULT_CFG)
    pred.load_state_dicts(seg.state_dict(), reg.state_dict())
    dirs, grids = [], []
    for i in range(n_scenes):
        a = O.synthetic_features(1, C, G, seed=40 + i)[0].permute(1, 2, 3, 0).contiguous().to(torch.float16).numpy()   # (D, D, D, C) fp16
        d = os.path.join(str(tmp_path), f"obj{i}")
        os.makedirs(d)
        np.save(os.path.join(d, V.FEATURE_FILE), a)
        dirs.append(d); grids.append(a)
    single = [pred.predict_packed_host(torch.from_numpy(a)[None].pin_memory()).clone() for a in grids]
    outs = pred.predict_packed_host_stream(V.scene_stream(dirs, n_buffers=2))
    assert len(outs) == n_scenes
    for i in range(n_scenes):
        assert (outs[i][:, :3] - single[i][:, :3]).abs().max() < 1e-4, i
        assert (outs[i][:, 3:] == single[i][:, 3:]).float().mean() > 0.9999, i
    # distinct scenes really give distinct fields (the test would pass trivially otherwise)
    assert (single[0][:, :3] - single[1][:, :3]).abs().max() > 1e-2


@pytest.mark.parametrize("C", [3, 32])
def test_projector_variants(built_lib, cuda_dev, C):
    """rgb / occupancy feature types: single-layer projector; feature_channels == cond_dim: none."""
    cfg = dict(cond_dim=32, model_channels=64, num_res_blocks=1, channel_mult=(1, 2), attention_resolutions=())
    ref = O.SegmentationUNet(feature_channels=C, grid_size=8, num_classes=8, **cfg).eval()
    ref.load_state_dict(O.seeded_state_dict(ref, 7))
    x = O.synthetic_features(1, C, 8, seed=5, scale=1.0)
    with torch.no_grad():
        y = ref(x)
    net = _mine("SegmentationUNet", C, 8, 8, "fp16x3", ref.state_dict(), cfg=cfg)
    z = net(x.cuda()).cpu()
    net.check()
    assert (z - y).abs().max() < 1e-3


def test_missing_weights_fail_loudly(built_lib, cuda_dev):
    from pixie_b200 import _lib
    from pixie_b200.unet import RegressionUNet
    net = RegressionUNet(64, 32, 64, 1, (1, 2), (), 8, 3).to("cuda:0")
    with pytest.raises(_lib.PixieError):
        net(torch.zeros(1, 64, 8, 8, 8))


def test_full_size_64_cubed_512(built_lib, cuda_dev):
    """BASELINE config 2 size. The oracle forward takes several seconds on the host; checked for both networks (the
    segmentation one in the default precision), plus size-independent properties: determinism to round-off (split-K
    uses float atomics at the coarse levels) and batch/single consistency through the staging path."""
    C, G = 512, 64
    seg, reg = O.build_pair(C, G, seed=0)
    x16 = (torch.randn(1, G, G, G, C, generator=torch.Generator().manual_seed(1)) * 0.05).to(torch.float16)
    with torch.no_grad():
        y_ref = reg(x16.float().permute(0, 4, 1, 2, 3).contiguous())
    for precision in ("fp16e5", "fp16x3", "fp16"):
        net = _mine("RegressionUNet", C, G, 3, precision, reg.state_dict(), max_batch=1)
        y = net.forward_channels_last_f16(x16.cuda())
        y2 = net.forward_channels_last_f16(x16.cuda())
        net.check()
        assert (y - y2).abs().max() < (1e-4 if precision == "fp16x3" else TOL[precision])
        print(f"64^3x512 {precision}: max-abs vs fp32 oracle {float((y.cpu() - y_ref).abs().max()):.3e}")
        assert (y.cpu() - y_ref).abs().max() < TOL[precision]
        del net
        torch.cuda.empty_cache()
    with torch.no_grad():
        ys = seg(x16.float().permute(0, 4, 1, 2, 3).contiguous())
    net = _mine("SegmentationUNet", C, G, 8, "fp16e5", seg.state_dict(), max_batch=1)
    zs = net.forward_channels_last_f16(x16.cuda()).cpu()
    net.check()
    assert (zs - ys).abs().max() < TOL["fp16e5"]
    top2 = ys.topk(2, dim=1).values
    confident = (top2[:, 0] - top2[:, 1]) > 10 * TOL["fp16e5"]
    assert (zs.argmax(1) == ys.argmax(1))[confident].all()
