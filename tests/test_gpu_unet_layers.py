"""Per-layer parity of the U-Net executor (needs an H100: pytest -m gpu).

Every activation the executor registers for `debug_fetch` (the outputs of projector.net.{0,3,6}, unet.input_blocks.k(.0),
unet.middle_block.{0,1,2} and unet.output_blocks.k.{0,1}) is compared with the same module's output in an fp64 copy of the
oracle network, as max|ours - ref| / max|ref| per layer. A registered name without a matching oracle module fails the
test, so the two lists stay in sync. Besides a bound per precision, every layer must keep the precisions in order,
fp16x3 < fp16e5 < fp16 / 4, so that a correction one layer silently drops is caught even where the error stays small.
The first convolution reads the fp16 input grid, which has no rounding residual: there fp16x3 and fp16e5 run the same
products, their errors differ only by the order of split-K atomics, and only the fp16 / 4 part of the order is required.

BOUND is at most 4x the largest per-layer error measured on an H100 SXM (80 GB HBM3, 400 W power limit) over all
configurations here: fp16x3 1.25e-5, fp16e5 1.45e-4, fp16 2.28e-3 (the worst layers are upsample outputs and the deepest
blocks; errors grow from ~2e-7 / 2e-7 / 9e-5 at the first convolution).
"""
import copy
import math
import types

import pytest
import torch
import torch.nn as nn

from oracle import unet_ref as O

pytestmark = pytest.mark.gpu
PRECISIONS = ("fp16x3", "fp16e5", "fp16")
BOUND = {"fp16x3": 4e-5, "fp16e5": 5e-4, "fp16": 8e-3}

SMALL_CFG = dict(cond_dim=32, model_channels=64, num_res_blocks=1, channel_mult=(1, 2), attention_resolutions=())
# (feature channels, grid side, network config, networks): G = 24 makes every tile ragged (sides 24/12/6/3) and the
# bottleneck attention run over T = 27 tokens; the last two are the single-layer and absent projectors
CONFIGS = {
    "C64_G16": (64, 16, O.DEFAULT_CFG, ("seg", "reg")),
    "C64_G24": (64, 24, O.DEFAULT_CFG, ("seg", "reg")),
    "C3_G8_light_projector": (3, 8, SMALL_CFG, ("seg",)),
    "C32_G8_no_projector": (32, 8, SMALL_CFG, ("seg",)),
}


def _unet_forward_f64(self, x):
    """MyUNetModel.forward without its fp32 casts (inputs here are even-sized, so no crop)."""
    hs = []
    h = x
    for module in self.input_blocks:
        h = module(h)
        hs.append(h)
    h = self.middle_block(h)
    for module in self.output_blocks:
        h = module(torch.cat([h, hs.pop()], dim=1))
    return self.out(h)


def _qkv_f64(self, qkv):
    ch = qkv.shape[1] // 3
    q, k, v = torch.split(qkv, ch, dim=1)
    scale = 1 / math.sqrt(math.sqrt(ch))
    weight = torch.softmax(torch.einsum("bct,bcs->bts", q * scale, k * scale), dim=-1)
    return torch.einsum("bts,bcs->bct", weight, v)


def _reference_activations(model, x, names):
    """fp64 forward of `model` on `x`, returning the output of every module in `names`."""
    m = copy.deepcopy(model).double().eval()
    for mod in m.modules():
        if isinstance(mod, O.MyUNetModel):
            mod.forward = types.MethodType(_unet_forward_f64, mod)
        elif isinstance(mod, O.QKVAttention):
            mod.forward = types.MethodType(_qkv_f64, mod)
        elif isinstance(mod, O.GroupNorm32):
            mod.forward = types.MethodType(nn.GroupNorm.forward, mod)
    mods = dict(m.named_modules())
    unknown = sorted(n for n in names if n not in mods)
    assert not unknown, f"activations registered by the executor without an oracle module: {unknown}"
    acts = {}
    hooks = [mods[n].register_forward_hook(lambda _m, _i, out, n=n: acts.__setitem__(n, out.detach().clone())) for n in names]
    with torch.no_grad():
        m(x.double())
    for h in hooks:
        h.remove()
    order = [n for n, _ in m.named_modules() if n in acts]
    return {n: acts[n] for n in order}


@pytest.mark.parametrize("config", list(CONFIGS))
def test_layers_match_fp64_oracle(built_lib, cuda_dev, config):
    from pixie_b200 import unet as U
    C, G, cfg, which = CONFIGS[config]
    seg, reg = O.build_pair(C, G, seed=21, cfg=cfg)
    x = O.synthetic_features(2, C, G, seed=22, scale=0.05 if C >= 64 else 1.0)   # batch of two different items
    failures = []
    for net_name in which:
        oracle = seg if net_name == "seg" else reg
        cls = "SegmentationUNet" if net_name == "seg" else "RegressionUNet"
        out_ch = 8 if net_name == "seg" else 3
        kw = dict(num_classes=out_ch) if net_name == "seg" else dict(out_channels=out_ch)
        errs = {}
        ref = None
        for precision in PRECISIONS:
            net = getattr(U, cls)(feature_channels=C, grid_size=G, max_batch=2, precision=precision, **cfg, **kw).to("cuda:0")
            net.load_state_dict(oracle.state_dict())
            net(x.cuda())
            net.check()
            names = net.debug_names()
            if ref is None:
                ref = _reference_activations(oracle, x, names)
            assert set(names) == set(ref)
            for name, r in ref.items():
                ch, sp = names[name]
                ours = net.debug_fetch(name, ch, sp, batch=2).double()
                assert ours.shape == r.shape, (name, ours.shape, r.shape)
                errs.setdefault(name, {})[precision] = float((ours - r).abs().max() / r.abs().max())
            del net
        first = next(iter(ref))
        print(f"\n{config} {net_name}: max|ours - fp64| / max|fp64| per layer")
        print(f"  {'layer':<28}" + "".join(f"{p:>11}" for p in PRECISIONS))
        for name, e in errs.items():
            print(f"  {name:<28}" + "".join(f"{e[p]:11.2e}" for p in PRECISIONS))
            for p in PRECISIONS:
                if not e[p] < BOUND[p]:
                    failures.append(f"{net_name} {name} {p}: {e[p]:.3e} >= bound {BOUND[p]:.1e}")
            if name != first and not e["fp16x3"] < e["fp16e5"]:
                failures.append(f"{net_name} {name}: fp16x3 {e['fp16x3']:.3e} not below fp16e5 {e['fp16e5']:.3e}")
            if not e["fp16e5"] < e["fp16"] / 4:
                failures.append(f"{net_name} {name}: fp16e5 {e['fp16e5']:.3e} not below fp16 / 4 = {e['fp16'] / 4:.3e}")
        worst = {p: max(e[p] for e in errs.values()) for p in PRECISIONS}
        print("  worst: " + ", ".join(f"{p} {worst[p]:.2e} (bound {BOUND[p]:.1e})" for p in PRECISIONS))
    assert not failures, "\n".join(failures)
