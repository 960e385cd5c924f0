"""ORACLE (test infrastructure, not product code): CPU restatement of the reference 3-D U-Net path.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import
this module.  It is the checker, never the thing shipped: pixie_b200/ must not import it.

Restates, in plain PyTorch (fp32, CPU), exactly the modules the reference's inference path runs:

  * FeatureProjector            third_party/Wavelet-Generation/models/module/diffusion_network.py:534-589
  * MyResBlock                  diffusion_network.py:639-710
  * Downsample / Upsample       diffusion_network.py:51-97
  * AttentionBlock/QKVAttention diffusion_network.py:192-242  (GroupNorm32: nn.py:17-19, 98-104)
  * MyUNetModel                 diffusion_network.py:712-935
  * SegmentationUNet            third_party/Wavelet-Generation/trainer/training_discrete.py:50-88
  * RegressionUNet              third_party/Wavelet-Generation/trainer/training_continuous_mse.py:48-89

Module attribute names are the reference's, so `state_dict()` keys are identical
(projector.net.N.*, unet.input_blocks.N.0.{in_layers,out_layers,skip_connection}.*, ...): a
reference checkpoint loads into these classes and vice versa.

Pinning: the reference has no tests or golden vectors for this path (SURVEY.md §4).  This
restatement is pinned against the reference *itself*: tests/golden/make_unet_golden.py runs the
reference modules on seeded parameters and inputs, and tests/test_oracle_unet.py requires this
restatement to reproduce their parameter names and outputs (unet_small.npz, unet_ref_modules.npz).
"""
from __future__ import annotations

import math
from typing import Optional, Sequence, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F


def zero_module(module: nn.Module) -> nn.Module:
    """nn.py:67-73 — the reference zero-initialises these convolutions."""
    for p in module.parameters():
        p.detach().zero_()
    return module


class GroupNorm32(nn.GroupNorm):
    """nn.py:17-19."""

    def forward(self, x):
        return super().forward(x.float()).type(x.dtype)


class Upsample(nn.Module):
    """diffusion_network.py:51-72 (dims=3, use_conv=True)."""

    def __init__(self, channels: int):
        super().__init__()
        self.channels = channels
        self.conv = nn.Conv3d(channels, channels, 3, padding=1)

    def forward(self, x):
        x = F.interpolate(x, scale_factor=2, mode="nearest")
        return self.conv(x)


class Downsample(nn.Module):
    """diffusion_network.py:75-97 (dims=3, use_conv=True)."""

    def __init__(self, channels: int):
        super().__init__()
        self.channels = channels
        self.op = nn.Conv3d(channels, channels, 3, stride=2, padding=1)

    def forward(self, x):
        return self.op(x)


class QKVAttention(nn.Module):
    """diffusion_network.py:224-242."""

    def forward(self, qkv):
        ch = qkv.shape[1] // 3
        q, k, v = torch.split(qkv, ch, dim=1)
        scale = 1 / math.sqrt(math.sqrt(ch))
        weight = torch.einsum("bct,bcs->bts", q * scale, k * scale)
        weight = torch.softmax(weight.float(), dim=-1).type(weight.dtype)
        return torch.einsum("bts,bcs->bct", weight, v)


class AttentionBlock(nn.Module):
    """diffusion_network.py:192-221 (num_heads=1)."""

    def __init__(self, channels: int, num_heads: int = 1):
        super().__init__()
        self.channels = channels
        self.num_heads = num_heads
        self.norm = GroupNorm32(32, channels)
        self.qkv = nn.Conv1d(channels, channels * 3, 1)
        self.attention = QKVAttention()
        self.proj_out = zero_module(nn.Conv1d(channels, channels, 1))

    def forward(self, x):
        b, c, *spatial = x.shape
        x = x.reshape(b, c, -1)
        qkv = self.qkv(self.norm(x))
        qkv = qkv.reshape(b * self.num_heads, -1, qkv.shape[2])
        h = self.attention(qkv)
        h = h.reshape(b, -1, h.shape[-1])
        h = self.proj_out(h)
        return (x + h).reshape(b, c, *spatial)


class MyResBlock(nn.Module):
    """diffusion_network.py:639-710 (dims=3, use_conv=False)."""

    def __init__(self, channels: int, sp: int, dropout: float, out_channels: Optional[int], activation: nn.Module):
        super().__init__()
        self.channels = channels
        self.out_channels = out_channels or channels
        self.in_layers = nn.Sequential(
            nn.LayerNorm(normalized_shape=[sp, sp, sp]),
            activation,
            nn.Conv3d(channels, self.out_channels, 3, padding=1),
        )
        self.out_layers = nn.Sequential(
            nn.LayerNorm(normalized_shape=[sp, sp, sp]),
            activation,
            nn.Dropout(p=dropout),
            zero_module(nn.Conv3d(self.out_channels, self.out_channels, 3, padding=1)),
        )
        if self.out_channels == channels:
            self.skip_connection = nn.Identity()
        else:
            self.skip_connection = nn.Conv3d(channels, self.out_channels, 1)

    def forward(self, x):
        h = self.in_layers(x)
        h = self.out_layers(h)
        return self.skip_connection(x) + h


class MyUNetModel(nn.Module):
    """diffusion_network.py:712-935 (dims=3, conv_resample=True, num_heads=1, no class conditioning)."""

    def __init__(self, in_channels: int, model_channels: int, out_channels: int, num_res_blocks: int,
                 attention_resolutions: Sequence[int], spatial_size: int, dropout: float = 0,
                 channel_mult: Sequence[int] = (1, 2, 4, 8), activation: Optional[nn.Module] = None):
        super().__init__()
        self.activation = activation if activation is not None else nn.SiLU()
        self.in_channels, self.model_channels, self.out_channels = in_channels, model_channels, out_channels
        self.num_res_blocks = num_res_blocks
        self.attention_resolutions = tuple(attention_resolutions)
        self.channel_mult = tuple(channel_mult)

        self.input_blocks = nn.ModuleList([nn.Sequential(nn.Conv3d(in_channels, model_channels, 3, padding=1))])
        input_block_chans = [model_channels]
        input_block_sizes = [spatial_size]
        ch, ds, current_sp = model_channels, 1, spatial_size
        for level, mult in enumerate(channel_mult):
            for _ in range(num_res_blocks):
                layers = [MyResBlock(ch, current_sp, dropout, mult * model_channels, self.activation)]
                ch = mult * model_channels
                if ds in self.attention_resolutions:
                    layers.append(AttentionBlock(ch))
                self.input_blocks.append(nn.Sequential(*layers))
                input_block_chans.append(ch)
            if level != len(channel_mult) - 1:
                self.input_blocks.append(nn.Sequential(Downsample(ch)))
                input_block_chans.append(ch)
                input_block_sizes.append(current_sp)
                ds *= 2
                current_sp = (current_sp + 1) // 2

        self.middle_block = nn.Sequential(
            MyResBlock(ch, current_sp, dropout, None, self.activation),
            AttentionBlock(ch),
            MyResBlock(ch, current_sp, dropout, None, self.activation),
        )

        self.output_blocks = nn.ModuleList([])
        for level, mult in list(enumerate(channel_mult))[::-1]:
            for i in range(num_res_blocks + 1):
                layers = [MyResBlock(ch + input_block_chans.pop(), current_sp, dropout, model_channels * mult, self.activation)]
                ch = model_channels * mult
                if ds in self.attention_resolutions:
                    layers.append(AttentionBlock(ch))
                if level and i == num_res_blocks:
                    layers.append(Upsample(ch))
                    ds //= 2
                    current_sp = input_block_sizes.pop()
                self.output_blocks.append(nn.Sequential(*layers))

        self.out = nn.Sequential(
            nn.LayerNorm(normalized_shape=[current_sp, current_sp, current_sp]),
            self.activation,
            zero_module(nn.Conv3d(model_channels, out_channels, 3, padding=1)),
        )

    def forward(self, x):
        hs = []
        h = x.float()                                    # inner_dtype is hard-wired fp32 (:891-897)
        for module in self.input_blocks:
            h = module(h)
            hs.append(h)
        h = self.middle_block(h)
        for module in self.output_blocks:
            if hs[-1].size(-1) < h.size(-1):
                h = h[..., :-1]
            if hs[-1].size(-2) < h.size(-2):
                h = h[..., :-1, :]
            if hs[-1].size(-3) < h.size(-3):
                h = h[..., :-1, :, :]
            h = module(torch.cat([h, hs.pop()], dim=1))
        h = h.type(x.dtype)
        return self.out(h)


class FeatureProjector(nn.Module):
    """diffusion_network.py:534-589."""

    def __init__(self, in_channels: int, out_channels: int, hidden_channels: Optional[int] = None):
        super().__init__()
        if hidden_channels is None:
            layers = [
                nn.Conv3d(in_channels, out_channels, kernel_size=1),
                nn.GroupNorm(num_groups=max(out_channels // 2, 1), num_channels=out_channels),
                nn.SiLU(),
            ]
        else:
            layers = [
                nn.Conv3d(in_channels, hidden_channels, kernel_size=1),
                nn.GroupNorm(num_groups=32, num_channels=hidden_channels),
                nn.SiLU(),
                nn.Conv3d(hidden_channels, hidden_channels, kernel_size=3, padding=1),
                nn.GroupNorm(num_groups=32, num_channels=hidden_channels),
                nn.SiLU(),
                nn.Conv3d(hidden_channels, out_channels, kernel_size=1),
                nn.GroupNorm(num_groups=32, num_channels=out_channels),
            ]
        self.net = nn.Sequential(*layers)

    def forward(self, x):
        return self.net(x)


class _ProjectedUNet(nn.Module):
    def __init__(self, feature_channels, cond_dim, model_channels, num_res_blocks, channel_mult,
                 attention_resolutions, grid_size, out_channels):
        super().__init__()
        hidden_ch = 128 if feature_channels > cond_dim else None
        self.projector = (None if feature_channels == cond_dim
                          else FeatureProjector(feature_channels, out_channels=cond_dim, hidden_channels=hidden_ch))
        self.unet = MyUNetModel(in_channels=cond_dim, model_channels=model_channels, out_channels=out_channels,
                                num_res_blocks=num_res_blocks, channel_mult=channel_mult,
                                attention_resolutions=attention_resolutions, spatial_size=grid_size,
                                activation=nn.LeakyReLU(0.02))

    def forward(self, feat_grid):
        x = feat_grid
        if self.projector is not None:
            x = self.projector(feat_grid)
        return self.unet(x)


class SegmentationUNet(_ProjectedUNet):
    """training_discrete.py:50-88."""

    def __init__(self, feature_channels: int, cond_dim: int, model_channels: int, num_res_blocks: int,
                 channel_mult: Tuple[int, ...], attention_resolutions: Tuple[int, ...], grid_size: int,
                 num_classes: int):
        super().__init__(feature_channels, cond_dim, model_channels, num_res_blocks, channel_mult,
                         attention_resolutions, grid_size, num_classes)


class RegressionUNet(_ProjectedUNet):
    """training_continuous_mse.py:48-89."""

    def __init__(self, feature_channels: int, cond_dim: int, model_channels: int, num_res_blocks: int,
                 channel_mult: Tuple[int, ...], attention_resolutions: Tuple[int, ...], grid_size: int,
                 out_channels: int = 3):
        super().__init__(feature_channels, cond_dim, model_channels, num_res_blocks, channel_mult,
                         attention_resolutions, grid_size, out_channels)


# --------------------------------------------------------------------------------------------------
# Seeded parameters.  A freshly constructed reference network outputs exactly 0 (every ResBlock's
# second conv, attention proj_out and the head conv are zero_module'd), so parity on default
# initialisation is vacuous: all parameters are overwritten with seeded values (SURVEY.md §8d).
# --------------------------------------------------------------------------------------------------
def seeded_state_dict(model: nn.Module, seed: int = 0, conv_gain: float = 1.0) -> dict:
    """Deterministic, well-conditioned parameters for every tensor of `model`.

    Conv weights ~ N(0, conv_gain/fan_in) (so activations keep O(1) magnitude through ~100 layers),
    conv biases ~ 0.1 N(0,1), norm scales 1 + 0.1 N(0,1), norm shifts 0.1 N(0,1).
    """
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for name, t in model.state_dict().items():
        if name.endswith("weight") and t.dim() >= 3 and not _is_norm(model, name):
            fan_in = t[0].numel()
            sd[name] = torch.randn(t.shape, generator=g) * math.sqrt(conv_gain / fan_in)
        elif name.endswith("weight"):
            sd[name] = 1.0 + 0.1 * torch.randn(t.shape, generator=g)
        else:
            sd[name] = 0.1 * torch.randn(t.shape, generator=g)
    return sd


def _is_norm(model: nn.Module, param_name: str) -> bool:
    mod = model
    for part in param_name.split(".")[:-1]:
        mod = getattr(mod, part) if not part.isdigit() else mod[int(part)]
    return isinstance(mod, (nn.LayerNorm, nn.GroupNorm))


DEFAULT_CFG = dict(cond_dim=32, model_channels=64, num_res_blocks=3, channel_mult=(1, 1, 2, 4),
                   attention_resolutions=())   # config/training/default.yaml:92-97


def build_pair(feature_channels: int, grid_size: int, seed: int = 0, cfg: Optional[dict] = None):
    """(SegmentationUNet 8-class, RegressionUNet 3-channel) with seeded parameters, eval mode."""
    cfg = dict(DEFAULT_CFG if cfg is None else cfg)
    seg = SegmentationUNet(feature_channels=feature_channels, grid_size=grid_size, num_classes=8, **cfg)
    reg = RegressionUNet(feature_channels=feature_channels, grid_size=grid_size, out_channels=3, **cfg)
    seg.load_state_dict(seeded_state_dict(seg, seed))
    reg.load_state_dict(seeded_state_dict(reg, seed + 1))
    return seg.eval(), reg.eval()


def synthetic_features(n: int, channels: int, grid: int, seed: int = 0, scale: float = 0.05) -> torch.Tensor:
    """Synthetic CLIP-like voxel features as the dataset would deliver them: generated fp16 in the
    on-disk (N, D, H, W, C) layout (voxelize.py:86,111), returned fp32 (N, C, D, H, W)
    (my_data.py:160-224)."""
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(n, grid, grid, grid, channels, generator=g) * scale).to(torch.float16)
    return x.float().permute(0, 4, 1, 2, 3).contiguous()
