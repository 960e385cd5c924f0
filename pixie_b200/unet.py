"""Drop-in `SegmentationUNet` / `RegressionUNet` for the reference's inference path.

Mirrors the constructor arguments, `load_state_dict` key names, `.to()/.eval()` and `__call__`
contract of
  third_party/Wavelet-Generation/trainer/training_discrete.py:50-88      (SegmentationUNet)
  third_party/Wavelet-Generation/trainer/training_continuous_mse.py:48-89 (RegressionUNet)
as used by inference_combined.py:81-105 (create_models), training_utils.py:191-225
(load_checkpoint -> load_state_dict(strict=False)) and inference_combined.py:124-126 (forward under
torch.no_grad()).  The forward itself runs in libpixie_b200.so (wgmma implicit-GEMM convolutions,
see pixie_b200/csrc); PyTorch only owns the tensors and the stream.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional, Sequence, Tuple

import torch

from . import _lib

#: numerics of the convolutions (pixie_unet_config.precision): one fp16 tensor-core pass; three fp16 passes on hi/lo split
#: operands; or one fp16 pass + one E5M2 pass carrying the first-order rounding terms (2 pass-equivalents, meets 1e-3)
PRECISIONS = {"fp16": 0, "fp16x3": 1, "fp16e5": 2}


def _expected_keys(feature_channels, cond_dim, model_channels, num_res_blocks, channel_mult, grid_size, out_channels):
    """State-dict keys and shapes of the reference module (SURVEY.md appendix A), derived from the
    constructor logic of MyUNetModel.__init__ (diffusion_network.py:734-873)."""
    keys: Dict[str, Tuple[int, ...]] = {}

    def conv(name, co, ci, k):
        keys[name + ".weight"] = (co, ci) + (k,) * 3
        keys[name + ".bias"] = (co,)

    def norm_c(name, c):
        keys[name + ".weight"] = (c,)
        keys[name + ".bias"] = (c,)

    def ln(name, sp):
        keys[name + ".weight"] = (sp, sp, sp)
        keys[name + ".bias"] = (sp, sp, sp)

    def resblock(path, cin, cout, sp):
        ln(path + ".in_layers.0", sp)
        conv(path + ".in_layers.2", cout, cin, 3)
        ln(path + ".out_layers.0", sp)
        conv(path + ".out_layers.3", cout, cout, 3)
        if cin != cout:
            conv(path + ".skip_connection", cout, cin, 1)

    if feature_channels != cond_dim:
        if feature_channels > cond_dim:
            conv("projector.net.0", 128, feature_channels, 1); norm_c("projector.net.1", 128)
            conv("projector.net.3", 128, 128, 3); norm_c("projector.net.4", 128)
            conv("projector.net.6", cond_dim, 128, 1); norm_c("projector.net.7", cond_dim)
        else:
            conv("projector.net.0", cond_dim, feature_channels, 1); norm_c("projector.net.1", cond_dim)
    mc = model_channels
    conv("unet.input_blocks.0.0", mc, cond_dim, 3)
    chans, ch, sp, blk = [mc], mc, grid_size, 1
    sizes = [grid_size]
    for level, mult in enumerate(channel_mult):
        for _ in range(num_res_blocks):
            resblock(f"unet.input_blocks.{blk}.0", ch, mult * mc, sp)
            ch = mult * mc
            chans.append(ch); blk += 1
        if level != len(channel_mult) - 1:
            conv(f"unet.input_blocks.{blk}.0.op", ch, ch, 3)
            chans.append(ch); sizes.append(sp); blk += 1
            sp = (sp + 1) // 2
    resblock("unet.middle_block.0", ch, ch, sp)
    norm_c("unet.middle_block.1.norm", ch)
    keys["unet.middle_block.1.qkv.weight"] = (3 * ch, ch, 1); keys["unet.middle_block.1.qkv.bias"] = (3 * ch,)
    keys["unet.middle_block.1.proj_out.weight"] = (ch, ch, 1); keys["unet.middle_block.1.proj_out.bias"] = (ch,)
    resblock("unet.middle_block.2", ch, ch, sp)
    ob = 0
    for level, mult in list(enumerate(channel_mult))[::-1]:
        for i in range(num_res_blocks + 1):
            resblock(f"unet.output_blocks.{ob}.0", ch + chans.pop(), mc * mult, sp)
            ch = mc * mult
            if level and i == num_res_blocks:
                conv(f"unet.output_blocks.{ob}.1.conv", ch, ch, 3)
                sp = sizes.pop()
            ob += 1
    ln("unet.out.0", sp)
    conv("unet.out.2", out_channels, mc, 3)
    return keys


class _B200UNet:
    """Common implementation; not a torch.nn.Module on purpose (no autograd, no parameters on the
    torch side) but it answers the calls the reference makes on its modules."""

    def __init__(self, feature_channels: int, cond_dim: int, model_channels: int, num_res_blocks: int,
                 channel_mult: Sequence[int], attention_resolutions: Sequence[int], grid_size: int,
                 out_channels: int, max_batch: int = 4, precision: str = "fp16"):
        if tuple(attention_resolutions) != ():
            raise NotImplementedError(
                "attention_resolutions must be () (config/training/default.yaml:96); the bottleneck "
                "AttentionBlock of middle_block is always built")
        if precision not in PRECISIONS:
            raise ValueError("precision must be one of " + ", ".join(repr(k) for k in PRECISIONS))
        self.feature_channels, self.cond_dim = int(feature_channels), int(cond_dim)
        self.model_channels, self.num_res_blocks = int(model_channels), int(num_res_blocks)
        self.channel_mult = tuple(int(m) for m in channel_mult)
        self.grid_size, self.out_channels = int(grid_size), int(out_channels)
        self.max_batch, self.precision = int(max_batch), precision
        self._keys = _expected_keys(self.feature_channels, self.cond_dim, self.model_channels, self.num_res_blocks,
                                    self.channel_mult, self.grid_size, self.out_channels)
        self._state: Dict[str, torch.Tensor] = {}
        self._handle: Optional[C.c_void_p] = None
        self._device: Optional[torch.device] = None
        self.training = False

    # ---- torch.nn.Module-like surface used by the reference -------------------------------------
    def to(self, device):                      # create_models(...).to(rank)  (inference_combined.py:92)
        self._device = torch.device("cuda", device) if isinstance(device, int) else torch.device(device)
        if self._device.type != "cuda":
            raise _lib.PixieError("pixie_b200 U-Net runs on CUDA (sm_90) only; there is no CPU fallback")
        return self

    def cuda(self, device=None):
        return self.to(torch.device("cuda", torch.cuda.current_device() if device is None else device))

    def eval(self):
        self.training = False
        return self

    def train(self, mode: bool = True):
        if mode:
            raise NotImplementedError("inference-only: the training loop is outside the hot path")
        return self

    def state_dict(self):
        return dict(self._state)

    def load_state_dict(self, state_dict, strict: bool = True):
        """Accepts the reference's key names (optionally with the DDP 'module.' prefix stripped by
        training_utils.load_checkpoint). Returns (missing_keys, unexpected_keys) like torch."""
        missing, unexpected = [], []
        new_state = {}
        for k, v in state_dict.items():
            if k.startswith("module."):
                k = k[len("module."):]
            if k not in self._keys:
                unexpected.append(k)
                continue
            if tuple(v.shape) != self._keys[k]:
                raise RuntimeError(f"size mismatch for {k}: checkpoint {tuple(v.shape)} vs model {self._keys[k]}")
            new_state[k] = v.detach().to(torch.float32).cpu().contiguous()
        for k in self._keys:
            if k not in new_state and k not in self._state:
                missing.append(k)
        if strict and (missing or unexpected):
            raise RuntimeError(f"Error(s) in loading state_dict: missing {missing[:5]}..., unexpected {unexpected[:5]}...")
        self._state.update(new_state)
        self._destroy()                      # weights changed: rebuild lazily
        return missing, unexpected

    # ---- execution --------------------------------------------------------------------------------
    def _ensure_built(self):
        if self._handle is not None:
            return
        lib = _lib.require_device()
        missing = [k for k in self._keys if k not in self._state]
        if missing:
            raise _lib.PixieError(f"state dict incomplete, e.g. {missing[:3]}: call load_state_dict first "
                                  "(a reference network that was never loaded is all zeros anyway)")
        cfg = _lib.UNetConfig()
        cfg.feature_channels, cfg.cond_dim = self.feature_channels, self.cond_dim
        cfg.model_channels, cfg.num_res_blocks = self.model_channels, self.num_res_blocks
        cfg.n_levels = len(self.channel_mult)
        for i, m in enumerate(self.channel_mult):
            cfg.channel_mult[i] = m
        cfg.grid_size, cfg.out_channels = self.grid_size, self.out_channels
        cfg.max_batch = self.max_batch
        cfg.precision = PRECISIONS[self.precision]
        h = C.c_void_p()
        dev = self._device or torch.device("cuda", torch.cuda.current_device())
        with torch.cuda.device(dev):
            _lib.check(lib.pixie_unet_create(C.byref(cfg), C.byref(h)))
            try:
                for k, v in self._state.items():
                    shape = (C.c_int64 * v.dim())(*v.shape)
                    _lib.check(lib.pixie_unet_set_tensor(h, k.encode(), _lib.ptr(v), shape, v.dim()))
                _lib.check(lib.pixie_unet_finalize(h))
            except Exception:
                lib.pixie_unet_destroy(h)
                raise
        self._handle, self._device = h, dev

    def _destroy(self):
        if self._handle is not None:
            _lib.load().pixie_unet_destroy(self._handle)
            self._handle = None

    def __del__(self):
        try:
            self._destroy()
        except Exception:
            pass

    def __call__(self, feat_grid: torch.Tensor) -> torch.Tensor:
        return self.forward(feat_grid)

    def forward(self, feat_grid: torch.Tensor) -> torch.Tensor:
        """feat_grid: float32 (N, C, D, H, W) as the reference's dataset delivers it
        (my_data.py:160-224) -> float32 (N, out_channels, D, H, W)."""
        self._ensure_built()
        lib = _lib.load()
        G = self.grid_size
        if feat_grid.dim() != 5 or tuple(feat_grid.shape[1:]) != (self.feature_channels, G, G, G):
            raise ValueError(f"expected (N,{self.feature_channels},{G},{G},{G}), got {tuple(feat_grid.shape)}")
        x = feat_grid.to(self._device, torch.float32).contiguous()
        n = x.shape[0]
        out = torch.empty((n, self.out_channels, G, G, G), dtype=torch.float32, device=self._device)
        with torch.cuda.device(self._device):
            st = _lib.stream(self._device)
            for b0 in range(0, n, self.max_batch):
                nb = min(self.max_batch, n - b0)
                _lib.check(lib.pixie_unet_forward_ncdhw(self._handle, _lib.ptr(x[b0:b0 + nb]), nb, _lib.ptr(out[b0:b0 + nb]), st))
        return out

    def forward_channels_last_f16(self, feat_ndhwc: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Fast path: float16 (N, D, H, W, C) on the device — the on-disk layout of
        clip_features_features.npy (voxelize.py:86,111), no conversion pass."""
        self._ensure_built()
        lib = _lib.load()
        G = self.grid_size
        if feat_ndhwc.dtype != torch.float16 or tuple(feat_ndhwc.shape[1:]) != (G, G, G, self.feature_channels):
            raise ValueError("expected float16 (N,D,H,W,C)")
        if self.feature_channels % 64:
            raise ValueError("channels-last fast path needs feature_channels % 64 == 0")
        x = feat_ndhwc.to(self._device).contiguous()
        n = x.shape[0]
        if out is None:
            out = torch.empty((n, self.out_channels, G, G, G), dtype=torch.float32, device=self._device)
        elif tuple(out.shape) != (n, self.out_channels, G, G, G) or out.dtype != torch.float32 or not out.is_contiguous():
            raise ValueError("out must be a contiguous float32 (N, out_channels, D, H, W) device tensor")
        with torch.cuda.device(self._device):
            st = _lib.stream(self._device)
            for b0 in range(0, n, self.max_batch):
                nb = min(self.max_batch, n - b0)
                _lib.check(lib.pixie_unet_forward(self._handle, _lib.ptr(x[b0:b0 + nb]), nb, _lib.ptr(out[b0:b0 + nb]), st))
        return out

    def forward_host(self, feat_ndhwc_pinned: torch.Tensor, out_pinned: Optional[torch.Tensor] = None) -> torch.Tensor:
        """End-to-end call with HOST buffers (pinned fp16 NDHWC in, fp32 NCDHW out): the H2D copy,
        the forward and the D2H copy all happen inside the C-ABI call."""
        self._ensure_built()
        lib = _lib.load()
        G = self.grid_size
        n = feat_ndhwc_pinned.shape[0]
        if n > self.max_batch:
            raise ValueError("batch exceeds max_batch")
        if out_pinned is None:
            out_pinned = torch.empty((n, self.out_channels, G, G, G), dtype=torch.float32).pin_memory()
        with torch.cuda.device(self._device):
            _lib.check(lib.pixie_unet_forward_host(self._handle, _lib.ptr(feat_ndhwc_pinned), n, _lib.ptr(out_pinned),
                                                   _lib.stream(self._device)))
        return out_pinned

    # ---- introspection used by bench/tests --------------------------------------------------------
    def check(self):
        _lib.check(_lib.load().pixie_unet_check(self._handle))

    def launch_count(self) -> int:
        self._ensure_built()
        return int(_lib.load().pixie_unet_launch_count(self._handle))

    def flops(self) -> float:
        self._ensure_built()
        return float(_lib.load().pixie_unet_flops(self._handle))

    def profile(self, feat_ndhwc: torch.Tensor):
        """Per-launch device times of one forward: list of (kind, ms, algorithmic_flops)."""
        self._ensure_built()
        lib = _lib.load()
        G = self.grid_size
        n = feat_ndhwc.shape[0]
        out = torch.empty((n, self.out_channels, G, G, G), dtype=torch.float32, device=self._device)
        cap = 1024
        ms, kinds, fl = (C.c_float * cap)(), (C.c_int * cap)(), (C.c_double * cap)()
        with torch.cuda.device(self._device):
            k = lib.pixie_unet_profile(self._handle, _lib.ptr(feat_ndhwc), n, _lib.ptr(out), _lib.stream(self._device), ms, kinds, fl, cap)
        if k < 0:
            raise _lib.last_error()
        names = {0: "conv", 1: "moments", 2: "norm", 3: "upsample", 4: "attention"}
        return [(names[kinds[i]], ms[i], fl[i]) for i in range(k)]

    def debug_fetch(self, name: str, channels: int, sp: int, batch: int = 1) -> torch.Tensor:
        """Intermediate activation by reference module path, returned as (N, C, D, H, W) fp32 (CPU)."""
        buf = torch.empty(batch * sp ** 3 * channels, dtype=torch.float32)
        n = _lib.load().pixie_unet_debug_fetch(self._handle, name.encode(), _lib.ptr(buf), buf.numel())
        if n < 0:
            raise _lib.last_error()
        return buf[:n].view(batch, sp, sp, sp, channels).permute(0, 4, 1, 2, 3).contiguous()

    def debug_names(self) -> Dict[str, Tuple[int, int]]:
        """Activations `debug_fetch` can copy: {module path: (channels, spatial side)}."""
        self._ensure_built()
        lib = _lib.load()
        n = lib.pixie_unet_debug_names(self._handle, None, 0)
        if n < 0:
            raise _lib.last_error()
        buf = C.create_string_buffer(n + 1)
        lib.pixie_unet_debug_names(self._handle, buf, n + 1)
        names = {}
        for line in buf.value.decode().splitlines():
            name, ch, sp = line.split()
            names[name] = (int(ch), int(sp))
        return names


class SegmentationUNet(_B200UNet):
    """training_discrete.py:50-88."""

    def __init__(self, feature_channels: int, cond_dim: int, model_channels: int, num_res_blocks: int,
                 channel_mult: Tuple[int, ...], attention_resolutions: Tuple[int, ...], grid_size: int,
                 num_classes: int, **kw):
        super().__init__(feature_channels, cond_dim, model_channels, num_res_blocks, channel_mult,
                         attention_resolutions, grid_size, num_classes, **kw)


class RegressionUNet(_B200UNet):
    """training_continuous_mse.py:48-89."""

    def __init__(self, feature_channels: int, cond_dim: int, model_channels: int, num_res_blocks: int,
                 channel_mult: Tuple[int, ...], attention_resolutions: Tuple[int, ...], grid_size: int,
                 out_channels: int = 3, **kw):
        super().__init__(feature_channels, cond_dim, model_channels, num_res_blocks, channel_mult,
                         attention_resolutions, grid_size, out_channels, **kw)
