"""Host-side mirror of the reference's inference hot loop
(third_party/Wavelet-Generation/trainer/inference_combined.py): create_models (:81-105),
process_batch's forward + argmax (:122-126) and save_predictions' (3 + n_classes, D, H, W) packing
(:173-199) — without the metrics / file I/O, which stay outside the hot path.
"""
from __future__ import annotations

import os
from typing import Optional, Tuple

import torch

from . import _lib
from .unet import RegressionUNet, SegmentationUNet


class MaterialFieldPredictor:
    """seg_network + cont_network resident on one GPU; one H2D of the voxel grid serves both."""

    def __init__(self, feature_channels: int, cond_dim: int = 32, model_channels: int = 64, num_res_blocks: int = 3,
                 channel_mult: Tuple[int, ...] = (1, 1, 2, 4), attention_resolutions: Tuple[int, ...] = (),
                 grid_size: int = 64, num_material_classes: int = 8, device="cuda:0", max_batch: int = 1,
                 precision: str = "fp16e5"):
        kw = dict(feature_channels=feature_channels, cond_dim=cond_dim, model_channels=model_channels,
                  num_res_blocks=num_res_blocks, channel_mult=channel_mult, attention_resolutions=attention_resolutions,
                  grid_size=grid_size, max_batch=max_batch, precision=precision)
        self.seg_network = SegmentationUNet(num_classes=num_material_classes, **kw).to(device)
        self.cont_network = RegressionUNet(out_channels=3, **kw).to(device)
        self.device = torch.device(device)
        self.grid_size, self.feature_channels = grid_size, feature_channels
        self.n_classes, self.max_batch = num_material_classes, max_batch
        self._pipe = None
        self._side: Optional[torch.cuda.Stream] = None
        self._two_streams = os.environ.get("PIXIE_UNET_STREAMS", "2") != "1"
        self._feat_dev: Optional[torch.Tensor] = None
        self._packed_dev: Optional[torch.Tensor] = None

    def load_state_dicts(self, seg_sd, cont_sd, strict: bool = True):
        self.seg_network.load_state_dict(seg_sd, strict=strict)
        self.cont_network.load_state_dict(cont_sd, strict=strict)
        return self

    def predict(self, feat_ndhwc_f16: torch.Tensor, seg_out: Optional[torch.Tensor] = None, cont_out: Optional[torch.Tensor] = None):
        """Device fp16 (N, D, H, W, C) -> (seg_logits (N, n_classes, D,H,W), cont_pred (N, 3, D,H,W)) fp32.

        The two networks are independent (inference_combined.py:122-126 calls them one after the other on the same grid): the
        regression network is enqueued on a side stream, so that the latency-bound 8^3 / 16^3 levels of one network (a few
        dozen 20-us launches that fill a fraction of the SMs) overlap with the other network's work. Both forwards are CUDA-graph
        replays; the caller's stream waits for the side stream before this returns."""
        if not self._two_streams:
            return (self.seg_network.forward_channels_last_f16(feat_ndhwc_f16, seg_out),
                    self.cont_network.forward_channels_last_f16(feat_ndhwc_f16, cont_out))
        main = torch.cuda.current_stream(self.device)
        if self._side is None:
            self._side = torch.cuda.Stream(device=self.device)
        side = self._side
        side.wait_stream(main)
        with torch.cuda.stream(side):
            cont = self.cont_network.forward_channels_last_f16(feat_ndhwc_f16, cont_out)
        seg = self.seg_network.forward_channels_last_f16(feat_ndhwc_f16, seg_out)
        main.wait_stream(side)
        cont.record_stream(main)
        feat_ndhwc_f16.record_stream(side)
        return seg, cont

    def pack(self, seg_logits: torch.Tensor, cont_pred: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """(N, 3 + n_classes, D, H, W): continuous channels + one-hot argmax, as sample_*_pred.npy."""
        n, G = seg_logits.shape[0], self.grid_size
        if out is None:
            out = torch.empty((n, 3 + self.n_classes, G, G, G), dtype=torch.float32, device=self.device)
        _lib.call("pixie_pack_predictions", self.device, seg_logits, cont_pred, out, n, G ** 3, self.n_classes)
        return out

    def check(self):
        """Raises PixieError if a convolution of either network gave up waiting on its pipeline (the flag the kernels set
        instead of hanging). Synchronises the device."""
        self.seg_network.check()
        self.cont_network.check()

    def predict_packed_host_stream(self, feats_pinned, outs_pinned=None):
        """Many scenes end to end with HOST buffers, software-pipelined: while scene i runs through the two networks, scene i+1's
        grid (268 MB at 64^3 x 512) is already crossing PCIe on a copy stream into the other of two device buffers. Per scene the
        same work as `predict_packed_host` (H2D grid, both networks, packing, D2H field); returns the list of pinned outputs after
        everything has finished.

        `feats_pinned`: iterable of pinned fp16 (N, D, H, W, C) tensors (N <= max_batch), or of objects with a `.tensor`
        attribute such as `voxel_io.scene_stream` yields. It is consumed LAZILY, one scene ahead of the networks, and every item
        that has an `h2d_done` attribute gets the CUDA event recorded after its host->device copy: a producer that recycles
        pinned buffers (scene_stream does) waits on that event before it overwrites the buffer."""
        G = self.grid_size
        outs = [] if outs_pinned is None else list(outs_pinned)
        with torch.cuda.device(self.device):
            if self._pipe is None:
                nb = self.max_batch
                self._pipe = {
                    "in": [torch.empty((nb, G, G, G, self.feature_channels), dtype=torch.float16, device=self.device) for _ in range(2)],
                    "out": [torch.empty((nb, 3 + self.n_classes, G, G, G), dtype=torch.float32, device=self.device) for _ in range(2)],
                    # fixed network outputs per slot: the forward is a CUDA graph keyed by its input / output addresses
                    "seg": [torch.empty((nb, self.n_classes, G, G, G), dtype=torch.float32, device=self.device) for _ in range(2)],
                    "cont": [torch.empty((nb, 3, G, G, G), dtype=torch.float32, device=self.device) for _ in range(2)],
                    "copy_stream": torch.cuda.Stream(device=self.device),
                }
            P = self._pipe
            main = torch.cuda.current_stream(self.device)
            cs = P["copy_stream"]
            consumed = []
            cs.wait_stream(main)
            for i, item in enumerate(feats_pinned):
                f = item.tensor if hasattr(item, "tensor") else item
                n, slot = f.shape[0], i % 2
                if n > self.max_batch:
                    raise ValueError("batch exceeds max_batch")
                if i >= len(outs):
                    outs.append(torch.empty((n, 3 + self.n_classes, G, G, G), dtype=torch.float32).pin_memory())
                copied = torch.cuda.Event()
                with torch.cuda.stream(cs):
                    if i >= 2:
                        cs.wait_event(consumed[i - 2])          # the networks are done reading this input slot
                    P["in"][slot][:n].copy_(f, non_blocking=True)
                    copied.record(cs)
                if hasattr(item, "h2d_done"):
                    item.h2d_done = copied                      # the producer may rewrite the pinned buffer after this event
                main.wait_event(copied)
                seg, cont = self.predict(P["in"][slot][:n], P["seg"][slot][:n], P["cont"][slot][:n])
                ev = torch.cuda.Event()
                ev.record(main)
                consumed.append(ev)
                self.pack(seg, cont, P["out"][slot][:n])
                outs[i].copy_(P["out"][slot][:n], non_blocking=True)     # stream-ordered: slot reuse two scenes later is safe
            main.synchronize()
            self.check()
        return outs

    def predict_packed_host(self, feat_pinned: torch.Tensor, out_pinned: Optional[torch.Tensor] = None) -> torch.Tensor:
        """End to end with HOST buffers: pinned fp16 (N, D, H, W, C) -> pinned fp32 (N, 3+n_classes, D,H,W).
        One H2D copy of the grid, both networks, packing, one D2H copy; returns after the stream syncs."""
        n, G = feat_pinned.shape[0], self.grid_size
        if self._feat_dev is None or self._feat_dev.shape[0] < n:
            self._feat_dev = torch.empty((max(n, self.max_batch), G, G, G, self.feature_channels), dtype=torch.float16, device=self.device)
            self._packed_dev = torch.empty((max(n, self.max_batch), 3 + self.n_classes, G, G, G), dtype=torch.float32, device=self.device)
        if out_pinned is None:
            out_pinned = torch.empty((n, 3 + self.n_classes, G, G, G), dtype=torch.float32).pin_memory()
        with torch.cuda.device(self.device):
            self._feat_dev[:n].copy_(feat_pinned, non_blocking=True)
            seg, cont = self.predict(self._feat_dev[:n])
            self.pack(seg, cont, self._packed_dev[:n])
            out_pinned.copy_(self._packed_dev[:n], non_blocking=True)
            torch.cuda.current_stream().synchronize()
            self.check()
        return out_pinned
