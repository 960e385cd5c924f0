"""Generates tests/golden/unet_small.npz and tests/golden/unet_ref_modules.npz by running the REFERENCE modules (imported
from a checkout of vlongle/pixie) on seeded inputs:

    PIXIE_REFERENCE=<checkout of the reference> python tests/golden/make_unet_golden.py

The vectors pin oracle/unet_ref.py (and through it the CUDA path) to the reference's own outputs.
Config is a reduced one (grid 8, 64 feature channels) so the fixture stays small; the architecture code
path (projector, 4 levels, 3 res blocks, bottleneck attention, concat skips, up/down-sampling) is the
full one of config/training/default.yaml.
"""
import os
import sys

import numpy as np
import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(os.environ["PIXIE_REFERENCE"], "third_party", "Wavelet-Generation"))

from models.module.diffusion_network import FeatureProjector, MyUNetModel  # noqa: E402  (the reference)
from oracle import unet_ref as O  # noqa: E402  (only for the seeded parameter / input generators)

C, G = 64, 8


class RefNet(nn.Module):
    """SegmentationUNet / RegressionUNet body (training_discrete.py:51-88) around the reference modules."""

    def __init__(self, out):
        super().__init__()
        self.projector = FeatureProjector(C, out_channels=32, hidden_channels=128)
        self.unet = MyUNetModel(in_channels=32, model_channels=64, out_channels=out, num_res_blocks=3,
                                channel_mult=(1, 1, 2, 4), attention_resolutions=(), spatial_size=G, dims=3,
                                activation=nn.LeakyReLU(0.02))

    def forward(self, x):
        return self.unet(self.projector(x))


def main():
    torch.manual_seed(0)
    torch.set_num_threads(1)
    out = {}
    x = O.synthetic_features(2, C, G, seed=11, scale=1.0)
    out["x"] = x.numpy()
    for name, oc, seed in (("reg", 3, 5), ("seg", 8, 6)):
        net = RefNet(oc).eval()
        sd = O.seeded_state_dict(net, seed)
        net.load_state_dict(sd)
        with torch.no_grad():
            y = net(x)
        out[f"{name}_y"] = y.numpy()
        out[f"{name}_seed"] = np.int64(seed)
    np.savez_compressed(os.path.join(os.path.dirname(__file__), "unet_small.npz"), **out)
    print({k: (v.shape if hasattr(v, "shape") else v) for k, v in out.items()})

    # unet_ref_modules.npz: the reference modules at a second configuration (96 feature channels, grid 16, no attention),
    # their parameter names in order, and their output; tests/test_oracle_unet.py requires the oracle to reproduce both
    ref = nn.Module()
    ref.projector = FeatureProjector(96, out_channels=32, hidden_channels=128)
    ref.unet = MyUNetModel(in_channels=32, model_channels=64, out_channels=3, num_res_blocks=3, channel_mult=(1, 1, 2, 4),
                           attention_resolutions=(), spatial_size=16, dims=3, activation=nn.LeakyReLU(0.02))
    ref.eval()
    mine = O.RegressionUNet(96, 32, 64, 3, (1, 1, 2, 4), (), 16, 3).eval()
    ref.load_state_dict(O.seeded_state_dict(mine, 0))
    x = O.synthetic_features(1, 96, 16, seed=3)
    with torch.no_grad():
        y = ref.unet(ref.projector(x))
    np.savez_compressed(os.path.join(os.path.dirname(__file__), "unet_ref_modules.npz"), y=y.numpy(),
                        keys=np.array(list(ref.state_dict().keys())), x_seed=np.int64(3), sd_seed=np.int64(0))


if __name__ == "__main__":
    main()
