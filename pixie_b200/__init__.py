"""pixie_b200 — H100-native (sm_90a) hot path of vlongle/pixie.

Two drop-in surfaces over one C-ABI library (include/pixie_b200.h, built in-tree as
pixie_b200/libpixie_b200.so):

  * pixie_b200.unet.SegmentationUNet / RegressionUNet   (material-field U-Net forward)
  * pixie_b200.mpm_solver_warp.MPM_Simulator_WARP       (PhysGaussian MLS-MPM rollout)

There is no CPU or PyTorch fallback: importing is cheap, but any compute call raises unless the CUDA
library is built and an sm_90 (H100) device is present.
"""
__version__ = "0.1.0"
