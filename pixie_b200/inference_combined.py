"""Command line of the reference's NEURAL_INFERENCE step (WG/trainer/inference_combined.py): evaluate the two material
networks on labelled scenes and write their predictions.

    python -m pixie_b200.inference_combined --render_outputs_dir <dir> --seg_checkpoint <seg .pth> \\
        --cont_checkpoint <cont .pth> --normalization_ranges <normalization_ranges.yaml> --output_dir <dir> \\
        [--obj_id ID] [--sample_id 0] [--batch_size 4] [--background_id 7] [--feature_channels 768] [--precision fp16e5] \\
        [--use_saved_test_split] [--train_size 0.9] [--dispersion sem|std]

The flags map to the reference's config keys (paths.render_outputs_dir, training.sample_id, training.inference.batch_size,
training.background_id, training.feature_channels, training.inference.use_saved_test_split, training.training.train_size).
Scenes are found as MaterialVoxelDataset finds them (problematic_objects.json is read next to the ranges file), the test
split is load_test_dataset's, and every object gets `<output_dir>/<obj_id>/sample_<id>_{pred,gt,mask,info}.npy`; rank 0
writes metrics.json and evaluated_obj_ids.json. Under torchrun the scenes are sharded in DistributedSampler(shuffle=False)
order and the metric lists are gathered to rank 0.

Per batch: the float16 feature grids go to the device as they are on disk (no fp32 NCDHW copy), both networks run, one
device pass (network_files.material_metrics) normalises the ground truth and reduces the accuracy counts and MSE sums, and
the packed prediction comes back to the host. The per-class table (generate_class_table) is not written.
"""
from __future__ import annotations

import argparse
import logging
import os
from typing import Optional, Sequence

import numpy as np
import torch

from . import dist_utils, network_files as NF, voxel_io
from .inference import MaterialFieldPredictor

log = logging.getLogger("pixie_b200.inference_combined")

#: config/training/default.yaml's U-Net (training.training.unet_*, cond_dim, attention_resolutions)
UNET_CFG = dict(cond_dim=32, model_channels=64, num_res_blocks=3, channel_mult=(1, 1, 2, 4))


def parser() -> argparse.ArgumentParser:
    p = argparse.ArgumentParser(prog="python -m pixie_b200.inference_combined", description=__doc__.split("\n\n")[0])
    p.add_argument("--render_outputs_dir", required=True)
    p.add_argument("--seg_checkpoint", required=True)
    p.add_argument("--cont_checkpoint", required=True)
    p.add_argument("--normalization_ranges", required=True, help="normalization_stats/normalization_ranges.yaml")
    p.add_argument("--output_dir", required=True)
    p.add_argument("--obj_id", default=None)
    p.add_argument("--sample_id", type=int, default=0)
    p.add_argument("--batch_size", type=int, default=4)
    p.add_argument("--background_id", type=int, default=7)
    p.add_argument("--feature_channels", type=int, default=768)
    p.add_argument("--grid_size", type=int, default=64)
    p.add_argument("--num_material_classes", type=int, default=8)
    p.add_argument("--precision", default="fp16e5", choices=["fp16e5", "fp16x3", "fp16"])
    p.add_argument("--use_saved_test_split", action="store_true")
    p.add_argument("--train_size", type=float, default=0.9)
    p.add_argument("--dispersion", default="sem", choices=["sem", "std"])
    return p


class _Evaluator:
    """Device buffers of one rank, sized for `batch_size` scenes and reused batch after batch (the network forwards are
    CUDA graphs keyed by their buffer addresses)."""

    def __init__(self, predictor: MaterialFieldPredictor, ds: NF.MaterialVoxelDataset, batch_size: int):
        D, dev = ds.D, predictor.device
        self.p, self.ds, self.dev = predictor, ds, dev
        pin = lambda t: t.pin_memory()                                                  # noqa: E731
        self.feat_h = pin(torch.empty((batch_size, D, D, D, ds.C_feat), dtype=torch.float16))
        self.mat_h = pin(torch.empty((batch_size, D, D, D, ds.C_mat), dtype=torch.float32))
        self.mask_h = pin(torch.empty((batch_size, D, D, D), dtype=torch.float32))
        self.feat = torch.empty(self.feat_h.shape, dtype=torch.float16, device=dev)
        self.mat = torch.empty(self.mat_h.shape, dtype=torch.float32, device=dev)
        self.mask = torch.empty(self.mask_h.shape, dtype=torch.float32, device=dev)
        self.seg = torch.empty((batch_size, ds.n_classes, D, D, D), dtype=torch.float32, device=dev)
        self.cont = torch.empty((batch_size, 3, D, D, D), dtype=torch.float32, device=dev)
        self.gt = torch.empty((batch_size, 4, D, D, D), dtype=torch.float32, device=dev)
        self.packed = torch.empty((batch_size, 3 + ds.n_classes, D, D, D), dtype=torch.float32, device=dev)

    def batch(self, idxs: Sequence[int], ranges, background_id: int, metrics: NF.InferenceMetrics, output_dir: Optional[str]):
        n, ds = len(idxs), self.ds
        for k, i in enumerate(idxs):
            voxel_io.load_feature_grid(ds.feature_files[i], out=self.feat_h[k:k + 1])
            mat, mask = ds.load_labels(i)
            self.mat_h[k].numpy()[...] = mat
            self.mask_h[k].numpy()[...] = mask
        with torch.cuda.device(self.dev):
            for d, h in ((self.feat, self.feat_h), (self.mat, self.mat_h), (self.mask, self.mask_h)):
                d[:n].copy_(h[:n], non_blocking=True)
            seg, cont = self.p.predict(self.feat[:n], self.seg[:n], self.cont[:n])
            _, counts, sums = NF.material_metrics(self.mat[:n], self.mask[:n], seg, cont, ranges, background_id, gt_out=self.gt[:n])
            if output_dir:
                self.p.pack(seg, cont, self.packed[:n])
                packed, gt = self.packed[:n].cpu().numpy(), self.gt[:n].cpu().numpy()
        batch, samples = NF.batch_metrics(counts, sums)
        metrics.add_batch_metrics(*batch)
        for k, i in enumerate(idxs):
            obj_id = ds.obj_ids[i]
            metrics.add_sample_metrics(obj_id, samples[k])
            metrics.local_obj_ids.append(obj_id)
            if output_dir:
                NF.save_predictions(output_dir, ds.info(i), packed[k], gt[k], self.mask_h[k].numpy().copy())


def main(argv: Optional[Sequence[str]] = None, device=None) -> int:
    args = parser().parse_args(argv)
    rank, world, local = dist_utils.env_rank_world()
    device = torch.device(device if device is not None else f"cuda:{local}")
    dist_utils.init(device=device if device.type == "cuda" else None)
    ranges = NF.load_normalization_ranges(args.normalization_ranges)
    ds = NF.MaterialVoxelDataset(args.render_outputs_dir, sample_id=args.sample_id, grid_size=args.grid_size,
                                 feature_channels=args.feature_channels, num_material_classes=args.num_material_classes,
                                 background_id=args.background_id,
                                 problematic_objects=os.path.join(os.path.dirname(os.path.abspath(args.normalization_ranges)),
                                                                  "problematic_objects.json"))
    try:
        test = NF.load_test_dataset(ds, args.obj_id, args.use_saved_test_split, args.seg_checkpoint, args.train_size)
    except ValueError as e:
        if rank == 0:
            log.error(str(e))
        return 1
    mine = [test[k] for k in dist_utils.shard_scenes(len(test), rank, world)]
    if rank == 0:
        os.makedirs(args.output_dir, exist_ok=True)
        log.info(f"Results will be saved to: {args.output_dir}")
        log.info(f"Testing on {len(test)} samples")
    seg_sd = NF.load_network_checkpoint(args.seg_checkpoint)
    cont_sd = NF.load_network_checkpoint(args.cont_checkpoint)
    if seg_sd is None or cont_sd is None:
        raise FileNotFoundError("both --seg_checkpoint and --cont_checkpoint must exist: an untrained network is not evaluated")
    predictor = MaterialFieldPredictor(args.feature_channels, grid_size=args.grid_size, num_material_classes=args.num_material_classes,
                                       device=device, max_batch=args.batch_size, precision=args.precision, **UNET_CFG)
    predictor.load_state_dicts(seg_sd, cont_sd, strict=False)              # training_utils.load_checkpoint loads non-strictly
    ev = _Evaluator(predictor, ds, args.batch_size)
    metrics = NF.InferenceMetrics()
    for b in range(0, len(mine), args.batch_size):
        ev.batch(mine[b:b + args.batch_size], ranges, args.background_id, metrics, args.output_dir)
    predictor.check()
    gathered = metrics.gather_all_metrics(rank, world)
    if rank == 0:
        NF.generate_metrics_report(gathered, args.output_dir, args.seg_checkpoint, args.cont_checkpoint, args.dispersion)
    dist_utils.barrier()
    return 0


if __name__ == "__main__":
    logging.basicConfig(level=logging.INFO)
    raise SystemExit(main())
