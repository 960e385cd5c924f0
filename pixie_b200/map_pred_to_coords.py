"""Command line of the reference's MAP_PRED_TO_COORDS step (pixie/voxel/map_pred_to_coords.py): turn a packed prediction
into the material point cloud `gs_simulation --point_cloud_path` reads.

    python -m pixie_b200.map_pred_to_coords --pred_path <sample_0_pred.npy> --mask_path <clip_features_mask.npy> \\
        --grid_feature_path <clip_features.npz> --output_path <mapped_preds.ply> \\
        --normalization_ranges <normalization_ranges.yaml> [--world_output_path <world_mapped_preds.ply>] \\
        [--dataparser_path <dataparser_transforms.json>]

With --world_output_path and no --dataparser_path, dataparser_transforms.json is looked for next to the grid file, as the
reference does. The unscaling and the vertex table run on the device (material_transfer.extract_material_points); the
files are the bytes plyfile writes.
"""
from __future__ import annotations

import argparse
import logging
from typing import Optional, Sequence

from . import network_files as NF


def parser() -> argparse.ArgumentParser:
    p = argparse.ArgumentParser(prog="python -m pixie_b200.map_pred_to_coords", description=__doc__.split("\n\n")[0])
    p.add_argument("--pred_path", required=True)
    p.add_argument("--mask_path", required=True)
    p.add_argument("--grid_feature_path", required=True, help="clip_features.npz with min_bounds, max_bounds, grid_shape")
    p.add_argument("--output_path", required=True)
    p.add_argument("--normalization_ranges", required=True, help="normalization_stats/normalization_ranges.yaml")
    p.add_argument("--obj_id", default=None)
    p.add_argument("--world_output_path", default=None)
    p.add_argument("--dataparser_path", default=None)
    return p


def main(argv: Optional[Sequence[str]] = None, device="cuda:0") -> int:
    args = parser().parse_args(argv)
    ranges = NF.load_normalization_ranges(args.normalization_ranges)
    NF.map_pred_to_ply(args.pred_path, args.mask_path, args.grid_feature_path, args.output_path, args.obj_id,
                       world_output_path=args.world_output_path, dataparser_path=args.dataparser_path, ranges=ranges, device=device)
    return 0


if __name__ == "__main__":
    logging.basicConfig(level=logging.INFO)
    raise SystemExit(main())
