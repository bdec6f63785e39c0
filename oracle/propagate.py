"""Torch restatement of the propagation grid (test infrastructure -- see oracle/__init__.py).

Reference: applications/propagate_to_images.py:62-73 (`make_visuals`: uncongeal_points on the flipped images, the x
mirror where flipped, splat_points and write()), with spatial_transformer.py:141-157 (`uncongeal_points`: F.grid_sample
of the sampling grid, 'border', and `unnormalize` :621-623) and oracle.labels' splat-and-grid composition.  In float32 it
is the reference's own composition; in float64 (float64 images, `return_values`) the accuracy reference of the CUDA op.
"""
import types

import torch
import torch.nn.functional as F

from . import labels as _labels
from . import training_vis as _training_vis


def lookup_points_ref(grid, query, flip, r):
    """(N, Hg, Wg, 2) grids x (1 or N, P, 2) queries -> (N, P, 2) pixels of the R x R images, mirrored where flip."""
    n = grid.size(0)
    q = query.expand(n, -1, -1).to(grid.dtype)
    pts = F.grid_sample(grid.permute(0, 3, 1, 2), q.unsqueeze(2), padding_mode="border",
                        align_corners=False).squeeze(3).permute(0, 2, 1)
    pts = pts.div((r - 1) / r).div(2).add(0.5).mul(r - 1)
    if flip is not None:
        pts = pts.clone()
        pts[:, :, 0] = torch.where(flip.view(-1, 1).bool(), r - 1 - pts[:, :, 0], pts[:, :, 0])
    return pts


def splat_lookup_composite_grid_ref(images, grid, query, flip, colors, alpha_channel, sigma, opacity, nrow, padding=2,
                                    return_values=False):
    """The op set's splat_lookup_composite_grid: -> ((Hg, Wg, 3) uint8, (N, P, 2) float32 points) (and, with
    return_values, the grid's values v * 255 + 0.5 before clamp and cast)."""
    r = images.size(-1)
    pts = lookup_points_ref(grid, query, flip, r).float()
    out = _labels.splat_composite_grid_ref(images.unsqueeze(0), pts.unsqueeze(0), colors, alpha_channel, sigma, opacity, nrow,
                                           padding=padding, return_values=return_values)
    if return_values:
        return out[0][0], pts, out[1][0]
    return out[0], pts


def cpu_ops():
    """oracle.training_vis.cpu_ops() plus `splat_lookup_composite_grid`: the op set that runs
    gangealing_b200.evaluation.propagate on the CPU restatement."""
    return types.SimpleNamespace(**vars(_training_vis.cpu_ops()), splat_lookup_composite_grid=splat_lookup_composite_grid_ref)
