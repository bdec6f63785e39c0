"""Mirror of reference utils/splat2d_cuda/__init__.py (`from .splat import *`)."""
import torch.nn as nn

from .blend import LaplacianBlender, laplacian_blend, splat_points
from .functional import (nn_argmin, splat2d, splat2d_lookup, splat_composite_grid, splat_lookup_composite_grid,
                         track_points_lerp)

__all__ = ["Splat2D", "splat2d", "splat2d_lookup", "nn_argmin", "track_points_lerp", "laplacian_blend", "LaplacianBlender",
           "splat_points", "splat_composite_grid", "splat_lookup_composite_grid"]


class Splat2D(nn.Module):
    """nn.Module face of splat2d.  (The reference's Splat2D.forward, splat.py:12-13, calls splat2d with a stale
    five-argument order and is dead code there; this one takes splat2d's real signature.)"""

    def forward(self, input, coordinates, values, sigma, soft_normalize=False):
        return splat2d(input, coordinates, values, sigma, soft_normalize)
