"""Torch restatement of the label-propagation frames (test infrastructure -- see oracle/__init__.py).

Reference: applications/vis_correspondence.py:133-158 (`visualize_label_propagation`) with utils/vis_tools/helpers.py:39-43
(`images2grid`: torchvision make_grid(normalize=True, range=(-1, 1)), then mul(255), add(0.5), clamp(0, 255) and a
truncating uint8 cast) and :134-194 (`splat_points`, alpha blending; oracle.splat.splat_points_ref).  In float32 it is
the reference's own composition; in float64 (`return_values`) it is the accuracy reference of the CUDA op.
"""
import types

import torch
from torchvision.utils import make_grid

from . import splat as _splat
from . import vis as _vis


def images2grid_ref(images, nrow, padding=2, return_values=False):
    """(N, 3, R, R) in [-1, 1] -> (Hg, Wg, 3) uint8 (and, with return_values, the value before clamp and cast)."""
    grid = make_grid(images, nrow=nrow, padding=padding, normalize=True, value_range=(-1, 1))
    v = grid.mul(255).add_(0.5)
    out = v.clamp(0, 255).permute(1, 2, 0).to(torch.uint8)
    return (out, v.permute(1, 2, 0)) if return_values else out


def splat_composite_grid_ref(images, points, colors, alpha_channel, sigma, opacity, nrow, max_workspace_bytes=None,
                             padding=2, return_values=False, splat_fn=_splat.splat2d_ref):
    """The op set's splat_composite_grid: per frame t, splat_points(images[t], points[t], ...) then images2grid.
    images (T, N, 3, R, R); points (T, N, P, 2) or None; colors / alpha_channel (N or 1, P, C) or None.
    max_workspace_bytes is accepted for the op's signature (the restatement needs no workspace).
    -> (T, Hg, Wg, 3) uint8 (and, with return_values, the (T, Hg, Wg, 3) values v * 255 + 0.5 before clamp and cast)."""
    t, n = images.shape[:2]
    frames = images
    if points is not None and points.size(2) > 0:
        p = points.size(2)
        flat = images.reshape(t * n, *images.shape[2:])
        col = colors.expand(n, p, 3).repeat(t, 1, 1)
        alpha = None if alpha_channel is None else alpha_channel.expand(n, p, 1).repeat(t, 1, 1)
        pts = points.reshape(t * n, p, 2).float()
        if images.dtype == torch.float64:    # the composite in float64 (splat2d_ref sums in float64, stores float32)
            sig = torch.full((t * n,), float(sigma))
            zeros = torch.zeros(t * n, 1, *images.shape[3:])
            alpha = torch.ones(t * n, p, 1) if alpha is None else alpha
            obj = splat_fn(zeros.repeat(1, 3, 1, 1), pts, col.float(), sig, False).double()
            mask = splat_fn(zeros, pts, alpha.float(), sig, True).double() * opacity
            out = mask * obj + (1 - mask) * flat
        else:
            out = _splat.splat_points_ref(flat, pts, sigma, opacity, col.float(), None if alpha is None else alpha.float(),
                                          splat_fn=splat_fn)
        frames = out.reshape(images.shape)
    grids = [images2grid_ref(f, nrow, padding, return_values) for f in frames]
    if return_values:
        return torch.stack([g[0] for g in grids]), torch.stack([g[1] for g in grids])
    return torch.stack(grids)


def cpu_ops():
    """oracle.vis.cpu_ops() plus `splat_composite_grid`: the op set that runs the label-propagation API
    (gangealing_b200.evaluation.visuals) on the CPU restatement."""
    return types.SimpleNamespace(**vars(_vis.cpu_ops()), splat_composite_grid=splat_composite_grid_ref)
