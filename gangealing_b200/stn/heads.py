"""Warp heads of the Spatial Transformer -- host-side mirror of reference
models/spatial_transformers/warping_heads.py (state-dict compatible: `linear`, `flow_out`, `mask_out`, buffer
`one_hot`), written against the fused sm_90a ops:

  SimilarityHead : regress (rot, scale, tx, ty) -> 2x3 matrix -> affine grid -> fused antialiased warp
  FlowHead       : regress low-res flow + convex-upsampling mask -> ONE flow_compose kernel (upsample, identity
                   add, affine composition, alpha lerp) -> fused antialiased warp
"""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F

from ..opset import cuda_ops
from ..stylegan2.networks import EqualConv2d
from .sampling import MipmapWarp, Warp


def _policy(warp_policy, img, num_heads):
    """Cluster routing shared by both heads (reference warping_heads.py:100-116, :218-233).
    -> (assignments or None).  'cartesian': every image x every head; 'assign_only': one head per image."""
    logits = None
    if isinstance(warp_policy, torch.Tensor):
        logits = warp_policy
    elif isinstance(warp_policy, nn.Module):
        logits = warp_policy(img)
    elif warp_policy != "cartesian":
        raise NotImplementedError
    if logits is None:
        return None
    return logits.max(dim=1).indices % num_heads  # the modulo folds the flipped copies onto their head


def check_if_warp_exceeds_image_boundaries(grid, image_bounds, img_size, split_size, threshold=0.025):
    """Fraction of output pixels sampled outside the (optionally letter-boxed) image > threshold, per sample
    (reference warping_heads.py:280-309)."""
    if image_bounds is None:
        boundary_y, boundary_x = img_size[-2], img_size[-1]
    else:
        image_bounds = image_bounds.repeat_interleave(split_size, dim=0)
        landscape = image_bounds[:, 0] < image_bounds[:, 1]
        full_h = torch.tensor(img_size[-2], dtype=torch.float, device=grid.device)
        full_w = torch.tensor(img_size[-1], dtype=torch.float, device=grid.device)
        boundary_y = torch.where(landscape, img_size[-2] * image_bounds[:, 0] / image_bounds[:, 1], full_h).round()
        boundary_x = torch.where(landscape, full_w, img_size[-1] * image_bounds[:, 1] / image_bounds[:, 0]).round()
    oob_x = grid[..., 0].flatten(1).abs().gt((boundary_x - 1) / img_size[-1]).float().mean(dim=1).gt(threshold)
    oob_y = grid[..., 1].flatten(1).abs().gt((boundary_y - 1) / img_size[-2]).float().mean(dim=1).gt(threshold)
    return torch.logical_or(oob_y, oob_x)


class SimilarityHead(nn.Module):
    """Regresses and applies a similarity warp (rotation, isotropic scale, x/y shift) per head."""

    def __init__(self, in_shape, antialias=True, num_heads=1, ops=None, **kwargs):
        super().__init__()
        self.num_warp_params = 4
        self.linear = nn.Linear(in_shape, self.num_warp_params * num_heads, bias=True)
        nn.init.zeros_(self.linear.bias)   # identity transform at initialisation
        nn.init.zeros_(self.linear.weight)
        self.warper = MipmapWarp(max_num_levels=3.5, ops=ops) if antialias else Warp(ops=ops)
        self.num_heads = num_heads
        self.register_buffer("one_hot", torch.tensor([0, 0, 1], dtype=torch.float).view(1, 1, 1, 3))
        self.ops = ops if ops is not None else cuda_ops()

    @staticmethod
    def make_affine_matrix(rot, scale, shift_x, shift_y):
        """(N, K) raw parameters -> (N, K, 2, 3): rot = tanh(.)*pi, scale = exp(.)."""
        n, k = rot.size()
        rot = torch.tanh(rot) * math.pi
        scale = torch.exp(scale)
        c, s = scale * torch.cos(rot), scale * torch.sin(rot)
        return torch.stack([c, -s, shift_x, s, c, shift_y], dim=2).reshape(n, k, 2, 3)

    def make_3x3(self, M):
        return torch.cat([M, self.one_hot.expand(M.size(0), M.size(1), 1, 3)], 2)

    def forward(self, img, features, output_resolution=None, alpha=None, base_warp=None, stop_grad=False,
                padding_mode="border", return_out_of_bounds=False, image_bounds=None, warp_policy="cartesian",
                unfold=False):
        n = features.size(0)
        params = self.linear(features)
        assignments = _policy(warp_policy, img, self.num_heads)
        if assignments is not None:  # one head per image
            params = params.reshape(-1, self.num_warp_params, self.num_heads).permute(0, 2, 1)
            params = params.gather(1, assignments.view(n, 1, 1).repeat(1, 1, self.num_warp_params)).squeeze(1)
            split = 1
        else:
            split = self.num_heads
        matrix = self.make_affine_matrix(*torch.split(params, split, dim=1))  # (N, split, 2, 3)
        if base_warp is not None:
            if base_warp.dim() == 3:
                base_warp = base_warp.unsqueeze(1)
            matrix = base_warp @ self.make_3x3(matrix)
        if alpha is not None:
            eye = torch.eye(2, 3, device=matrix.device)[None, None]
            matrix = eye.lerp(matrix, alpha[:, None, None, None])
        res = (img.size(2), img.size(3)) if output_resolution is None else (output_resolution, output_resolution)
        img_size = torch.Size([img.size(0) * split, img.size(1), res[0], res[1]])
        if stop_grad:
            matrix = matrix.detach() + 0 * matrix  # keeps every parameter in the autograd graph for DDP
        matrix = matrix.reshape(n * split, 2, 3)
        if split > 1:
            img = img.repeat_interleave(split, dim=0)
        fused = getattr(self.ops, "stn_sample_affine", None)
        if fused is not None and img.is_cuda:
            # one pass: the affine sampling grid is generated inside the (antialiased) sampler and returned as a by-product
            mip = isinstance(self.warper, MipmapWarp)
            out, grid, levels = fused(img, matrix, (img_size[2], img_size[3]), self.warper.max_num_levels if mip else None,
                                      0.0, padding_mode)
            if mip:
                self.warper._levels = levels
        else:
            grid = F.affine_grid(matrix, img_size, align_corners=False)
            out = self.warper(img, grid, padding_mode=padding_mode)
        oob = check_if_warp_exceeds_image_boundaries(grid, image_bounds, img_size, split) if return_out_of_bounds else None
        if unfold:
            out = out.reshape(n, -1, img_size[1], img_size[2], img_size[3])
            matrix = matrix.reshape(n, -1, 2, 3)
            grid = grid.reshape(n, -1, img_size[2], img_size[3], 2)
        return out, grid, matrix, oob


def resize_grid(flow, output_resolution):
    """The sampling grid at output_resolution: resizing the grid beats resizing pixels (scale 1 is the identity)."""
    if output_resolution == flow.size(2):
        return flow
    return F.interpolate(flow.permute(0, 3, 1, 2), scale_factor=output_resolution / flow.size(2),
                         mode="bilinear").permute(0, 2, 3, 1)


class FlowHead(nn.Module):
    """Regresses a dense sampling grid: low-res residual flow + RAFT-style convex upsampling mask."""

    def __init__(self, in_shape, antialias=True, num_heads=1, flow_downsample=8, ops=None, **kwargs):
        super().__init__()
        self.flow_downsample = flow_downsample
        # the reference keeps this as a plain .cuda() attribute (warping_heads.py:158); a non-persistent buffer
        # follows .to(device) and stays out of the state dict just the same
        self.register_buffer("identity_flow", self.initialize_flow(in_shape), persistent=False)
        c = in_shape[1]
        self.flow_out = nn.Sequential(EqualConv2d(c, c, 3, padding=1, ops=ops), nn.ReLU(),
                                      EqualConv2d(c, num_heads * 2, 3, padding=1, ops=ops))
        nn.init.zeros_(self.flow_out[-1].weight)  # identity transformation at initialisation
        nn.init.zeros_(self.flow_out[-1].bias)
        self.mask_out = nn.Sequential(EqualConv2d(c, c, 3, padding=1, ops=ops), nn.ReLU(),
                                      EqualConv2d(c, num_heads * 9 * flow_downsample * flow_downsample, 3, padding=1, ops=ops))
        self.warper = MipmapWarp(max_num_levels=3.5, ops=ops) if antialias else Warp(ops=ops)
        self.num_heads = num_heads
        self.ops = ops if ops is not None else cuda_ops()

    def initialize_flow(self, in_shape):
        n, c, h, w = in_shape
        return F.affine_grid(torch.eye(2, 3).unsqueeze(0), (n, c, self.flow_downsample * h, self.flow_downsample * w),
                             align_corners=False)

    def upsample_flow(self, flow, mask):
        """[H/s, W/s, 2] -> [H, W, 2] by convex combination (RAFT)."""
        return self._compose(flow, mask, None, None)[0]

    def _compose(self, low, mask, base_warp, alpha):
        return self.ops.flow_compose(low, mask, self.identity_flow, base_warp, alpha, self.flow_downsample)

    def compute_flow(self, features):
        flow = self.flow_out(features)
        n, _, h, w = flow.size()
        flow = flow.reshape(n, self.num_heads, 2, h, w).permute(0, 1, 3, 4, 2)  # (N, K, H, W, 2)
        mask = self.mask_out(features).reshape(n, self.num_heads, 9 * self.flow_downsample ** 2, h, w)
        return flow, mask

    def forward(self, img, features, output_resolution=None, alpha=None, base_warp=None, stop_grad=False,
                padding_mode="border", return_out_of_bounds=False, image_bounds=None, warp_policy="cartesian",
                unfold=False):
        low, mask = self.compute_flow(features)
        n, _, h, w, _ = low.size()
        if isinstance(warp_policy, torch.Tensor):
            assignments = warp_policy.max(dim=1).indices % self.num_heads
            pick = torch.arange(n, device=low.device)   # on the device: indexing with a CPU tensor is a pageable H2D copy (not capturable)
            low, mask = low[pick, assignments], mask[pick, assignments]
            split = 1
        elif warp_policy == "cartesian":
            split = self.num_heads
        else:
            raise NotImplementedError
        low = low.reshape(n * split, h, w, 2)
        mask = mask.reshape(n * split, -1, h, w)
        if base_warp is not None and base_warp.dim() == 4:
            base_warp = base_warp.reshape(-1, 2, 3)
        fused = getattr(self.ops, "stn_sample_flow", None)
        s_ = self.flow_downsample
        one_pass = (fused is not None and img.is_cuda and not stop_grad
                    and (output_resolution is None or output_resolution == s_ * h) and h == w)
        if one_pass:
            # ONE pass: convex up-sampling + identity + affine + alpha generated inside the antialiased sampler
            if split > 1:
                img = img.repeat_interleave(split, dim=0)
            mip = isinstance(self.warper, MipmapWarp)
            out, flow, delta_flow, levels = fused(img, low, mask, self.identity_flow, base_warp, alpha, s_,
                                                  self.warper.max_num_levels if mip else None, 0.0, padding_mode)
            if mip:
                self.warper._levels = levels
            img_size = torch.Size([img.size(0), img.size(1), flow.size(1), flow.size(2)])
            oob = check_if_warp_exceeds_image_boundaries(flow, image_bounds, img_size, split) if return_out_of_bounds else None
            if unfold:
                k = self.num_heads
                out = out.reshape(out.size(0) // k, k, out.size(1), out.size(2), out.size(3))
                flow = flow.reshape(flow.size(0) // k, k, out.size(3), out.size(4), 2)
                delta_flow = delta_flow.reshape(delta_flow.size(0) // k, k, s_ * h, s_ * w, 2)
            return out, flow, delta_flow, oob
        delta_flow, flow = self._compose(low, mask, base_warp, alpha)
        if output_resolution is None:
            img_size = torch.Size([img.size(0) * split, flow.size(1), flow.size(2)])
        else:
            img_size = torch.Size([img.size(0) * split, img.size(1), output_resolution, output_resolution])
            flow = resize_grid(flow, output_resolution)
        if stop_grad:
            flow = flow.detach() + 0 * flow
        if split > 1:
            img = img.repeat_interleave(split, dim=0)
        out = self.warper(img, flow, padding_mode=padding_mode)
        oob = check_if_warp_exceeds_image_boundaries(flow, image_bounds, img_size, split) if return_out_of_bounds else None
        if unfold:
            k = self.num_heads
            out = out.reshape(out.size(0) // k, k, out.size(1), out.size(2), out.size(3))
            flow = flow.reshape(flow.size(0) // k, k, out.size(3), out.size(4), 2)
            s = self.flow_downsample
            delta_flow = delta_flow.reshape(delta_flow.size(0) // k, k, s * h, s * w, 2)
        return out, flow, delta_flow, oob
