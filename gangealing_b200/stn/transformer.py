"""SpatialTransformer / ComposedSTN / get_stn -- host-side mirror of reference
models/spatial_transformers/spatial_transformer.py (same module tree, argument names and return conventions,
so checkpoints and call sites carry over), running on the fused sm_90a ops of this package.
"""
import math

import torch
import torch.nn as nn

from ..opset import cuda_ops
from ..splat2d.blend import BLEND_PRESETS
from ..stylegan2.networks import ConvLayer, EqualLinear, ResBlock, channel_table
from .heads import FlowHead, SimilarityHead, resize_grid
from .sampling import BilinearDownsample


class _TVLoss(torch.autograd.Function):
    """total_variation_loss(reduce_batch=True) as one reduction kernel per direction (csrc/optim.cu)."""

    @staticmethod
    def forward(ctx, flow):
        from .. import _lib
        f = flow.detach()
        if f.dtype != torch.float32 or not f.is_contiguous():
            f = f.float().contiguous()
        n, h, w, _ = f.shape
        lib = _lib.load()
        out = torch.empty(1, dtype=torch.float32, device=f.device)
        ws = torch.empty(max(1, lib.gg_tv_loss_workspace(n, h, w) // 4), dtype=torch.float32, device=f.device)
        _lib.check(lib.gg_tv_loss_forward(out.data_ptr(), ws.data_ptr(), f.data_ptr(), n, h, w, _lib.stream()), "gg_tv_loss_forward")
        ctx.save_for_backward(f)
        ctx.dtype = flow.dtype
        return out.reshape(())

    @staticmethod
    def backward(ctx, g):
        from .. import _lib
        (f,) = ctx.saved_tensors
        n, h, w, _ = f.shape
        go = g.detach().float().reshape(1).contiguous()
        grad = torch.empty_like(f)
        _lib.check(_lib.load().gg_tv_loss_backward(grad.data_ptr(), go.data_ptr(), f.data_ptr(), n, h, w, _lib.stream()),
                   "gg_tv_loss_backward")
        return grad.to(ctx.dtype)


def total_variation_loss(delta_flow, reduce_batch=True):
    """Huber-penalised finite differences of a (N, H, W, 2) residual flow (reference models/losses/loss.py:4-12).
    On CUDA the batch-reduced form (the training loss) is one fused reduction kernel forward and one gather kernel backward;
    the per-sample form (forward_with_flip's tie-break) and CPU tensors (the oracle's legs) use the tensor formulation."""
    dims = (0, 1, 2, 3) if reduce_batch else (1, 2, 3)
    assert delta_flow.size(-1) == 2
    if reduce_batch and delta_flow.is_cuda and delta_flow.dim() == 4 and delta_flow.size(1) > 1 and delta_flow.size(2) > 1:
        return _TVLoss.apply(delta_flow)

    def huber(a):
        return torch.where(a <= 1.0, 0.5 * a.pow(2), a - 0.5).mean(dim=dims)

    dy = huber((delta_flow[:, :-1] - delta_flow[:, 1:]).abs())
    dx = huber((delta_flow[:, :, :-1] - delta_flow[:, :, 1:]).abs())
    return dx + dy


def get_stn(transforms, **stn_kwargs):
    if isinstance(transforms, str):
        transforms = [transforms]
    assert isinstance(transforms, list)
    if len(transforms) == 1:
        return SpatialTransformer(transform=transforms[0], **stn_kwargs)
    return ComposedSTN(transforms, **stn_kwargs)


def unravel_index(indices, shape):
    coord = []
    for dim in reversed(shape):
        coord.append(indices % dim)
        indices = indices // dim
    return torch.stack(coord, dim=-1)


def match_pick(tv):
    """match_flows' choice (reference spatial_transformer.py:269-278) from the per-sample smoothness of the 4N batch
    [A, B, flip(A), flip(B)]: 0 = neither flipped, 1 = A flipped, 2 = B flipped, 3 = both.  -> (N, 1, 1, 1) int64."""
    tvA, tvB, tvAf, tvBf = tv.chunk(4, dim=0)
    return torch.stack([tvA + tvB, tvAf + tvB, tvA + tvBf, tvAf + tvBf], 0).argmin(dim=0).view(tvA.size(0), 1, 1, 1)


def flip_key_points(pick, pointsA, pointsB, permutation, size):
    """match_flows' key-point update (reference spatial_transformer.py:282-292) for images of width `size`: mirror x where
    an image was flipped and relabel with `permutation`.  The reference's quirk is kept: when pointsB is given, the second
    relabelling permutes pointsA again (where B was flipped) and never touches pointsB.  -> (pointsA, pointsB or None)."""
    keepA = (pick % 2 == 0).view(pick.size(0), 1)
    pointsA = pointsA.clone()
    pointsA[:, :, 0] = torch.where(keepA, pointsA[:, :, 0], size - 1 - pointsA[:, :, 0])
    if permutation is not None:
        pointsA = torch.where(keepA.view(pick.size(0), 1, 1), pointsA, pointsA[:, permutation])
    if pointsB is None:
        return pointsA, None
    keepB = (pick <= 1).view(pick.size(0), 1)
    pointsB = pointsB.clone()
    pointsB[:, :, 0] = torch.where(keepB, pointsB[:, :, 0], size - 1 - pointsB[:, :, 0])
    if permutation is not None:
        pointsA = torch.where(keepB.view(pick.size(0), 1, 1), pointsA, pointsA[:, permutation])
    return pointsA, pointsB


def _pack(values, flags):
    out = [values[0]] + [v for v, f in zip(values[1:], flags) if f]
    return out[0] if len(out) == 1 else out


_IGNORED_KEYS = ("warp_head.one_hot", "warp_head.rebias", "input_downsample.kernel_horz", "input_downsample.kernel_vert")


class SpatialTransformer(nn.Module):
    """image -> conv trunk at (flow_size x flow_size) -> warp head -> warped image (reference :388-726)."""

    def __init__(self, flow_size, supersize, channel_multiplier=0.5, blur_kernel=[1, 3, 3, 1], num_heads=1,
                 transform="similarity", flow_downsample=8, ops=None):
        super().__init__()
        self.ops = ops if ops is not None else cuda_ops()
        if supersize > flow_size:
            self.input_downsample = BilinearDownsample(supersize // flow_size, 3, ops=ops)
        self.input_downsample_required = supersize > flow_size
        self.stn_in_size = flow_size
        self.is_flow = transform == "flow"
        self.channels_last = False        # run the conv trunk on NHWC activations (cuDNN's native layout; CUDA only)
        self.act_dtype = torch.float32    # storage type of the trunk's activations (bf16: BASELINE config 3); the warp
        #                                   heads, the sampling grid and the warped image always stay fp32
        channels = channel_table(channel_multiplier)
        convs = [ConvLayer(3, int(channels[flow_size]), 1, ops=ops)]
        log_size = int(math.log(flow_size, 2))
        log_down = int(math.log(flow_downsample, 2))
        in_channel = channels[flow_size]
        end_log = log_size - 4 if self.is_flow else 2
        assert end_log >= 0
        n_down = 0
        for i in range(log_size, end_log, -1):
            down = (not self.is_flow) or (n_down < log_down)
            n_down += down
            out_channel = channels[2 ** (i - 1)]
            convs.append(ResBlock(int(in_channel), int(out_channel), blur_kernel, down, ops=ops))
            in_channel = out_channel
        self.convs = nn.Sequential(*convs)
        self.final_conv = ConvLayer(int(in_channel), channels[4], 3, ops=ops)
        if not self.is_flow:
            self.final_linear = EqualLinear(channels[4] * 4 * 4, channels[4], activation="fused_lrelu", ops=ops)
        if transform == "similarity":
            self.warp_head = SimilarityHead(channels[4], antialias=True, num_heads=num_heads,
                                            flow_downsample=flow_downsample, ops=ops)
        elif transform == "flow":
            shape = (1, int(in_channel), flow_size // flow_downsample, flow_size // flow_downsample)
            self.warp_head = FlowHead(shape, antialias=True, num_heads=num_heads, flow_downsample=flow_downsample, ops=ops)
        else:
            raise NotImplementedError

    @property
    def identity_flow(self):
        return self.warp_head.identity_flow

    # -------------------------------------------------------------------------------------------- forward
    def forward(self, input_img, output_resolution=None, iters=1, return_warp=False, return_flow=False,
                return_intermediates=False, return_out_of_bounds=False, intermediate_output_resolution=None,
                stop_grad=False, alpha=None, padding_mode="border", input_img_for_sampling=None, image_bounds=None,
                warp_policy="cartesian", unfold=False, base_warp=None):
        common = dict(stop_grad=stop_grad, padding_mode=padding_mode, input_img_for_sampling=input_img_for_sampling,
                      image_bounds=image_bounds, warp_policy=warp_policy, base_warp=base_warp)
        if iters == 1:
            return self.single_forward(input_img, output_resolution=output_resolution, return_warp=return_warp,
                                       return_flow=return_flow, alpha=alpha, unfold=unfold,
                                       return_out_of_bounds=return_out_of_bounds, **common)
        return self.iterated_forward(input_img, output_resolution=output_resolution, iters=iters, return_warp=return_warp,
                                     return_flow=return_flow, return_intermediates=return_intermediates,
                                     intermediate_output_resolution=intermediate_output_resolution, alpha=alpha,
                                     unfold=unfold, return_out_of_bounds=return_out_of_bounds, **common)

    def iterated_forward(self, input_img, output_resolution=None, iters=1, return_warp=False, return_flow=False,
                         return_intermediates=False, intermediate_output_resolution=None, stop_grad=False, alpha=None,
                         padding_mode="border", input_img_for_sampling=None, return_out_of_bounds=False,
                         image_bounds=None, warp_policy="cartesian", unfold=False, base_warp=None):
        """Feed the STN its own output `iters` times, composing the similarity warps (reference :523-567)."""
        assert not self.is_flow, "iterated_forward is currently only supported for similarity STNs"
        out = input_img
        source = input_img if input_img_for_sampling is None else input_img_for_sampling
        mid_res = self.stn_in_size if intermediate_output_resolution is None else intermediate_output_resolution
        M = base_warp
        outs, mats, oob_final = [], [], None
        for it in range(iters):
            last = it == iters - 1
            out, grid, M, oob = self.single_forward(
                out, output_resolution=output_resolution if last else mid_res, return_warp=True, return_flow=True,
                return_out_of_bounds=return_out_of_bounds and last, base_warp=M, input_img_for_sampling=source,
                stop_grad=stop_grad, alpha=alpha if last else None, padding_mode=padding_mode, image_bounds=image_bounds,
                warp_policy=warp_policy, unfold=unfold and last, pack=True)
            if return_out_of_bounds and last:
                oob_final = oob
            outs.append(out)
            mats.append(M)
        if return_intermediates:
            return outs, mats
        return _pack([out, grid, M, oob_final], [return_warp, return_flow, return_out_of_bounds])

    def single_forward(self, input_img, output_resolution=None, return_warp=False, return_flow=False,
                       return_out_of_bounds=False, base_warp=None, input_img_for_sampling=None, stop_grad=False,
                       alpha=None, padding_mode="border", image_bounds=None, warp_policy="cartesian", unfold=False,
                       pack=False):
        regression_input = self.input_downsample(input_img) if input_img.size(-1) > self.stn_in_size else input_img
        source = input_img if input_img_for_sampling is None else input_img_for_sampling
        if self.channels_last and regression_input.is_cuda:
            regression_input = regression_input.to(self.act_dtype).contiguous(memory_format=torch.channels_last)
        feat = self.final_conv(self.convs(regression_input))
        if feat.dtype != torch.float32:   # grid coordinates need more than 8 bits of mantissa: heads run in fp32
            feat = feat.float()
        if not self.is_flow:
            feat = self.final_linear(feat.reshape(feat.shape[0], -1))   # logical (C, H, W) order in either layout
        res = output_resolution if output_resolution is not None else self.stn_in_size
        out, grid, M, oob = self.warp_head(source, feat, output_resolution=res, base_warp=base_warp, stop_grad=stop_grad,
                                           alpha=alpha, padding_mode=padding_mode,
                                           return_out_of_bounds=return_out_of_bounds, image_bounds=image_bounds,
                                           warp_policy=warp_policy, unfold=unfold)
        if pack:
            return [out, grid, M, oob]
        return _pack([out, grid, M, oob], [return_warp, return_flow, return_out_of_bounds])

    # -------------------------------------------------------------------------------------------- point transfer
    @staticmethod
    def normalize(points, res, out_res):
        return points.div(out_res - 1).add(-0.5).mul(2).mul((res - 1) / res)

    @staticmethod
    def unnormalize(points, res, out_res):
        return points.div((res - 1) / res).div(2).add(0.5).mul(out_res - 1)

    @staticmethod
    def convert(points, current_res, target_res):
        points = SpatialTransformer.normalize(points, target_res, current_res)
        return SpatialTransformer.unnormalize(points, target_res, target_res)

    def _lookup(self, grid, points):
        """Sample the sampling grid itself at query points (bilinear, border): (N, H, W, 2) x (N, P, 2) -> (N, P, 2)."""
        sampled = self.ops.grid_sample(grid.permute(0, 3, 1, 2).contiguous(), points.unsqueeze(2).float().contiguous(), "border")
        return sampled.squeeze(3).permute(0, 2, 1)

    def congeal_points(self, imgA, pointsA, normalize_input_points=True, unnormalize_output_points=False,
                       output_resolution=None, iters=1, input_img_for_sampling=None, return_full=False,
                       **stn_forward_kwargs):
        """Map key points of imgA into the congealed frame (reference :631-672)."""
        assert imgA.size(0) == pointsA.size(0)
        n, num_points = imgA.size(0), pointsA.size(1)
        source_res = imgA.size(-1) if input_img_for_sampling is None else input_img_for_sampling.size(-1)
        outA, gridA, fmA = self.forward(imgA, return_warp=True, return_flow=True, output_resolution=output_resolution,
                                        input_img_for_sampling=input_img_for_sampling, iters=iters, **stn_forward_kwargs)
        if normalize_input_points:
            pointsA = self.normalize(pointsA, source_res, source_res)
        if not self.is_flow:  # closed form: invert the similarity
            hom = torch.cat([pointsA, torch.ones(n, num_points, 1, device=pointsA.device)], 2)
            last = torch.tensor([[[0, 0, 1]]], dtype=torch.float, device=fmA.device).repeat(n, 1, 1)
            inv = torch.inverse(torch.cat([fmA, last], 1)).permute(0, 2, 1)
            congealed = (hom @ inv)[..., [0, 1]]
            if unnormalize_output_points:
                congealed = self.unnormalize(congealed, source_res, source_res)
        else:  # brute-force nearest neighbour on the reverse sampling grid
            assert fmA.size(-1) == 2
            g = fmA + self.identity_flow                                   # (N, H, W, 2)
            fused = getattr(self.ops, "nn_argmin", None)
            if fused is not None and g.is_cuda:
                # tiled argmin kernel (csrc/points.cu): same expanded distance and first-minimum rule, no (N, H, W, P) tensor
                nearest = fused(g, pointsA)
            else:
                gg_ = g.reshape(n, fmA.size(1), fmA.size(2), 1, 1, 2)
                pts = pointsA.reshape(n, 1, 1, num_points, 2, 1)
                sim = (gg_ @ pts)[..., 0, 0]
                dist = pts.pow(2).squeeze(-1).sum(dim=-1) + gg_.pow(2).sum(dim=-1).squeeze(-1) - 2 * sim
                nearest = dist.reshape(n, g.size(1) * g.size(2), num_points).argmin(dim=1)
            congealed = unravel_index(nearest, (g.size(1), g.size(2)))
        if return_full:
            return outA, fmA, congealed
        return congealed

    def uncongeal_points(self, imgB, points_congealed, unnormalize_output_points=True, normalize_input_points=False,
                         output_resolution=None, iters=1, input_img_for_sampling=None, **stn_forward_kwargs):
        """Map key points of the congealed frame into imgB (reference :674-712)."""
        assert imgB.size(0) == points_congealed.size(0)
        n, num_points = imgB.size(0), points_congealed.size(1)
        source_res = imgB.size(-1) if input_img_for_sampling is None else input_img_for_sampling.size(-1)
        outB, gridB, fmB = self.forward(imgB, return_warp=True, return_flow=True, output_resolution=output_resolution,
                                        iters=iters, input_img_for_sampling=input_img_for_sampling, **stn_forward_kwargs)
        if normalize_input_points:
            points_congealed = self.normalize(points_congealed, source_res, imgB.size(-1))
        if not self.is_flow:
            last = torch.tensor([[[0, 0, 1]]], dtype=torch.float, device=fmB.device).repeat(n, 1, 1)
            hom = torch.cat([points_congealed, torch.ones(n, num_points, 1, device=points_congealed.device)], 2)
            pointsB = (hom @ torch.cat([fmB, last], 1).permute(0, 2, 1))[..., [0, 1]]
        else:
            assert gridB.size(-1) == 2
            pointsB = self._lookup(gridB, points_congealed)
        if unnormalize_output_points:
            pointsB = self.unnormalize(pointsB, imgB.size(-1), source_res)
        return pointsB

    def transfer_points(self, imgA, imgB, pointsA, output_resolution=None, iters=1, **stn_forward_kwargs):
        congealed = self.congeal_points(imgA, pointsA, output_resolution=output_resolution, iters=iters, **stn_forward_kwargs)
        return self.uncongeal_points(imgB, congealed, output_resolution=output_resolution, normalize_input_points=False,
                                     iters=iters, **stn_forward_kwargs)

    def load_state_dict(self, state_dict, strict=True):
        return super().load_state_dict({k: v for k, v in state_dict.items() if k not in _IGNORED_KEYS}, False)


class ComposedSTN(nn.Module):
    """Chain of STNs whose warps compose (similarity -> flow is the tested configuration; reference :47-385)."""

    def __init__(self, transforms, **stn_kwargs):
        super().__init__()
        self.stns = nn.ModuleList([SpatialTransformer(transform=t, **stn_kwargs) for t in transforms])
        if transforms != ["similarity", "flow"]:
            print('WARNING: ComposedSTN is only tested for transforms=["similarity", "flow"].')
        self.transforms = transforms[:]
        self.stn_in_size = stn_kwargs["flow_size"]
        self.N_minus_1 = len(self.stns) - 1
        self.is_flow = "flow" in transforms
        self.num_heads = self.stns[0].warp_head.num_heads
        if self.num_heads > 1:
            self.cluster_assignments = torch.eye(self.num_heads)
        self.ops = stn_kwargs.get("ops") or cuda_ops()

    @property
    def identity_flow(self):
        return self.stns[self.transforms.index("flow")].identity_flow

    def forward(self, input_img, return_warp=None, return_flow=False, return_sim=False, return_intermediates=False,
                output_resolution=None, unfold=False, iters=1, alpha=None, warp_policy="cartesian",
                input_img_for_sampling=None, **stn_forward_kwargs):
        out = input_img
        source = input_img if input_img_for_sampling is None else input_img_for_sampling
        warp = None  # identity
        imgs, warps = [], []
        n = source.size(0)
        sim_out = grid = flow_or_matrix = None
        for i, stn in enumerate(self.stns):
            last = i == self.N_minus_1
            if self.num_heads > 1 and warp_policy == "cartesian" and i > 0:
                # reference :109 copies the (K, K) identity host -> device on every call; memoised per device here so that the
                # step stays CUDA-graph capturable (a pageable H2D copy is illegal during capture)
                eye = getattr(self, "_cluster_assignments_dev", None)
                if eye is None or eye.device != source.device:
                    eye = self._cluster_assignments_dev = self.cluster_assignments.to(source.device)
                policy = eye.repeat(n, 1)
            else:
                policy = warp_policy
            out, grid, flow_or_matrix = stn(
                out, return_warp=True, return_flow=True, return_intermediates=False, input_img_for_sampling=source,
                base_warp=warp, output_resolution=output_resolution if last else self.stn_in_size,
                unfold=unfold if last else False, iters=iters if i == 0 else 1, alpha=alpha if last else None,
                warp_policy=policy, **stn_forward_kwargs)
            if self.num_heads > 1 and warp_policy == "cartesian" and i == 0:
                source = source.repeat_interleave(self.num_heads, dim=0)
            imgs.append(out)
            warps.append(grid)
            if i == 0:
                sim_out = out
            warp = flow_or_matrix
        if return_intermediates:
            return imgs, warps
        return _pack([out, grid, flow_or_matrix, sim_out], [return_warp, return_flow, return_sim])

    def uncongeal_points(self, imgB, points_congealed, output_resolution=None, iters=1, unnormalize_output_points=True,
                         normalize_input_points=False, return_congealed_img=False, **stn_forward_kwargs):
        assert imgB.size(0) == points_congealed.size(0)
        if normalize_input_points:
            points_congealed = SpatialTransformer.normalize(points_congealed, imgB.size(-1), self.stn_in_size)
        congealed_img, gridB = self.forward(imgB, return_warp=True, output_resolution=output_resolution, iters=iters,
                                            **stn_forward_kwargs)
        pointsB = self.stns[0]._lookup(gridB, points_congealed)
        if unnormalize_output_points:
            pointsB = SpatialTransformer.unnormalize(pointsB, imgB.size(-1), imgB.size(-1))
        return (pointsB, congealed_img) if return_congealed_img else pointsB

    def uncongeal_and_splat(self, imgB, points_congealed, colors, sigma, opacity, alpha_channel=None, output_resolution=None,
                            iters=1, normalize_input_points=False, blend_alg="alpha", **stn_forward_kwargs):
        """`uncongeal_points(imgB, points)` followed by `splat_points(imgB, points, sigma, opacity, colors=...,
        blend_alg=...)` (reference applications/propagate_to_images.py:44-78 + utils/vis_tools/helpers.py:134-194) with the
        grid lookup fused into the first splat's point load (csrc/splat.cu LOOKUP).  blend_alg: 'alpha' (alpha compositing),
        'laplacian' or 'laplacian_light' (the op set's laplacian_blend with splat_points' presets).
        -> (propagated images, points (N, P, 2) in pixels)."""
        if blend_alg != "alpha" and blend_alg not in BLEND_PRESETS:
            raise ValueError("blend_alg must be 'alpha', 'laplacian' or 'laplacian_light' (got %r)" % (blend_alg,))
        assert imgB.size(0) == points_congealed.size(0)
        if normalize_input_points:
            points_congealed = SpatialTransformer.normalize(points_congealed, imgB.size(-1), self.stn_in_size)
        _, gridB = self.forward(imgB, return_warp=True, output_resolution=output_resolution, iters=iters, **stn_forward_kwargs)
        n, _, h, w = imgB.shape
        res = imgB.size(-1)
        sig = torch.full((n,), float(sigma), device=imgB.device) if not torch.is_tensor(sigma) else sigma
        if alpha_channel is None:
            alpha_channel = torch.ones(n, points_congealed.size(1), 1, device=imgB.device)
        fused = getattr(self.ops, "splat2d_lookup", None)
        blank_img = torch.zeros(n, colors.shape[-1], h, w, device=imgB.device)
        blank_mask = torch.zeros(n, 1, h, w, device=imgB.device)
        if fused is not None and imgB.is_cuda and colors.shape[-1] <= 3:
            prop_obj, pointsB = fused(blank_img, gridB, points_congealed, colors, sig, res, res, False)
        else:
            pointsB = SpatialTransformer.unnormalize(self.stns[0]._lookup(gridB, points_congealed), res, res)
            prop_obj = self.ops.splat2d(blank_img, pointsB, colors, sig, False)
        prop_mask = self.ops.splat2d(blank_mask, pointsB, alpha_channel, sig, True) * opacity
        if blend_alg != "alpha":
            kw = BLEND_PRESETS[blend_alg]
            prop_obj, prop_mask = prop_obj.to(imgB.device), prop_mask.to(imgB.device)
            return self.ops.laplacian_blend(imgB, prop_obj, prop_mask, kw["levels"], kw["gaussian_kernel_size"],
                                            kw["gaussian_sigma"]), pointsB
        return prop_mask * prop_obj + (1 - prop_mask) * imgB, pointsB

    def congeal_points(self, imgA, pointsA, output_resolution=None, iters=1, normalize_input_points=True,
                       unnormalize_output_points=False, return_full=False, **stn_forward_kwargs):
        assert imgA.size(0) == pointsA.size(0)
        outA, warpA, pts = imgA, None, pointsA
        for i, stn in enumerate(self.stns):
            last = i == self.N_minus_1
            outA, warpA, pts = stn.congeal_points(
                outA, pts, normalize_input_points=normalize_input_points if i == 0 else True,
                unnormalize_output_points=unnormalize_output_points if last else True, iters=iters if i == 0 else 1,
                output_resolution=output_resolution if last else self.stn_in_size, base_warp=warpA,
                input_img_for_sampling=imgA, return_full=True, **stn_forward_kwargs)
        return (outA, warpA, pts) if return_full else pts

    def transfer_points(self, imgA, imgB, pointsA, output_resolution=None, iters=1, congeal_kwargs={},
                        uncongeal_kwargs={}, **stn_forward_kwargs):
        assert imgA.size(0) == imgB.size(0) == pointsA.size(0)
        congealed = self.congeal_points(imgA, pointsA, output_resolution=output_resolution, normalize_input_points=True,
                                        iters=iters, **congeal_kwargs, **stn_forward_kwargs)
        return self.uncongeal_points(imgB, congealed, output_resolution=output_resolution, normalize_input_points=True,
                                     unnormalize_output_points=True, iters=iters, **uncongeal_kwargs, **stn_forward_kwargs)

    def forward_with_flip(self, input_img, return_flow=False, return_warp=False, return_inputs=False,
                          return_flip_indices=False, **stn_forward_kwargs):
        """Run the image and its mirror; keep, per sample, whichever yields the smoother flow (reference :200-240)."""
        congealed, warp, flow = self.forward(input_img, return_warp=True, return_flow=True, **stn_forward_kwargs)
        mirrored = input_img.flip(3,)
        congealedF, warpF, flowF = self.forward(mirrored, return_warp=True, return_flow=True, **stn_forward_kwargs)
        tv = torch.stack([total_variation_loss(flow, reduce_batch=False), total_variation_loss(flowF, reduce_batch=False)], 0)
        use_flip = tv.argmin(dim=0).view(input_img.size(0), 1, 1, 1).bool()
        out = [torch.where(use_flip, congealedF, congealed)]
        if return_warp:
            warpF = warpF.clone()
            warpF[:, :, :, 0] = -warpF[:, :, :, 0]
            out.append(torch.where(use_flip, warpF, warp))
        if return_flow:
            out.append(torch.where(use_flip, flowF, flow))
        if return_inputs:
            out.append(torch.where(use_flip, mirrored, input_img))
        if return_flip_indices:
            out.append(use_flip)
        return out[0] if len(out) == 1 else out

    def match_flows(self, imgA, imgB, pointsA, pointsB=None, permutation=None, **stn_forward_kwargs):
        """Flip neither, one or both images of each pair so that their residual flows are smoothest; update the key points
        to follow (reference :242-295, quirks in flip_key_points).  ONE STN forward over [A, B, flip(A), flip(B)] and one
        per-sample smoothness (the op set's tv_per_sample).
        -> (imgA, imgB, pointsA, [pointsB,] pick) with pick (N, 1, 1, 1) in {0: none, 1: A, 2: B, 3: both flipped}."""
        imgA_flip, imgB_flip = imgA.flip(3,), imgB.flip(3,)
        _, flows = self.forward(torch.cat([imgA, imgB, imgA_flip, imgB_flip], 0), return_flow=True, **stn_forward_kwargs)
        pick = match_pick(self.ops.tv_per_sample(flows))
        imgA = torch.where(pick % 2 == 0, imgA, imgA_flip)
        imgB = torch.where(pick <= 1, imgB, imgB_flip)
        pointsA, pointsB_out = flip_key_points(pick, pointsA, pointsB, permutation, imgA.size(-1))
        if pointsB is not None:
            return imgA, imgB, pointsA, pointsB_out, pick
        return imgA, imgB, pointsA, pick

    def congeal_and_grid(self, input_img, infer_flip=True, output_resolution=None, iters=1, padding_mode="border",
                         warp_policy="cartesian"):
        """Everything propagate_to_images reads from the STN (reference applications/propagate_to_images.py:44-78, which
        runs it on 4N images: determine_flips' forward_with_flip (2N), t(reals_flipped) (N) and uncongeal_points (N)), from
        ONE forward.  infer_flip: the forward runs over cat([x, flip(x)]) (2N images) and each image keeps the variant
        with the smoother residual flow, by the op set's tv_per_sample and argmin as match_flows decides (a tie keeps x,
        as forward_with_flip does).  Otherwise input_img (already flipped by the caller, e.g. by a cluster classifier)
        runs once (N images) with warp_policy.  The forward samples at the flow size; at another output_resolution the
        congealed image is sampled again on the grid resized as the flow head resizes it (heads.py), with no second
        forward.  -> (flip (N,) bool or None, the congealed images (N, C, R, R) at output_resolution (None: the flow
        size), the sampling grid (N, F, F, 2) at the flow size: the grid uncongeal_points(output_resolution=None) reads)."""
        if not self.is_flow or not isinstance(self.stns[-1].warp_head, FlowHead):
            raise ValueError("congeal_and_grid needs a ComposedSTN whose last stage is a flow")
        if infer_flip and self.num_heads > 1:
            raise ValueError("congeal_and_grid: a clustering STN takes its flips from the cluster classifier")
        n = input_img.size(0)
        x = torch.cat([input_img, input_img.flip(3,)], 0) if infer_flip else input_img
        out, grid, delta = self.forward(x, return_warp=True, return_flow=True, iters=iters, padding_mode=padding_mode,
                                        warp_policy=warp_policy)
        flip = None
        if infer_flip:
            tv = self.ops.tv_per_sample(delta)
            flip = torch.stack(tv.chunk(2), 0).argmin(dim=0).bool()
            rows = torch.arange(n, device=x.device) + n * flip.long()
            out, grid, x = out[rows], grid[rows], x[rows]
        if output_resolution is not None and output_resolution != grid.size(2):
            out = self.stns[-1].warp_head.warper(x, resize_grid(grid, output_resolution), padding_mode=padding_mode)
        return flip, out, grid

    def _matrix_flow_grid(self, input_img, iters=1, **stn_forward_kwargs):
        """forward(input_img) of a similarity -> flow STN, returning what point transfer reads from it: the similarity
        matrix (N, 2, 3), the residual flow (N, F, F, 2) and the composed sampling grid (N, F, F, 2).  The calls are
        forward's (same arguments, same order), so each output equals the one congeal_points / uncongeal_points get."""
        if self.transforms != ["similarity", "flow"] or self.num_heads > 1:
            raise ValueError("point transfer from one forward needs a single-head similarity -> flow ComposedSTN")
        sim, flow = self.stns
        out, _, matrix = sim(input_img, return_warp=True, return_flow=True, return_intermediates=False,
                             input_img_for_sampling=input_img, base_warp=None, output_resolution=self.stn_in_size,
                             unfold=False, iters=iters, alpha=None, warp_policy="cartesian", **stn_forward_kwargs)
        _, grid, delta = flow(out, return_warp=True, return_flow=True, return_intermediates=False,
                              input_img_for_sampling=input_img, base_warp=matrix, output_resolution=None, unfold=False,
                              iters=1, alpha=None, warp_policy="cartesian", **stn_forward_kwargs)
        return matrix, delta, grid

    def load_single_state_dict(self, state_dict, index, strict=True):
        return self.stns[index].load_state_dict(state_dict, strict)

    def load_several_state_dicts(self, state_dicts, indices, strict=True):
        assert len(state_dicts) == len(indices)
        for sd, index in zip(state_dicts, indices):
            self.load_single_state_dict(sd, index, strict)

    def load_state_dict(self, state_dict, strict=True):
        ignore = {"warp_head.one_hot"}
        for i in range(len(self.stns)):
            ignore.update({f"stns.{i}.input_downsample.kernel_horz", f"stns.{i}.input_downsample.kernel_vert",
                           f"stns.{i}.warp_head.rebias"})
        return super().load_state_dict({k: v for k, v in state_dict.items() if k not in ignore}, False)
