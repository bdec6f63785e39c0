"""Congealing visualisations: the average congealed image, the average-image animation and the congealing animation of a
few images with their dense labels tracked (reference applications/vis_correspondence.py and
applications/propagate_to_images.py:81-104).  The reference's `args` fields are keyword arguments here, as in flips.py.

The reference re-runs the flip inference and the STN for every frame of the average-image animation, although only the
lerp weight changes from one frame to the next.  Here every image runs through the STN three times in all (twice for the
flip decision, once for the grids of every stage) and every stage's frames come from one call per batch of the op set's
`mipmap_warp_lerp_mean` (sums over the batch, no per-sample frames written) or `mipmap_warp_lerp` (the congealed frames),
and the label points of a stage are tracked by one `track_points_lerp` launch instead of one Unfold per frame.

Quirks of the reference that published visuals come from, kept here:
  * without `vis_in_stages`, the average-image animation (`congealing_average_frames`) animates grids[0], the similarity
    stage, while the congealing animation (`smooth_congealing`) animates grids[-1], the full warp;
  * `average_congealed_image` averages whole batches until at least n_mean // world images are seen (run_loader_mean),
    so it may use more than n_mean images; it samples the flipped images, while the animations sample the unflipped
    images on flipped grids (create_average_image, smoothly_sample_image);
  * the point tracker's window positions beyond pad_grid's ring are Unfold's (0, 0) zero padding and stay candidates, and
    a window that leaves the padded grid wraps around in the flat index (see track_points_lerp).
"""
import math

import torch
import torch.nn.functional as F

from ..training import distributed as dist
from .flips import determine_flips

WARP_LEVELS = 3.5   # the reference's warper: MipmapWarp(3.5), border padding


def cosine_alphas(length, device):
    """The lerp weight of every frame, with the reference's float32 expression (vis_correspondence.py:192, :409)."""
    if length < 2:
        raise ValueError("an animation needs length >= 2 frames (the reference divides by length - 1), got %d" % length)
    a = [1 - 0.5 * (1 + torch.cos(torch.tensor(math.pi * i / (length - 1)))) for i in range(length)]
    return torch.stack(a).to(device)


def flip_grid(grid, flip_indices):
    """vis_correspondence.py:166-169: negate x where the image was flipped."""
    grid = grid.clone()
    grid[..., 0] = torch.where(flip_indices.view(1, -1, 1, 1), -grid[..., 0], grid[..., 0])
    return grid


def get_patch_size(length):
    """vis_correspondence.py:172-180: the tracking window grows as the animation gets shorter."""
    patch_size = math.ceil(9 * max(1, 240 / length))
    return patch_size + 1 if patch_size % 2 == 0 else patch_size


def _resize(grid, res):
    if res == grid.size(1):
        return grid
    return F.interpolate(grid.permute(0, 3, 1, 2), scale_factor=res / grid.size(1), mode="bilinear").permute(0, 2, 3, 1)


def _identity(n, res, like):
    """F.affine_grid of the identity, built on the CPU and moved as the reference does."""
    return F.affine_grid(torch.eye(2, 3).unsqueeze(0).repeat(n, 1, 1), (n, 3, res, res), align_corners=False).to(like)


def _flips(t, data, classifier, cluster, num_heads, no_flip_inference, iters, padding_mode):
    return determine_flips(t, classifier, data, cluster=cluster, num_heads=num_heads, no_flip_inference=no_flip_inference,
                           iters=iters, padding_mode=padding_mode)


def _num_stages(t, vis_in_stages):
    return len(t.stns) if hasattr(t, "stns") and vis_in_stages else 1


@torch.no_grad()
def average_congealed_image(t, loader, n_mean, classifier=None, cluster=None, num_heads=1, no_flip_inference=False,
                            output_resolution=None, iters=1, padding_mode="border"):
    """propagate_to_images.average + run_loader_mean(unfold=False) + utils/distributed.all_reduce: the mean of the
    congealed (flipped) images of whole batches until this rank has seen at least n_mean // world images, over all ranks.
    The sum is kept on the device instead of a host-side list of every congealed image.  -> (1, C, R, R)."""
    world = dist.get_world_size()
    acc, total = None, 0
    for x in loader:
        flipped, _, policy = _flips(t, x, classifier, cluster, num_heads, no_flip_inference, iters, padding_mode)
        out = t(flipped, warp_policy=policy, unfold=False, iters=iters, padding_mode=padding_mode,
                output_resolution=output_resolution)
        s = out.float().sum(dim=0, keepdim=True)
        acc = s if acc is None else acc + s
        total += x.size(0)
        if total >= n_mean // world:
            break
    if acc is None:
        raise ValueError("average_congealed_image: the loader yielded no images")
    num = dist.all_gather(torch.tensor([float(total)], device=acc.device)).sum()
    return dist.all_gather(acc).sum(dim=0, keepdim=True) / num


@torch.no_grad()
def congealing_average_frames(t, loader, n_mean, length=240, flip_length=40, vis_in_stages=False, stage_flip=False,
                              output_resolution=None, classifier=None, cluster=None, num_heads=1, no_flip_inference=False,
                              iters=1, padding_mode="border"):
    """The frames of average_and_congeal (vis_correspondence.py:384-419) before its `normalize`: frame t of a stage is
    the mean over n_mean images of the image warped by lerp(base, grid, alpha_t).  Stages: the flip (with stage_flip;
    flip_length frames, the identity lerped to the flipped identity), then every STN stage with vis_in_stages or else
    grids[0] alone (the similarity stage: the reference's quirk), length frames each, from the previous stage's grid (the
    identity for the first).  Every batch runs the flip decision and the STN once; each stage's frames are one
    `mipmap_warp_lerp_mean` call into a (F, C, R, R) sum, divided by n_mean // world and averaged over ranks.
    The loader yields (N, C, H, W) batches in a fixed order; output_resolution None: the images' size.  -> (F, C, R, R)."""
    world = dist.get_world_size()
    per_rank = n_mean // world
    if per_rank * world != n_mean:
        raise ValueError("n_mean (%d) must be divisible by the number of processes (%d)" % (n_mean, world))
    ops = t.ops
    num_stages = _num_stages(t, vis_in_stages) + int(stage_flip)
    lengths = [flip_length if (stage_flip and i == 0) else length for i in range(num_stages)]
    acc, alphas, identity, total = None, None, None, 0
    for data in loader:
        n_batch = data.size(0)
        if acc is None:
            if per_rank // n_batch != per_rank / n_batch:
                raise ValueError("the batch size (%d) must evenly divide the images each process needs (%d)" % (n_batch, per_rank))
            res = output_resolution or data.size(-1)
            acc = torch.zeros((sum(lengths), data.size(1), res, res), dtype=torch.float32, device=data.device)
            alphas = [cosine_alphas(n, data.device) for n in lengths]
            identity = _identity(1, res, data)
        flipped, flip_indices, policy = _flips(t, data, classifier, cluster, num_heads, no_flip_inference, iters, padding_mode)
        _, grids = t(flipped, warp_policy=policy, return_intermediates=True, iters=iters, padding_mode=padding_mode)
        n = min(n_batch, per_rank - total)
        f0 = 0
        for i in range(num_stages):
            warp_index = i - int(stage_flip)
            if warp_index >= 0:
                target = flip_grid(grids[warp_index], flip_indices)
                base = identity.repeat(n_batch, 1, 1, 1) if warp_index == 0 else grids[warp_index - 1]
                base = _resize(flip_grid(base, flip_indices), res)[:n]
            else:
                target = flip_grid(identity.repeat(n_batch, 1, 1, 1), flip_indices)
                base = identity
            target = _resize(target, res)[:n]
            ops.mipmap_warp_lerp_mean(data[:n], base, target, alphas[i], acc[f0:f0 + lengths[i]], WARP_LEVELS)
            f0 += lengths[i]
        total += n
        if total >= per_rank:
            break
    if total != per_rank:
        raise ValueError("needed %d images per process but the loader gave %d" % (per_rank, total))
    dist.synchronize()
    return torch.stack(dist.all_gather(acc / per_rank, cat=False), 0).mean(dim=0)


@torch.no_grad()
def smooth_congealing(t, data, label_points=None, resolution=256, length=240, flip_length=40, vis_in_stages=False,
                      stage_flip=False, output_resolution=None, classifier=None, cluster=None, num_heads=1,
                      no_flip_inference=False, iters=1, padding_mode="border"):
    """smoothly_congeal_and_propagate (vis_correspondence.py:208-298) with sample_images_and_points' label handling
    (:48-54): the congealing animation of `data` (N, C, H, W) and the dense label tracked through it.
    label_points: (P, 2) integer (x, y) pixel coordinates of the label in the congealed frame at `resolution`, or None.
    Stages: the flip (with stage_flip), then every STN stage with vis_in_stages or else grids[-1] alone (the full warp).
    The unflipped images are sampled on flipped grids.  The points are tracked forward from where the label lands in each
    image, then backward from the label itself, and the two runs are blended as the reference does (:279-287).
    -> (frames (F, N, C, R, R); points (stages * length, N, P, 2) fp32 pixel positions in the frames, or None;
        the label's unaligned-space pixel positions (N, P, 2) that the flip stage's splat uses, or None)."""
    ops = t.ops
    res = output_resolution or data.size(-1)
    n = data.size(0)
    flipped, flip_indices, policy = _flips(t, data, classifier, cluster, num_heads, no_flip_inference, iters, padding_mode)
    _, grids = t(flipped, return_intermediates=True, warp_policy=policy, padding_mode=padding_mode, iters=iters)
    if not vis_in_stages:
        grids = [grids[-1]]
    grids = flip_grid(torch.stack(grids), flip_indices.view(1, -1, 1, 1))
    flow_size = grids.size(2)
    if res != flow_size:
        g = grids.reshape(-1, flow_size, flow_size, 2)
        g = F.interpolate(g.permute(0, 3, 1, 2), scale_factor=res / flow_size, mode="bilinear").permute(0, 2, 3, 1)
        grids = g.reshape(-1, n, res, res, 2)
    identity = _identity(n, res, data)
    num_stages = grids.size(0)
    flipping = flip_grid(identity, flip_indices)
    grids = torch.cat([flipping.unsqueeze(0), grids], 0)
    alphas = cosine_alphas(length, data.device)
    frames = []
    if stage_flip:
        frames.append(ops.mipmap_warp_lerp(data, identity, flipping, cosine_alphas(flip_length, data.device), WARP_LEVELS)[0])
    for i in range(num_stages):
        frames.append(ops.mipmap_warp_lerp(data, grids[i], grids[i + 1], alphas, WARP_LEVELS)[0])
    frames = torch.cat(frames, 0)
    if label_points is None:
        return frames, None, None
    # sample_images_and_points (:48-54) and :240-253
    points = label_points.to(data.device).unsqueeze(0).repeat(n, 1, 1)
    points_normalized = _normalize(points, res, resolution)
    if resolution != res:
        points = _unnormalize(_normalize(points, res, resolution), res, res).round().long()
    lookup = ops.grid_sample(grids[-1].permute(0, 3, 1, 2).contiguous(), points_normalized.unsqueeze(2).float().contiguous(),
                             "border")
    normalized_unaligned = lookup.squeeze(3).permute(0, 2, 1).contiguous()
    unaligned = _unnormalize(normalized_unaligned, res, res)
    centers = unaligned.round().long().clamp(0, res - 1)
    centers[..., 0] = torch.where(flip_indices.view(-1, 1), res - 1 - centers[..., 0], centers[..., 0])
    patch = get_patch_size(length)
    propagated = []
    for i in range(num_stages):
        track, centers = ops.track_points_lerp(grids[i], grids[i + 1], alphas, normalized_unaligned, centers, patch)
        propagated.append(track.float())
    congealed_centers = points.long()
    blend = torch.linspace(0, 1, steps=length, device=data.device).view(length, 1, 1, 1)
    for i in range(num_stages):     # the reverse pass, congealed -> unaligned (:279-287)
        rev, congealed_centers = ops.track_points_lerp(grids[-i - 1], grids[-i - 2], alphas, normalized_unaligned,
                                                       congealed_centers, patch)
        propagated[-i - 1].lerp_(rev.float().flip(0), blend)
    return frames, torch.cat(propagated, 0), unaligned


def _normalize(points, res, out_res):
    return points.div(out_res - 1).add(-0.5).mul(2).mul((res - 1) / res)


def _unnormalize(points, res, out_res):
    return points.div((res - 1) / res).div(2).add(0.5).mul(out_res - 1)
